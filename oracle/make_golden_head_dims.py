"""Golden vectors for TimeSformer and ViViT at head widths 32, 96 and 128, from the REAL reference classes.

    python oracle/make_golden_head_dims.py [name ...]

Each case builds the reference model with `embed_dims` and `num_heads` chosen for the width (D = 128 with 4 heads: 32,
D = 384 with 4 heads: 96, D = 128 with 1 head: 128; D stays a multiple of 128 for the row-map LayerNorm), loads a state
drawn by `random_state` from a seed, and records in fp64 the eval output, the train-mode output with seeded DropPath,
the input gradient of frame 0, every parameter gradient and rows of the last-layer attention map.  The state and the
input are not stored: `random_state` and `random_input` regenerate them from the seed, so the fixtures stay small at
D = 384.  The eval output is also checked against the oracle restatement (oracle/vt_oracle.py).
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle.make_golden import GOLD, import_reference, pack_grads, rel  # noqa: E402

WIDTHS = {32: dict(embed_dims=128, num_heads=4), 96: dict(embed_dims=384, num_heads=4), 128: dict(embed_dims=128, num_heads=1)}
# (model, attention_type, geometry, rows of the last attention map kept: every `attn_step`-th query row)
KINDS = {
    # temporal pass N = 8 (warp-per-problem kernel), spatial pass N = 37 (tiled tensor-core kernels), probs at N = 37
    'ts_divided': ('TimeSformer', 'divided_space_time', dict(num_frames=8, img_size=96), 1),
    # one 289-token pass per clip: tiled kernels past 256 tokens, probabilities from the row-tile kernel
    'ts_joint': ('TimeSformer', 'joint_space_time', dict(num_frames=8, img_size=96), 7),
    # spatial N = 5, temporal N = 9 (generic kernels)
    'vivit_fact': ('ViViT', 'fact_encoder', dict(num_frames=16, img_size=32), 1),
    # temporal N = 4 (generic), spatial N = 10 (generic), on tubelets
    'vivit_divided': ('ViViT', 'divided_space_time', dict(num_frames=8, img_size=48), 1),
}
SEEDS = {'ts_divided': 21, 'ts_joint': 22, 'vivit_fact': 23, 'vivit_divided': 24}


def case_names():
    return [f'{kind}_hd{hd}' for kind in KINDS for hd in WIDTHS]


def case_config(name):
    """-> (model class name, attention_type, constructor kwargs, attention row step, seed) of fixture `name`"""
    kind, hd = name.rsplit('_hd', 1)
    model, attention_type, geo, step = KINDS[kind]
    kw = dict(geo, patch_size=16, num_transformer_layers=1, attention_type=attention_type, **WIDTHS[int(hd)])
    return model, attention_type, kw, step, SEEDS[kind] * 1000 + int(hd)


def random_state(shapes, seed):
    """A state for the parameter names / shapes `shapes` (in state_dict order), fp32 values: matrices and convolutions
    N(0, 1 / fan_in), so the attention logits are O(1) at every width; LayerNorm weights 1 + N(0, 0.1^2), other vectors
    (biases) N(0, 0.05^2), tokens and embeddings N(0, 0.02^2)."""
    g = torch.Generator().manual_seed(seed)
    out = {}
    for n, shape in shapes.items():
        z = torch.randn(tuple(shape), generator=g, dtype=torch.float64)
        if 'token' in n or n.endswith('pos_embed') or n.endswith('time_embed'):
            v = 0.02 * z
        elif len(shape) >= 2:
            v = z * float(np.prod(shape[1:])) ** -0.5
        elif 'norm' in n and n.endswith('weight'):
            v = 1.0 + 0.1 * z
        else:
            v = 0.05 * z
        out[n] = v.float()
    return out


def random_input(kw, B, seed):
    g = torch.Generator().manual_seed(seed + 1)
    return torch.randn(B, kw['num_frames'], 3, kw['img_size'], kw['img_size'], generator=g, dtype=torch.float64).float()


def make_case(vt, name, B=1):
    from oracle import vt_oracle as O
    model, attention_type, kw, step, seed = case_config(name)
    cls = getattr(vt, model)
    m = cls(**kw)
    sd = random_state({k: tuple(v.shape) for k, v in m.state_dict().items()}, seed)
    m.load_state_dict(sd, strict=True)
    m = m.double()
    x = random_input(kw, B, seed).double()
    save = {'seed': np.int64(seed), 'B': np.int64(B), 'train_seed': np.int64(seed + 7), 'attn_step': np.int64(step)}
    m.eval()
    with torch.no_grad():
        y_eval = m(x)
        attn = m.get_last_selfattention(x)
    sd64 = {k: v.double() for k, v in sd.items()}
    cfg = dict(kw, num_frames_in=kw['num_frames'])
    with torch.no_grad():
        if model == 'TimeSformer' and attention_type == 'divided_space_time':
            y_o = O.timesformer_forward(sd64, x, cfg)
        elif model == 'TimeSformer':
            y_o = O.timesformer_joint_forward(sd64, x, cfg)
        elif attention_type == 'fact_encoder':
            y_o = O.vivit_forward(sd64, x, cfg)
        else:
            y_o = O.vivit_variant_forward(sd64, x, cfg, attention_type)
    assert rel(y_o, y_eval) < 1e-12, (name, rel(y_o, y_eval))
    m.train()
    xg = x.clone().requires_grad_(True)
    torch.manual_seed(seed + 7)
    y_tr = m(xg)
    w = torch.linspace(-1, 1, y_tr.numel(), dtype=torch.float64).reshape(y_tr.shape)
    (y_tr * w).sum().backward()
    grads = {n: p.grad.detach().clone() for n, p in m.named_parameters()}
    save['out::y_eval'] = y_eval.numpy()
    save['out::y_train'] = y_tr.detach().numpy()
    save['out::dx0'] = xg.grad[:, 0].float().numpy()                   # input gradient of frame 0
    save['out::last_attn_rows'] = attn[..., ::step, :].float().numpy()
    save['attn_shape'] = np.asarray(attn.shape, dtype=np.int64)
    pack_grads(save, grads)
    path = os.path.join(GOLD, name + '.npz')
    np.savez_compressed(path, **save)
    print(f'[{name}] {model} {attention_type} D={kw["embed_dims"]} H={kw["num_heads"]}: y {tuple(y_eval.shape)}, '
          f'attention {tuple(attn.shape)}, {len(grads)} grads, {os.path.getsize(path) / 1024:.0f} KB')


def main():
    _, vt, _ = import_reference()
    only = set(sys.argv[1:])
    for name in case_names():
        if not only or name in only:
            make_case(vt, name)


if __name__ == '__main__':
    main()
