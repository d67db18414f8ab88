"""Generate tests/golden/resize_*.npz from the REAL reference TimeSformer fed clips of other sizes than img_size.

Run in the build container only (needs /root/reference):

    python oracle/make_resize_golden.py [resize_divided] [resize_space_only] [resize_joint]

Uses the reference import and helpers of oracle/make_golden.py.  For every case the script also runs the restatement
in oracle/resize_oracle.py and asserts agreement (eval and train outputs to 1e-12, every gradient to 1e-9), i.e. this
script is what pins that oracle.
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle.make_golden import GOLD, import_reference, pack_grads, randomize, rel  # noqa: E402


def save_split(name, save, budget=700_000):
    """np.savez_compressed in <name>.npz, <name>.1.npz, ... with at most `budget` raw bytes per file (tests/conftest.py
    load_golden reads them back together)."""
    parts, cur, size = [], {}, 0
    for k, v in save.items():
        n = np.asarray(v).nbytes
        if cur and size + n > budget:
            parts.append(cur)
            cur, size = {}, 0
        cur[k] = v
        size += n
    parts.append(cur)
    for i, part in enumerate(parts):
        np.savez_compressed(os.path.join(GOLD, name + ('' if i == 0 else f'.{i}') + '.npz'), **part)


def resize_family(vt, name, cfg, attention_type, seed, cases):
    """One model per attention type; each case is an input size (h, w), a batch B and whether the position tables are
    learnable.  Inputs are int8 codes / 32 (stored as codes).  Stores eval output, seeded train output and every
    gradient (pos_embed included) per case."""
    from oracle import resize_oracle as RO
    oracle_fwd = RO.FORWARD[attention_type]
    torch.manual_seed(seed)
    kw = dict(num_frames=cfg['num_frames'], img_size=cfg['img_size'], patch_size=cfg['patch_size'],
              embed_dims=cfg['embed_dims'], num_heads=cfg['num_heads'],
              num_transformer_layers=cfg['num_transformer_layers'], attention_type=attention_type)
    m = vt.TimeSformer(**kw)
    randomize(m, seed + 1)
    sd = {k: v.detach().clone().float().double() for k, v in m.state_dict().items()}
    save = {'sd::' + k: v.float().numpy() for k, v in sd.items()}
    save.update({'cfg_' + k: np.int64(v) for k, v in cfg.items()})
    save['cases'] = np.array([c[0] for c in cases])
    g = torch.Generator().manual_seed(seed + 2)
    for ci, (tag, (h, w), B, learnable) in enumerate(cases):
        if learnable:
            ref = vt.TimeSformer(**kw).double()
            ref.load_state_dict(sd, strict=True)
            sdo = dict(sd)
        else:
            ref = vt.TimeSformer(use_learnable_pos_emb=False, **kw).double()
            ref.load_state_dict({k: v for k, v in sd.items() if k not in ('pos_embed', 'time_embed')}, strict=True)
            sdo = dict(sd, pos_embed=ref.pos_embed)            # the fp32 sine-cosine tables, resized in fp32 (:211)
            if attention_type != 'space_only':
                sdo['time_embed'] = ref.time_embed
        code = torch.randint(-128, 128, (B, cfg['num_frames'], 3, h, w), generator=g, dtype=torch.int8)
        x = code.double() / 32
        ref.eval()
        with torch.no_grad():
            y_eval = ref(x)
            assert rel(oracle_fwd(sdo, x, cfg), y_eval) < 1e-12
        ref.train()
        seed_tr = 5000 + 10 * seed + ci
        torch.manual_seed(seed_tr)
        y_tr = ref(x)
        wgt = torch.linspace(-1, 1, y_tr.numel(), dtype=torch.float64).reshape(y_tr.shape)
        (y_tr * wgt).sum().backward()
        grads = {n: p.grad.detach().clone() for n, p in ref.named_parameters()}
        assert ('pos_embed' in grads) == learnable
        sdg = {k: (v.clone().requires_grad_(True) if k in grads else v) for k, v in sdo.items()}
        torch.manual_seed(seed_tr)
        yo = oracle_fwd(sdg, x, cfg, training=True)
        (yo * wgt).sum().backward()
        assert rel(yo.detach(), y_tr.detach()) < 1e-12
        for n, gr in grads.items():
            assert rel(sdg[n].grad, gr) < 1e-9, (tag, n, rel(sdg[n].grad, gr))
        save[f'xq::{tag}'] = code.numpy()
        save[f'meta::{tag}'] = np.array([h, w, B, int(learnable), seed_tr], dtype=np.int64)
        save[f'out::{tag}::y_eval'] = y_eval.numpy()
        save[f'out::{tag}::y_train'] = y_tr.detach().numpy()
        sub = {}
        pack_grads(sub, grads)
        save.update({k.replace('::', f'::{tag}::', 1): v for k, v in sub.items()})
        print(f'[{name}:{tag}] {h}x{w} B={B} learnable={learnable}: oracle == reference (eval, train fwd, '
              f'all {len(grads)} grads)')
    save_split(name, save)


def main():
    _, vt, _ = import_reference()
    only = set(sys.argv[1:])
    want = lambda n: not only or n in only
    base = dict(img_size=32, patch_size=16, embed_dims=128, num_heads=2)   # D % 128 == 0: the row-map LayerNorm
    square = [('up48', (48, 48), 2, True), ('down16', (16, 16), 2, True),        # 2x2 grid -> 3x3 / 1x1
              ('h48w64', (48, 64), 2, True), ('h64w48', (64, 48), 2, True),      # both orientations of the axis quirk
              ('fixed_h48w64', (48, 64), 2, False)]                               # sine-cosine tables, no gradient
    if want('resize_divided'):
        # + 272 x 272: 17 x 17 = 289 patches, spatial attention over 290 tokens (past the single-pass kernels)
        resize_family(vt, 'resize_divided', dict(base, num_frames=2, num_transformer_layers=1), 'divided_space_time',
                      21, square + [('big272', (272, 272), 1, True)])
    if want('resize_space_only'):
        resize_family(vt, 'resize_space_only', dict(base, num_frames=3, num_transformer_layers=2), 'space_only', 22,
                      square)
    if want('resize_joint'):
        resize_family(vt, 'resize_joint', dict(base, num_frames=4, num_transformer_layers=1), 'joint_space_time', 23,
                      square)


if __name__ == '__main__':
    main()
