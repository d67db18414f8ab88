"""CUDA hot path vs the oracle / reference goldens at module level.  -m gpu

Tolerance contract (SURVEY.md §8c, measured on the reference itself): bf16 operands with fp32
accumulation and an fp32 residual stream give <= 1e-3 rel-L2 on residual-inclusive block outputs;
gradients and end-to-end outputs are gated at 1.5x the error the *reference* shows under bf16 autocast
(computed here on the CPU with the oracle under torch.autocast) plus a small floor.
"""
import pytest
import torch

from tests.conftest import check_grads, rel_err

pytestmark = pytest.mark.gpu


def build_ts(cfg, sd, dev='cuda'):
    from videotransformer_pytorch_b200 import TimeSformer
    m = TimeSformer(num_frames=cfg['num_frames'], img_size=cfg['img_size'], patch_size=cfg['patch_size'],
                    embed_dims=cfg['embed_dims'], num_heads=cfg['num_heads'],
                    num_transformer_layers=cfg['num_transformer_layers'], attention_type='divided_space_time')
    m.load_state_dict(sd, strict=True)
    return m.to(dev)


def test_timesformer_hd64_golden_eval_and_train(golden):
    g = golden('timesformer_hd64')
    m = build_ts(g.cfg, g.sd).eval()
    x = g.x.cuda()
    with torch.no_grad():
        y = m(x)
        tok, _ = m.prepare_tokens(x)
        attn = m.get_last_selfattention(x)
    e_tok, e_y, e_attn = rel_err(tok.cpu(), g.out['tokens']), rel_err(y.cpu(), g.out['y_eval']), rel_err(attn.cpu(), g.out['last_attn'])
    print(f'hd64 golden: tokens {e_tok:.2e}  y_eval {e_y:.2e}  last_attn {e_attn:.2e}')
    assert e_tok < 3e-3 and e_y < 1.5e-2 and e_attn < 1e-2
    m.train()
    xg = x.clone().requires_grad_(True)
    torch.manual_seed(g.train_seed)
    yt = m(xg)
    e_tr = rel_err(yt.detach().cpu(), g.out['y_train'])
    (yt.double() * g.out['loss_w'].cuda()).sum().backward()
    e_dx = rel_err(xg.grad.cpu(), g.out['dx'])
    print(f'hd64 golden: y_train {e_tr:.2e}  dx {e_dx:.2e}')
    assert e_tr < 1.5e-2 and e_dx < 3e-2
    worst = check_grads({n: p.grad for n, p in m.named_parameters()}, g, 3e-2)
    print(f'hd64 golden: worst small-grad rel err {worst:.2e}')


def _autocast_err(fn_fp64, fn_ac):
    """reference-under-bf16-autocast error of the same computation (CPU)."""
    with torch.no_grad():
        ref = fn_fp64()
    with torch.no_grad(), torch.autocast('cpu', dtype=torch.bfloat16):
        ac = fn_ac()
    return ref, rel_err(ac.float(), ref)


@pytest.mark.parametrize('B', [1, 2])
def test_blocks_at_timesformer_b_shape(B):
    """One full TimeSformer-B layer (D=768, H=12, T=8, P=196) sub-block by sub-block vs the fp64 oracle."""
    from oracle import vt_oracle as O
    from videotransformer_pytorch_b200.transformer import BasicTransformerBlock
    cfg = dict(O.TIMESFORMER_B, num_transformer_layers=1)
    sd = O.random_timesformer_state(cfg, seed=3)
    D, H, T, P = 768, 12, 8, 196
    blk = BasicTransformerBlock(embed_dims=D, num_heads=H, num_frames=T, hidden_channels=4 * D,
                                operator_order=['time_attn', 'space_attn', 'ffn'], dpr=0.0)
    pre = 'transformer_layers.layers.0.'
    blk.load_state_dict({k[len(pre):]: v for k, v in sd.items() if k.startswith(pre)}, strict=True)
    blk = blk.cuda().train()
    torch.manual_seed(0)
    x = torch.randn(B, 1 + P * T, D)
    sd64 = {k: v.double() for k, v in sd.items()}
    sd32 = sd
    steps = [('temporal', lambda s, t: O.divided_temporal(t, s, pre + 'attentions.0.', T, H, 0.0, False), blk.attentions[0]),
             ('spatial', lambda s, t: O.divided_spatial(t, s, pre + 'attentions.1.', T, H, 0.0, False), blk.attentions[1]),
             ('ffn', lambda s, t: O.ffn_prenorm(t, s, pre + 'ffns.0.', 0.0, False), blk.ffns[0])]
    cur = x
    for name, fn, mod in steps:
        ref, ac_err = _autocast_err(lambda: fn(sd64, cur.double()), lambda: fn(sd32, cur))
        with torch.no_grad():
            got = mod(cur.cuda())
        e = rel_err(got.cpu(), ref)
        print(f'[B={B}] {name}: rel-L2 {e:.2e} (reference under bf16 autocast: {ac_err:.2e})')
        assert e < 1e-3, (name, e)
        cur = ref.float()


def test_layer_backward_at_timesformer_b_shape():
    from oracle import vt_oracle as O
    from videotransformer_pytorch_b200.transformer import BasicTransformerBlock
    cfg = dict(O.TIMESFORMER_B, num_transformer_layers=1)
    sd = O.random_timesformer_state(cfg, seed=4)
    D, H, T, P, B = 768, 12, 8, 196, 1
    pre = 'transformer_layers.layers.0.'
    blk = BasicTransformerBlock(embed_dims=D, num_heads=H, num_frames=T, hidden_channels=4 * D,
                                operator_order=['time_attn', 'space_attn', 'ffn'], dpr=0.0)
    blk.load_state_dict({k[len(pre):]: v for k, v in sd.items() if k.startswith(pre)}, strict=True)
    blk = blk.cuda().train()
    torch.manual_seed(1)
    x = torch.randn(B, 1 + P * T, D)
    w = torch.randn(B, 1 + P * T, D) / 40

    def run(sdx, xx, dtype):
        s = {k: v.to(dtype).requires_grad_(True) for k, v in sdx.items() if k.startswith(pre)}
        xx = xx.detach().clone().to(dtype).requires_grad_(True)
        y = O.container(xx, s, 'transformer_layers.', 1, ['time_attn', 'space_attn', 'ffn'], T, H, False)
        (y * w.to(y.dtype)).sum().backward()
        return y.detach(), xx.grad, {k: v.grad for k, v in s.items()}

    y64, dx64, g64 = run(sd, x, torch.float64)
    with torch.autocast('cpu', dtype=torch.bfloat16):
        yac, dxac, gac = run(sd, x, torch.float32)
    xg = x.detach().clone().cuda().requires_grad_(True)
    y = blk(xg)
    (y * w.cuda()).sum().backward()
    e_y, e_dx = rel_err(y.detach().cpu(), y64), rel_err(xg.grad.cpu(), dx64)
    print(f'layer: y {e_y:.2e} (ref-autocast {rel_err(yac.float(), y64):.2e})  dx {e_dx:.2e} (ref-autocast {rel_err(dxac, dx64):.2e})')
    assert e_y < 1e-3
    assert e_dx < max(1.5 * rel_err(dxac, dx64), 5e-3)
    for n, p in blk.named_parameters():
        ref = g64[pre + n]
        e, eac = rel_err(p.grad.cpu(), ref), rel_err(gac[pre + n], ref)
        print(f'  grad {n}: {e:.2e} (ref-autocast {eac:.2e})')
        assert e < max(1.5 * eac, 1e-2), (n, e, eac)


def test_vivit_small_vs_oracle():
    from oracle import vt_oracle as O
    from videotransformer_pytorch_b200 import ViViT
    torch.manual_seed(5)
    m = ViViT(num_frames=8, img_size=48, patch_size=16, embed_dims=128, num_heads=2, num_transformer_layers=2)
    with torch.no_grad():
        for n, p in m.named_parameters():
            if 'norm' in n or n.endswith('bias'):
                p.add_(torch.randn_like(p) * 0.05)
    sd = {k: v.detach().clone() for k, v in m.state_dict().items()}
    cfg = dict(num_frames_in=8, img_size=48, patch_size=16, embed_dims=128, num_heads=2, num_transformer_layers=2)
    x = torch.randn(3, 8, 3, 48, 48)
    with torch.no_grad():
        ref = O.vivit_forward({k: v.double() for k, v in sd.items()}, x.double(), cfg)
        got = m.cuda().eval()(x.cuda())
    e = rel_err(got.cpu(), ref)
    print(f'vivit small eval: {e:.2e}')
    assert e < 1.5e-2
    # train step incl. DropPath RNG parity and the cls-gather quirk, grads vs fp64 oracle
    m.train()
    torch.manual_seed(77)
    y = m(x.cuda())
    y.square().sum().backward()
    sdg = {k: v.double().requires_grad_(True) for k, v in sd.items()}
    torch.manual_seed(77)
    yo = O.vivit_forward(sdg, x.double(), cfg, training=True)
    yo.square().sum().backward()
    assert rel_err(y.detach().cpu(), yo.detach()) < 1.5e-2
    worst = max(rel_err(p.grad.cpu(), sdg[n].grad) for n, p in m.named_parameters())
    print(f'vivit small train: worst grad rel err {worst:.2e}')
    assert worst < 5e-2


def test_no_silent_fallback_on_cpu_tensor():
    from videotransformer_pytorch_b200 import FFNWithPreNorm
    f = FFNWithPreNorm(embed_dims=128, hidden_channels=512)
    with pytest.raises(RuntimeError):
        f(torch.randn(2, 4, 128))


def test_space_only_small_vs_oracle():
    from oracle import vt_oracle as O
    from videotransformer_pytorch_b200 import TimeSformer
    torch.manual_seed(6)
    cfg = dict(num_frames=4, img_size=48, patch_size=16, embed_dims=128, num_heads=2, num_transformer_layers=2)
    m = TimeSformer(attention_type='space_only', **cfg)
    sd = {k: v.detach().clone() for k, v in m.state_dict().items()}
    x = torch.randn(2, 4, 3, 48, 48)
    with torch.no_grad():
        ref = O.timesformer_space_only_forward({k: v.double() for k, v in sd.items()}, x.double(), cfg)
        got = m.cuda().eval()(x.cuda())
    e = rel_err(got.cpu(), ref)
    print(f'space_only small eval: {e:.2e}')
    assert e < 1.5e-2


def test_joint_space_time_vs_golden(golden):
    """joint_space_time with 289 tokens per clip (past the single-pass kernels): tiled tensor-core attention, head dim 64."""
    from videotransformer_pytorch_b200 import TimeSformer
    g = golden('timesformer_joint_n289')
    c = g.cfg
    m = TimeSformer(num_frames=c['num_frames'], img_size=c['img_size'], patch_size=c['patch_size'],
                    embed_dims=c['embed_dims'], num_heads=c['num_heads'],
                    num_transformer_layers=c['num_transformer_layers'], attention_type='joint_space_time')
    m.load_state_dict(g.sd, strict=True)
    m = m.cuda().eval()
    with torch.no_grad():
        e = rel_err(m(g.x.cuda()).cpu(), g.out['y_eval'])
    print(f'joint_space_time n289 eval: {e:.2e}')
    assert e < 1.5e-2
    m.train()
    torch.manual_seed(g.train_seed)
    y = m(g.x.cuda())
    assert rel_err(y.detach().cpu(), g.out['y_train']) < 1.5e-2
    (y.double() * g.out['loss_w'].cuda()).sum().backward()
    worst = 0.0
    for n, p in m.named_parameters():
        if n in g.grad:
            worst = max(worst, rel_err(p.grad.cpu(), g.grad[n]))
        elif n in g.gradsum:
            ref = g.gradsum[n]
            worst = max(worst, abs(p.grad.double().norm().item() - ref[1]) / ref[1])
    print(f'joint_space_time n289 train: worst grad rel err {worst:.2e}')
    assert worst < 5e-2


@pytest.mark.parametrize('name,attention_type', [('vivit_joint_hd64', 'joint_space_time'),
                                                 ('vivit_divided_hd64', 'divided_space_time')])
def test_vivit_joint_and_divided_variants_vs_golden(golden, name, attention_type):
    """ViViT models 1 / 3 (reference video_transformer.py:349-373) on the kernels vs goldens from the real reference."""
    from videotransformer_pytorch_b200 import ViViT
    g = golden(name)
    c = g.cfg
    m = ViViT(num_frames=c['num_frames_in'], img_size=c['img_size'], patch_size=c['patch_size'],
              embed_dims=c['embed_dims'], num_heads=c['num_heads'],
              num_transformer_layers=c['num_transformer_layers'], attention_type=attention_type)
    m.load_state_dict(g.sd, strict=True)
    m = m.cuda().eval()
    with torch.no_grad():
        e = rel_err(m(g.x.cuda()).cpu(), g.out['y_eval'])
    print(f'ViViT {attention_type} eval: {e:.2e}')
    assert e < 1.5e-2
    m.train()
    torch.manual_seed(g.train_seed)
    y = m(g.x.cuda())
    assert rel_err(y.detach().cpu(), g.out['y_train']) < 1.5e-2
    (y.double() * g.out['loss_w'].cuda()).sum().backward()
    worst = check_grads({n: p.grad for n, p in m.named_parameters()}, g, 5e-2)
    print(f'ViViT {attention_type} train: worst small-grad rel err {worst:.2e}')


def test_vivit_b_joint_space_time_1569_tokens_vs_oracle():
    """ViViT-B model 1 at 16x224 (1 + 196*8 = 1569 tokens per clip, tiled tensor-core attention), one layer, B=1."""
    from oracle import vt_oracle as O
    from videotransformer_pytorch_b200 import ViViT
    torch.manual_seed(8)
    kw = dict(num_frames=16, img_size=224, patch_size=16, embed_dims=768, num_heads=12, num_transformer_layers=1)
    m = ViViT(attention_type='joint_space_time', **kw)
    sd = {k: v.detach().clone() for k, v in m.state_dict().items()}
    cfg = dict(img_size=224, patch_size=16, embed_dims=768, num_heads=12, num_transformer_layers=1)
    x = torch.randn(1, 16, 3, 224, 224)
    with torch.no_grad():
        ref = O.vivit_variant_forward({k: v.double() for k, v in sd.items()}, x.double(), cfg, 'joint_space_time')
        got = m.cuda().eval()(x.cuda())
    e = rel_err(got.cpu(), ref)
    print(f'ViViT-B joint_space_time 1569 tokens: {e:.2e}')
    assert e < 5e-3
