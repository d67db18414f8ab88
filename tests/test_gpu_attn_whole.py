"""The whole-problem attention kernels (attn_whole_*: one CTA per (b, h), operands resident in shared memory) against the
64-row tiled kernels they replace on the packed-qkv path, bit for bit.  -m gpu

VT_ATTN_WHOLE=0 selects the tiled kernels.  Both run through vt_attn_fwd / vt_attn_bwd with the tensor-core implementation
asked for by name, with the guarded buffers of test_gpu_attention_edges (NaN guard rows around every output, NaN rows past
the end of the inputs), so a store outside the outputs or a read past N shows as well as any changed bit.
"""
import pytest
import torch

from tests.test_gpu_attention_edges import TC, Guarded, _call, _lib, inputs, run_attn

pytestmark = pytest.mark.gpu

NS = [1, 17, 33, 63, 64, 65, 128, 129, 197, 255, 256]
OUTS = ('o', 'lse', 'dq', 'dk', 'dv')


def run(monkeypatch, whole, q, k, v, do, scale):
    monkeypatch.setenv('VT_ATTN_WHOLE', '1' if whole else '0')
    return run_attn(q, k, v, do, scale, TC)


def assert_same_bits(a, b, tag, sel=lambda x: x):
    for n in OUTS:
        x, y = sel(a[n]), sel(b[n])
        assert torch.equal(x, y), f'{tag} {n}: {int((x != y).sum())} of {x.numel()} differ, max {float((x - y).abs().max()):.3e}'


@pytest.mark.parametrize('Bp,H', [(1, 1), (2, 3)])
@pytest.mark.parametrize('N', NS)
def test_whole_matches_tiled_bitwise(monkeypatch, N, Bp, H):
    scale = 64 ** -0.5
    q, k, v, do = inputs(Bp, H, N, N, 64, scale, seed=N)
    assert_same_bits(run(monkeypatch, True, q, k, v, do, scale), run(monkeypatch, False, q, k, v, do, scale), f'N={N}')


@pytest.mark.parametrize('regime', ['benign', 'max_last'])
def test_whole_matches_tiled_at_the_spatial_shape(monkeypatch, regime):
    """TimeSformer / ViViT spatial attention: 64 frames x 12 heads, 197 tokens, with
    ordinary logits and with the running max moving in the last key tile"""
    scale = 64 ** -0.5
    q, k, v, do = inputs(64, 12, 197, 197, 64, scale, regime, seed=5)
    assert_same_bits(run(monkeypatch, True, q, k, v, do, scale), run(monkeypatch, False, q, k, v, do, scale), regime)


@pytest.mark.parametrize('N', [65, 197, 256])
def test_whole_forward_without_lse(monkeypatch, N):
    """the forward-only form (lse = NULL) writes the same ctx as the saving form, and no lse"""
    lib_, _ = _lib()
    Bp, H, hd = 2, 3, 64
    d = H * hd
    q, k, v, _ = inputs(Bp, H, N, N, hd, hd ** -0.5, seed=3)
    qkv = Guarded(Bp * N, 3 * d, torch.bfloat16)
    qkv.inner.view(Bp * N, 3, H, hd).copy_(torch.stack([x.permute(0, 2, 1, 3).reshape(Bp * N, H, hd) for x in (q, k, v)], 1)
                                          .to(torch.bfloat16).cuda())
    ctxs = {}
    for whole in (True, False):
        for want_lse in (True, False):
            monkeypatch.setenv('VT_ATTN_WHOLE', '1' if whole else '0')
            ctx, lse = Guarded(Bp * N, d, torch.bfloat16), Guarded(Bp * H, N, torch.float32)
            p = lib_.AttnFwdParams()
            p.qkv, p.ctx, p.lse, p.probs = qkv.inner.data_ptr(), ctx.inner.data_ptr(), lse.inner.data_ptr() if want_lse else None, None
            p.Bp, p.N, p.H, p.hd, p.scale, p.impl = Bp, N, H, hd, hd ** -0.5, TC
            _call('vt_attn_fwd', p, 'vt_attn_fwd')
            ctx.check('ctx')
            if not want_lse:
                assert bool(torch.isnan(lse.buf).all()), 'lse written by the forward-only form'
            ctxs[whole, want_lse] = ctx.inner.clone()
    ref = ctxs[False, True]
    for key, c in ctxs.items():
        assert torch.equal(c.view(torch.int16), ref.view(torch.int16)), key


def test_whole_problems_are_independent(monkeypatch):
    """scaling every other (b, h) problem's q, k, v and dO by 50 leaves problem (0, 0)'s bits unchanged"""
    scale = 64 ** -0.5
    q, k, v, do = inputs(3, 2, 197, 197, 64, scale, seed=11)
    base = run(monkeypatch, True, q, k, v, do, scale)
    mask = torch.full((3, 2, 1, 1), 50.0, dtype=torch.float64)
    mask[0, 0] = 1.0
    scaled = [(x * mask).to(torch.bfloat16).double() for x in (q, k, v, do)]
    other = run(monkeypatch, True, *scaled, scale)
    assert_same_bits(base, other, 'problem (0, 0)', sel=lambda x: x[0, 0])


def test_whole_runs_repeat_bitwise(monkeypatch):
    scale = 64 ** -0.5
    q, k, v, do = inputs(8, 12, 197, 197, 64, scale, seed=2)
    assert_same_bits(run(monkeypatch, True, q, k, v, do, scale), run(monkeypatch, True, q, k, v, do, scale), 'repeat')


def test_auto_takes_the_whole_kernels(monkeypatch):
    """automatic choice at N = 197 equals the tensor-core implementation by name, whole kernels on"""
    from tests.test_gpu_attention_edges import AUTO
    monkeypatch.setenv('VT_ATTN_WHOLE', '1')
    scale = 64 ** -0.5
    q, k, v, do = inputs(2, 2, 197, 197, 64, scale, seed=4)
    assert_same_bits(run_attn(q, k, v, do, scale, AUTO), run_attn(q, k, v, do, scale, TC), 'auto')
