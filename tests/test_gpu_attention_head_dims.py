"""Packed-qkv attention (vt_attn_*) at head widths 32, 96 and 128, row by row against fp64, and TimeSformer / ViViT at
those widths against fixtures from the reference classes.  -m gpu

The kernel checks are those of tests/test_gpu_attention_edges.py (its drivers and gates, unchanged): NaN-guarded outputs
and inputs, every output row within the budget the CPU model of the same kernel (tests/attn_mma_emu.py) sets, the
tensor-core kernels also close to that model directly.  Each sequence length runs every implementation the ABI offers
for it: the generic kernels (N <= 256), the tensor-core kernels (any N) and the warp-per-problem kernel (N = 8).
"""
import pytest
import torch

from tests import attn_mma_emu as AE
from tests import head_dim_goldens as HG
from tests import test_gpu_attention_edges as E

pytestmark = pytest.mark.gpu

WIDTHS = [32, 96, 128]
EDGE_N = [1, 8, 9, 17, 32, 33, 64, 65, 197, 256, 257, 1569]


def _batch(N):
    return (1, 2) if N > 1000 else (2, 3)


@pytest.mark.parametrize('impl', [E.SIMT, E.TC, E.WARP8])
@pytest.mark.parametrize('N', EDGE_N)
@pytest.mark.parametrize('hd', WIDTHS)
def test_attn_packed_each_implementation_at_head_width(hd, N, impl):
    if impl == E.WARP8 and N != 8:
        pytest.skip('the warp-per-problem kernel takes N = 8 only')
    if impl == E.SIMT and N > 256:
        pytest.skip('the generic kernel takes N <= 256 only')
    if impl == E.SIMT and hd == 128 and N == 256:
        pytest.skip('the generic backward holds Q, K, V, dO of 256 rows at width 128 in no SM (refusal checked below)')
    scale = hd ** -0.5
    B, H = _batch(N)
    q, k, v, do = E.inputs(B, H, N, N, hd, scale, seed=N * 3 + hd + impl)
    got = E.run_attn(q, k, v, do, scale, impl)
    E.check_against_fp64(f'attn impl{impl} hd{hd} N{N}', got, q, k, v, do, scale, 'bf16' if impl == E.TC else 'bf16_out', True)


@pytest.mark.parametrize('N', EDGE_N)
@pytest.mark.parametrize('hd', WIDTHS)
def test_attn_packed_auto_dispatch_at_head_width(hd, N):
    """impl 0 picks the same kernel at every width: bitwise the results of the implementation asked for by name"""
    B, H = _batch(N)
    q, k, v, do = E.inputs(B, H, N, N, hd, hd ** -0.5, seed=N + hd)
    a, b = E.run_attn(q, k, v, do, hd ** -0.5, E.AUTO), E.run_attn(q, k, v, do, hd ** -0.5, E.picked(N))
    for n in a:
        assert torch.equal(a[n], b[n]), (hd, N, n)


@pytest.mark.parametrize('regime', AE.REGIMES)
@pytest.mark.parametrize('hd', WIDTHS)
def test_attn_packed_tensor_core_logit_regimes_at_head_width(hd, regime):
    q, k, v, do = E.inputs(2, 2, 197, 197, hd, 0.05, regime, seed=hd)
    got = E.run_attn(q, k, v, do, 0.05, E.TC)
    E.check_against_fp64(f'attn tc hd{hd} {regime}', got, q, k, v, do, 0.05, 'bf16', True)


def run_probs(q, k, scale, impl):
    """probabilities of vt_attn_fwd into a guarded [Bp, H, N, N] output -> CPU fp64"""
    lib_, _ = E._lib()
    Bp, H, N, hd = q.shape
    d = H * hd
    qkv = E.Guarded(Bp * N, 3 * d, torch.bfloat16)
    qkv.inner.view(Bp * N, 3, H, hd).copy_(torch.stack([x.permute(0, 2, 1, 3).reshape(Bp * N, H, hd) for x in (q, k, k)], 1)
                                          .to(torch.bfloat16).cuda())
    ctx, probs = E.Guarded(Bp * N, d, torch.bfloat16), E.Guarded(Bp * H * N, N, torch.float32)
    p = lib_.AttnFwdParams()
    p.qkv, p.ctx, p.lse, p.probs = qkv.inner.data_ptr(), ctx.inner.data_ptr(), None, probs.inner.data_ptr()
    p.Bp, p.N, p.H, p.hd, p.scale, p.impl = Bp, N, H, hd, scale, impl
    E._call('vt_attn_fwd', p, 'vt_attn_fwd')
    ctx.check('ctx')
    probs.check('probs')
    return probs.inner.view(Bp, H, N, N).double().cpu()


@pytest.mark.parametrize('N', [9, 197, 256, 257, 1569])
@pytest.mark.parametrize('hd', WIDTHS)
def test_attn_probabilities_at_head_width(hd, N):
    """the probability output (get_last_selfattention): the generic kernel up to 256 tokens, the row-tile kernel past
    them; fp32 scores of bf16 operands, so each row is within a few fp32 ulps of the fp64 softmax"""
    B, H = _batch(N)
    q, k, _, _ = E.inputs(B, H, N, N, hd, hd ** -0.5, seed=N + 7 * hd)
    got = run_probs(q, k, hd ** -0.5, E.AUTO)
    ref = torch.softmax(q @ k.transpose(-1, -2) * hd ** -0.5, -1)
    err = float(((got - ref).norm(dim=-1) / ref.norm(dim=-1)).max())
    assert err < 1e-5, (hd, N, err)


def test_attn_packed_refusals_at_head_width():
    q, k, v, do = E.inputs(1, 1, 256, 256, 128, 0.1)
    with pytest.raises(RuntimeError, match='N=256 at head dim 128 needs .* bytes of shared memory'):
        E.run_attn(q, k, v, do, 0.1, E.SIMT)
    for hd in (48, 80, 160):
        q, k, v, do = E.inputs(1, 1, 9, 9, hd, 0.1)
        for impl in (E.AUTO, E.SIMT, E.TC):
            with pytest.raises(RuntimeError, match=fr'head dim {hd} unsupported \(32, 64, 96 or 128\)'):
                E.run_attn(q, k, v, do, 0.1, impl)


# ---- TimeSformer / ViViT at the new widths against the reference ----------------------------------------------------------
@pytest.mark.parametrize('name', HG.NAMES)
def test_head_dim_golden_eval_and_train(name):
    """the tolerances of the width-64 goldens (tests/test_gpu_modules.py): features 1.5e-2, last-layer attention 1e-2,
    input gradient 3e-2, parameter gradients 3e-2 (divided TimeSformer) or 5e-2"""
    g = HG.HeadDimGolden(name)
    grad_tol = 3e-2 if name.startswith('ts_divided') else 5e-2
    err = HG.run(g, 'cuda', grad_tol)
    print(f'[head dims] {name}: ' + ', '.join(f'{k} {v:.2e}' for k, v in err.items()))
    assert err['y_eval'] < 1.5e-2 and err['y_train'] < 1.5e-2, err
    assert err['last_attn'] < 1e-2, err
    assert err['dx'] < 3e-2, err


@pytest.mark.parametrize('name', [n for n in HG.NAMES if not n.startswith('vivit_fact')])
def test_head_dim_golden_fp8_forward(name):
    """the forward-only fp8 form (set_inference_precision('fp8')) at the new widths, gated as the width-64 goldens are in
    tests/test_gpu_fp8.py: within 1.5x the error of its fp64 emulation plus the bf16 form's error"""
    from tests import test_gpu_fp8 as F8
    g = HG.HeadDimGolden(name)
    F8._check_model(name, g.build, g.x, g.out['y_eval'])
