"""Attention core kernels (generic / tensor-core flash / warp-per-problem) vs torch fp32 on the same bf16 qkv.  -m gpu"""
import pytest
import torch

pytestmark = pytest.mark.gpu

GENERIC, TC, WARP8 = 1, 2, 3


def K():
    from videotransformer_pytorch_b200 import _lib
    return _lib.K


def rel(a, b):
    a, b = a.detach().double(), b.detach().double()
    return float((a - b).norm() / (b.norm() + 1e-30))


def ref_attn(qkv, Bp, N, H, hd, scale):
    q = qkv.reshape(Bp, N, 3, H, hd).permute(2, 0, 3, 1, 4)
    s = (q[0] @ q[1].transpose(-1, -2)) * scale
    p = s.softmax(-1)
    o = (p @ q[2]).transpose(1, 2).reshape(Bp * N, H * hd)
    return o, p, torch.logsumexp(s, -1)


CASES = [(6, 8, 2, GENERIC), (3, 9, 12, GENERIC), (4, 33, 2, GENERIC), (5, 197, 3, GENERIC), (2, 256, 1, GENERIC),
         (6, 8, 2, WARP8), (1568, 8, 12, WARP8), (37, 8, 5, WARP8),
         (4, 33, 2, TC), (3, 64, 2, TC), (2, 128, 3, TC), (3, 130, 2, TC), (5, 197, 3, TC), (2, 256, 1, TC),
         (64, 197, 12, TC), (64, 197, 12, 0), (1568, 8, 12, 0)]


@pytest.mark.parametrize('Bp,N,H,impl', CASES)
def test_attn_fwd_bwd(Bp, N, H, impl):
    hd = 64
    torch.manual_seed(N * 7 + impl)
    qkv = (torch.randn(Bp, N, 3, H, hd) * 0.7).cuda().bfloat16()
    scale = hd ** -0.5
    want_probs = impl == GENERIC
    ctx, lse, probs = K().attn_fwd(qkv, Bp, N, H, hd, scale, want_probs=want_probs, impl=impl)
    torch.cuda.synchronize()
    qf = qkv.float().requires_grad_(True)
    o, p, l = ref_attn(qf, Bp, N, H, hd, scale)
    assert rel(ctx, o) < 5e-3, rel(ctx, o)
    if want_probs:
        assert rel(probs, p) < 1e-4
    assert rel(lse, l) < 1e-5, rel(lse, l)
    dctx = torch.randn(Bp * N, H * hd).cuda().bfloat16()
    o.backward(dctx.float())
    dqkv = K().attn_bwd(qkv, ctx, dctx, lse, Bp, N, H, hd, scale, impl=impl)
    torch.cuda.synchronize()
    assert dqkv.shape == qkv.shape
    for i, nm in enumerate('qkv'):
        e = rel(dqkv[:, :, i], qf.grad[:, :, i])
        assert e < 1.2e-2, (nm, e)


def test_attn_kernels_agree_on_adjacent_problems():
    """The tensor-core kernel stages whole 64-row tiles next to the rows of the next (frame) problem; results must
    not depend on what those rows hold."""
    Bp, N, H, hd = 3, 197, 2, 64
    torch.manual_seed(0)
    qkv = (torch.randn(Bp, N, 3, H, hd) * 0.7).cuda().bfloat16()
    c1, l1, _ = K().attn_fwd(qkv, Bp, N, H, hd, 0.125, impl=TC)
    q2 = qkv.clone()
    q2[1:] = (torch.randn(Bp - 1, N, 3, H, hd) * 50).cuda().bfloat16()   # wild neighbours
    c2, l2, _ = K().attn_fwd(q2, Bp, N, H, hd, 0.125, impl=TC)
    assert torch.equal(c1[:N], c2[:N]) and torch.equal(l1[0], l2[0])
    d = torch.randn(Bp * N, H * hd).cuda().bfloat16()
    g1 = K().attn_bwd(qkv, c1, d, l1, Bp, N, H, hd, 0.125, impl=TC)
    g2 = K().attn_bwd(q2, c2, d, l2, Bp, N, H, hd, 0.125, impl=TC)
    assert torch.equal(g1[0], g2[0])
