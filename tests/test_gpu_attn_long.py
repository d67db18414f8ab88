"""Packed-qkv attention past 256 tokens (the joint space-time passes, spatial passes of frames of 256 patches or more) through
vt_attn_fwd / vt_attn_bwd, bit for bit against the same tensor-core kernels driven through vt_xattn_* on strided views of the
packed projection, with their fp32 dK / dV rounded into the packed gradient by torch.  -m gpu

Both routes run attn_mma_fwd / attn_mma_bwd at head dim 64 on the same strides, so every output must be the same bits: dK /
dV start from the same fp32 values, rounded to nearest-even once in the kernel (vt_attn_bwd) or by copy_ (the strided route).
"""
import pytest
import torch

pytestmark = pytest.mark.gpu

HD = 64
TC = 2


def K():
    from videotransformer_pytorch_b200 import _lib
    return _lib.K


def heads(packed, Bp, N, H):
    """q, k, v slots of a packed [Bp * N, 3 * H * 64] tensor as [Bp, H, N, 64] views (no copy)"""
    v5 = packed.view(Bp, N, 3, H, HD)
    return [v5[:, :, s].permute(0, 2, 1, 3) for s in range(3)]


def strided_route(qkv, dctx, Bp, N, H):
    q4, k4, v4 = heads(qkv, Bp, N, H)
    ctx, lse = K().xattn_fwd(q4, k4, v4, HD ** -0.5, impl=TC)
    dqkv = torch.empty_like(qkv)
    dq4, dk4, dv4 = heads(dqkv, Bp, N, H)
    dk, dv = K().xattn_bwd(q4, k4, v4, ctx, dctx.view(Bp, N, H * HD), lse, HD ** -0.5, dq4, impl=TC)
    dk4.copy_(dk)
    dv4.copy_(dv)
    return ctx.view(Bp * N, H * HD), lse, dqkv


@pytest.mark.parametrize('Bp,H,N', [(3, 2, 257), (2, 12, 289), (4, 3, 401), (1, 12, 1569), (2, 5, 1569)])
def test_attn_past_256_tokens_matches_the_strided_route(Bp, H, N):
    g = torch.Generator().manual_seed(N * 16 + H)
    qkv = (torch.randn(Bp * N, 3 * H * HD, generator=g) * 0.7).bfloat16().cuda()
    dctx = torch.randn(Bp * N, H * HD, generator=g).bfloat16().cuda()
    ctx, lse, _ = K().attn_fwd(qkv, Bp, N, H, HD, HD ** -0.5)
    dqkv = K().attn_bwd(qkv, ctx, dctx, lse, Bp, N, H, HD, HD ** -0.5)
    ctx_s, lse_s, dqkv_s = strided_route(qkv, dctx, Bp, N, H)
    assert torch.equal(ctx, ctx_s)
    assert torch.equal(lse, lse_s)
    for name, a, b in zip(('dq', 'dk', 'dv'), heads(dqkv, Bp, N, H), heads(dqkv_s, Bp, N, H)):
        assert torch.equal(a, b), (name, int((a != b).sum()))
    ctx0, none, _ = K().attn_fwd(qkv, Bp, N, H, HD, HD ** -0.5, want_lse=False)       # the forward-only form
    assert none is None and torch.equal(ctx0, ctx)
