"""MaskFeat / MViT kernels and modules on the GPU.  -m gpu

Kernel level: each new kernel of csrc/vt_mvit.cu against the contract emulation (tests/emu_kernels.py, fp32 on CPU, fed the
same bf16-rounded operands).  Module level: MaskFeat forward / loss / gradients against the reference-generated goldens
(oracle/make_golden.py).  Tolerances at module level come from running the same pipeline with bf16 rounding emulated
on CPU: features 0.9-1.5e-2 rel-L2 after 16 blocks, gradients median 1.4-2.2e-2, worst single tensor 0.13.
"""
import pytest
import torch

from tests.conftest import rel_err
from tests.emu_kernels import EmuKernels

pytestmark = pytest.mark.gpu
HD = 96


def K():
    from videotransformer_pytorch_b200 import _lib
    return _lib.K


def emu():
    return EmuKernels(exact=True, dtype=torch.float32)


def rn(shape, seed, scale=1.0, dtype=torch.float32):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(shape, generator=g) * scale).to(dtype)


# ---- LayerNorm, narrow rows ---------------------------------------------------------------------------
@pytest.mark.parametrize('D', [96, 192, 32, 256, 64, 160, 224])
@pytest.mark.parametrize('rows', [1, 77, 4099])
def test_layernorm_small(D, rows):
    x, g, b = rn((rows, D), 1), 1 + rn((D,), 2, 0.1), rn((D,), 3, 0.1)
    y, mean, rstd = K().ln_fwd(x.cuda(), g.cuda(), b.cuda(), 1e-6)
    ref = torch.nn.functional.layer_norm(x, (D,), g, b, 1e-6)
    assert y.dtype == torch.bfloat16 and rel_err(y.float().cpu(), ref) < 4e-3
    y32, _, _ = K().ln_fwd(x.cuda(), g.cuda(), b.cuda(), 1e-6, out_fp32=True)
    assert rel_err(y32.cpu(), ref) < 1e-5
    assert rel_err(mean.cpu(), x.mean(-1)) < 1e-5
    for dy_dtype in (torch.float32, torch.bfloat16):
        dy = rn((rows, D), 4).to(dy_dtype)
        dres = rn((rows, D), 5)
        xr = x.clone().requires_grad_(True)
        gr, br = g.clone().requires_grad_(True), b.clone().requires_grad_(True)
        torch.nn.functional.layer_norm(xr, (D,), gr, br, 1e-6).backward(dy.float())
        dx, _, dg, db = K().ln_bwd(dy.cuda(), x.cuda(), mean, rstd, g.cuda(), dres=dres.cuda())
        assert rel_err(dx.cpu(), xr.grad + dres) < 1e-4
        assert rel_err(dg.cpu(), gr.grad) < 1e-4 and rel_err(db.cpu(), br.grad) < 1e-4


# ---- q/k/v pooling --------------------------------------------------------------------------------------
@pytest.mark.parametrize('thw,stride,H,B', [((2, 4, 4), (1, 2, 2), 2, 2), ((3, 5, 6), (1, 4, 4), 1, 1),
                                            ((2, 3, 3), (1, 1, 1), 2, 1), ((4, 16, 16), (1, 8, 8), 1, 3),
                                            ((8, 14, 14), (1, 2, 2), 4, 2), ((8, 7, 7), (1, 1, 1), 8, 2),
                                            ((2, 9, 11), (2, 2, 2), 2, 1), ((3, 28, 28), (1, 4, 4), 2, 2)])
def test_pool_fwd_bwd(thw, stride, H, B):
    N1 = 1 + thw[0] * thw[1] * thw[2]
    d = H * HD
    qkv = rn((B * N1, 3 * d), 10).bfloat16()
    w, gamma, beta = rn((HD, 27), 11, 0.3), 1 + rn((HD,), 12, 0.1), rn((HD,), 13, 0.1)
    e = emu()
    for slot in (0, 2):
        src_c = qkv.float().view(B, N1, 3 * d)[:, :, slot * d:(slot + 1) * d]
        out_r, pooled_r, mean_r, rstd_r, othw = e.pool_fwd(src_c, H, HD, thw, stride, w, gamma, beta, 1e-5)
        qg = qkv.cuda()
        src_g = qg.view(B, N1, 3 * d)[:, :, slot * d:(slot + 1) * d]
        out, pooled, mean, rstd, othw_g = K().pool_fwd(src_g, H, HD, thw, stride, w.cuda(), gamma.cuda(), beta.cuda(), 1e-5)
        assert tuple(othw_g) == tuple(othw)
        assert rel_err(pooled.cpu(), pooled_r) < 1e-5
        assert rel_err(out.float().cpu(), out_r) < 4e-3
        assert rel_err(rstd.cpu(), rstd_r) < 1e-4
        for dt in (torch.float32, torch.bfloat16):
            dout = rn(tuple(pooled_r.shape), 14).to(dt)
            dq_c = torch.zeros(B * N1, 3 * d)
            din_c = dq_c.view(B, N1, 3 * d)[:, :, slot * d:(slot + 1) * d]
            dw_r, dg_r, db_r = e.pool_bwd(dout.float(), pooled_r, mean_r, rstd_r, gamma, src_c, w, din_c, H, HD, thw, stride)
            dq_g = torch.full((B * N1, 3 * d), 7.0, dtype=torch.bfloat16, device='cuda')
            din_g = dq_g.view(B, N1, 3 * d)[:, :, slot * d:(slot + 1) * d]
            dw, dg, db = K().pool_bwd(dout.cuda(), pooled, mean, rstd, gamma.cuda(), src_g, w.cuda(), din_g, H, HD, thw, stride)
            assert rel_err(din_g.float().cpu(), din_c) < 5e-3
            other = [s for s in range(3) if s != slot]
            for s in other:                                   # neighbouring slots untouched
                assert bool((dq_g.view(B, N1, 3, d)[:, :, s] == 7.0).all())
            assert rel_err(dw.cpu(), dw_r) < 1e-4
            assert rel_err(dg.cpu(), dg_r) < 1e-4 and rel_err(db.cpu(), db_r) < 1e-4


# ---- pooling attention -----------------------------------------------------------------------------------
XATTN_SHAPES = [(2, 2, 70, 37), (1, 1, 300, 393), (1, 4, 64, 16), (2, 1, 5, 1), (1, 2, 129, 50), (1, 1, 1100, 393),
                (1, 2, 300, 700), (1, 1, 2300, 200), (3, 2, 128, 128)]


@pytest.mark.parametrize('impl', [1, 2], ids=['simt', 'mma'])
@pytest.mark.parametrize('B,H,Nq,Nk', XATTN_SHAPES)
def test_xattn_fwd_bwd(B, H, Nq, Nk, impl):
    d = H * HD
    scale = HD ** -0.5
    e = emu()
    tol_o, tol_g = (5e-3, 1e-2) if impl == 1 else (1e-2, 2e-2)       # the tensor-core path rounds P / dS to bf16
    # q read in place from a fused projection buffer, k/v contiguous pooled tensors
    qkv = rn((B * Nq, 3 * d), 20).bfloat16()
    k4, v4 = rn((B, H, Nk, HD), 21).bfloat16(), rn((B, H, Nk, HD), 22).bfloat16()
    q4_c = qkv.float().view(B, Nq, 3, H, HD)[:, :, 0].permute(0, 2, 1, 3)
    o_r, lse_r = e.xattn_fwd(q4_c, k4.float(), v4.float(), scale)
    qg = qkv.cuda()
    q4_g = qg.view(B, Nq, 3, H, HD)[:, :, 0].permute(0, 2, 1, 3)
    kg, vg = k4.cuda(), v4.cuda()
    o, lse = K().xattn_fwd(q4_g, kg, vg, scale, impl=impl)
    assert o.shape == (B, Nq, d)
    assert rel_err(o.float().cpu(), o_r) < tol_o
    assert rel_err(lse.cpu(), lse_r) < 1e-4
    dout = rn((B, Nq, d), 23).bfloat16()
    dq_c = torch.zeros(B, H, Nq, HD)
    dk_r, dv_r = e.xattn_bwd(q4_c, k4.float(), v4.float(), o.float().cpu(), dout.float(), lse.cpu(), scale, dq_c)
    dqkv = torch.full((B * Nq, 3 * d), 3.0, dtype=torch.bfloat16, device='cuda')
    dq_g = dqkv.view(B, Nq, 3, H, HD)[:, :, 0].permute(0, 2, 1, 3)
    dk, dv = K().xattn_bwd(q4_g, kg, vg, o, dout.cuda(), lse, scale, dq_g, impl=impl)
    assert bool((dqkv.view(B, Nq, 3, d)[:, :, 1:] == 3.0).all())          # k / v slots of the gradient buffer untouched
    assert rel_err(dv.cpu(), dv_r) < tol_g
    if Nk > 1:                              # with a single key dq and dk are zero up to rounding of o
        assert rel_err(dq_g.float().cpu(), dq_c) < tol_g
        assert rel_err(dk.cpu(), dk_r) < tol_g
    else:
        assert bool(torch.isfinite(dq_g.float()).all()) and bool(torch.isfinite(dk).all())
        assert float(dq_g.float().abs().max()) < 0.1
    # pooled (contiguous, head-major) q and dq as well
    qp = rn((B, H, Nq, HD), 24).bfloat16()
    o2_r, lse2_r = e.xattn_fwd(qp.float(), k4.float(), v4.float(), scale)
    o2, lse2 = K().xattn_fwd(qp.cuda(), kg, vg, scale, impl=impl)
    assert rel_err(o2.float().cpu(), o2_r) < tol_o
    dq2_c = torch.zeros(B, H, Nq, HD)
    dk2_r, dv2_r = e.xattn_bwd(qp.float(), k4.float(), v4.float(), o2.float().cpu(), dout.float(), lse2.cpu(), scale, dq2_c)
    dq2 = torch.empty((B, H, Nq, HD), dtype=torch.bfloat16, device='cuda')
    dk2, dv2 = K().xattn_bwd(qp.cuda(), kg, vg, o2, dout.cuda(), lse2, scale, dq2, impl=impl)
    assert rel_err(dv2.cpu(), dv2_r) < tol_g
    if Nk > 1:
        assert rel_err(dq2.float().cpu(), dq2_c) < tol_g and rel_err(dk2.cpu(), dk2_r) < tol_g


@pytest.mark.parametrize('B,H,N', [(1, 2, 300), (2, 12, 289), (1, 2, 1569), (3, 1, 128)])
def test_xattn_head_dim_64_self_attention(B, H, N):
    """The same kernels at head dim 64 with q, k, v all read in place from one packed [B*N, 3*H*64] projection
    (TimeSformer joint space-time attention)."""
    hd = 64
    d = H * hd
    scale = hd ** -0.5
    e = emu()
    qkv = rn((B * N, 3 * d), 80).bfloat16()
    views = lambda t: tuple(t.view(B, N, 3, H, hd)[:, :, s].permute(0, 2, 1, 3) for s in range(3))
    qc, kc, vc = views(qkv.float())
    o_r, lse_r = e.xattn_fwd(qc, kc, vc, scale)
    qg = qkv.cuda()
    q4, k4, v4 = views(qg)
    o, lse = K().xattn_fwd(q4, k4, v4, scale)
    assert rel_err(o.float().cpu(), o_r) < 1e-2 and rel_err(lse.cpu(), lse_r) < 1e-4
    dout = rn((B, N, d), 81).bfloat16()
    dq_c = torch.zeros(B, H, N, hd)
    dk_r, dv_r = e.xattn_bwd(qc, kc, vc, o.float().cpu(), dout.float(), lse.cpu(), scale, dq_c)
    dqkv = torch.full((B * N, 3 * d), 3.0, dtype=torch.bfloat16, device='cuda')
    dq4, _, _ = views(dqkv)
    dk, dv = K().xattn_bwd(q4, k4, v4, o, dout.cuda(), lse, scale, dq4)
    assert rel_err(dq4.float().cpu(), dq_c) < 2e-2
    assert rel_err(dk.cpu(), dk_r) < 2e-2 and rel_err(dv.cpu(), dv_r) < 2e-2
    assert bool((dqkv.view(B, N, 3, d)[:, :, 1:] == 3.0).all())


def test_xattn_head_dim_64_cuda_core_kernels():
    """Head dim 64 on the CUDA-core kernels (impl=1), q/k/v read in place from one packed projection, against the emulation."""
    B, H, N, hd = 1, 2, 300, 64
    d = H * hd
    scale = hd ** -0.5
    e = emu()
    qkv = rn((B * N, 3 * d), 82).bfloat16()
    views = lambda t: tuple(t.view(B, N, 3, H, hd)[:, :, s].permute(0, 2, 1, 3) for s in range(3))
    qc, kc, vc = views(qkv.float())
    o_r, lse_r = e.xattn_fwd(qc, kc, vc, scale)
    q4, k4, v4 = views(qkv.cuda())
    o, lse = K().xattn_fwd(q4, k4, v4, scale, impl=1)
    assert rel_err(o.float().cpu(), o_r) < 5e-3 and rel_err(lse.cpu(), lse_r) < 1e-4
    dout = rn((B, N, d), 83).bfloat16()
    dq_c = torch.zeros(B, H, N, hd)
    dk_r, dv_r = e.xattn_bwd(qc, kc, vc, o.float().cpu(), dout.float(), lse.cpu(), scale, dq_c)
    dqkv = torch.full((B * N, 3 * d), 3.0, dtype=torch.bfloat16, device='cuda')
    dq4, _, _ = views(dqkv)
    dk, dv = K().xattn_bwd(q4, k4, v4, o, dout.cuda(), lse, scale, dq4, impl=1)
    assert rel_err(dq4.float().cpu(), dq_c) < 1e-2
    assert rel_err(dk.cpu(), dk_r) < 1e-2 and rel_err(dv.cpu(), dv_r) < 1e-2
    assert bool((dqkv.view(B, N, 3, d)[:, :, 1:] == 3.0).all())


def test_xattn_auto_picks_tensor_cores_and_rejects_bad_layouts():
    B, H, Nq, Nk = 1, 2, 64, 32
    q = rn((B, H, Nq, HD), 25).bfloat16().cuda()
    k, v = rn((B, H, Nk, HD), 26).bfloat16().cuda(), rn((B, H, Nk, HD), 27).bfloat16().cuda()
    o_auto, _ = K().xattn_fwd(q, k, v, 0.1)
    o_tc, _ = K().xattn_fwd(q, k, v, 0.1, impl=2)
    assert torch.equal(o_auto, o_tc)
    q_odd = torch.empty((B, H, Nq, HD + 8), dtype=torch.bfloat16, device='cuda')[..., :HD]     # row pitch 104: no TMA view
    q_odd.copy_(q)
    o_simt, _ = K().xattn_fwd(q_odd, k, v, 0.1)                   # auto falls back to the CUDA-core kernel
    assert rel_err(o_simt.float(), o_tc.float()) < 1e-2
    with pytest.raises(RuntimeError, match='unsupported q layout'):
        K().xattn_fwd(q_odd, k, v, 0.1, impl=2)


# ---- skip-path max pooling ------------------------------------------------------------------------------
@pytest.mark.parametrize('thw,stride,D,B', [((2, 4, 4), (1, 2, 2), 96, 2), ((3, 5, 7), (1, 2, 2), 192, 1),
                                            ((8, 28, 28), (1, 2, 2), 384, 1)])
def test_maxpool_fwd_bwd(thw, stride, D, B):
    kernel = tuple(s + 1 if s > 1 else s for s in stride)
    x = rn((B, 1 + thw[0] * thw[1] * thw[2], D), 30)
    e = emu()
    y_r, idx_r, othw = e.maxpool_fwd(x, thw, kernel, stride)
    y, idx, othw_g = K().maxpool_fwd(x.cuda(), thw, kernel, stride)
    assert tuple(othw) == tuple(othw_g)
    assert torch.equal(y.cpu(), y_r)
    dy = rn(tuple(y_r.shape), 31)
    dx_r = e.maxpool_bwd(dy, idx_r, thw, kernel, stride)
    dx = K().maxpool_bwd(dy.cuda(), idx, thw, kernel, stride)
    assert rel_err(dx.cpu(), dx_r) < 1e-6


# ---- conv3d patch embedding operand, token preparation, loss ---------------------------------------------
def test_im2col3d_and_conv_gemm():
    B, T, C, S = 2, 8, 3, 32
    kernel, stride, padding, kpad = (3, 7, 7), (2, 4, 4), (1, 3, 3), 448
    x = rn((B, T, C, S, S), 40)
    cols_r, othw = emu().im2col3d(x, kernel, stride, padding, kpad)
    cols, othw_g = K().im2col3d(x.cuda(), kernel, stride, padding, kpad)
    assert tuple(othw) == tuple(othw_g)
    assert torch.equal(cols.float().cpu(), cols_r.bfloat16().float())
    w, b = rn((96, C, 3, 7, 7), 41, 0.05), rn((96,), 42, 0.1)
    wp = torch.nn.functional.pad(w.reshape(96, -1), (0, kpad - 441)).bfloat16().cuda()
    t = K().gemm(cols, wp, cols.shape[0], 96, kpad, bias=b.cuda(), epi='f32')
    ref = torch.nn.functional.conv3d(x.bfloat16().float().transpose(1, 2), w.bfloat16().float(), b, stride=stride, padding=padding)
    ref = ref.flatten(2).transpose(1, 2).reshape(-1, 96)
    assert rel_err(t.cpu(), ref) < 1e-4


@pytest.mark.parametrize('with_mask', [True, False])
def test_tokens_fwd_bwd(with_mask):
    B, T, HW, C = 2, 3, 20, 96
    L = T * HW
    t = rn((B * L, C), 50)
    wm = (torch.rand(B, L, generator=torch.Generator().manual_seed(51)) < 0.4).float() if with_mask else None
    mt, ct, ps, pt, pc = rn((C,), 52), rn((C,), 53), rn((HW, C), 54), rn((T, C), 55), rn((C,), 56)
    e = emu()
    x_r = e.mvit_tokens_fwd(t, wm, mt, ct, ps, pt, pc, B, T, HW)
    g = lambda v: None if v is None else v.cuda()
    x = K().mvit_tokens_fwd(t.cuda(), g(wm), mt.cuda(), ct.cuda(), ps.cuda(), pt.cuda(), pc.cuda(), B, T, HW)
    assert rel_err(x.cpu(), x_r) < 1e-6
    dx = rn((B, 1 + L, C), 57)
    dt_r = e.mvit_tokens_bwd(dx, wm, B, T, HW)
    dt = K().mvit_tokens_bwd(dx.cuda(), g(wm), B, T, HW)
    assert rel_err(dt.float().cpu(), dt_r) < 4e-3


def test_mse_fwd_bwd():
    dims = (B, t, dt, h, w, dc) = (2, 4, 2, 3, 3, 108)
    L1 = 1 + t * h * w
    pred, target = rn((B * L1, dt * dc), 60), rn((B, t * dt, h, w, dc), 61)
    mask = (torch.rand(B, t * dt, h, w, generator=torch.Generator().manual_seed(62)) < 0.3).float()
    e = emu()
    num_r = e.mse_fwd(pred, target, mask, dims)
    num = K().mse_fwd(pred.cuda(), target.cuda(), mask.cuda(), dims)
    assert abs(num[0].item() - num_r[0].item()) < 1e-4 * abs(num_r[0].item())
    coef = torch.tensor([0.125])
    dp_r = e.mse_bwd(pred, target, mask, coef, dims)
    dp = K().mse_bwd(pred.cuda(), target.cuda(), mask.cuda(), coef.cuda(), dims)
    assert rel_err(dp.float().cpu(), dp_r) < 4e-3
    assert bool((dp.view(B, L1, dt * dc)[:, 0] == 0).all())


# ---- GEMM shapes of the narrow MViT stages (K = 96, N = 96 / 288: k-block and n-tile tails) ---------------
@pytest.mark.parametrize('M,N,Kd', [(1000, 288, 96), (1000, 96, 288), (1000, 384, 96), (520, 96, 448), (3000, 192, 192),
                                    (777, 216, 768)])
def test_gemm_narrow_shapes(M, N, Kd):
    a, b, bias = rn((M, Kd), 70).bfloat16(), rn((N, Kd), 71).bfloat16(), rn((N,), 72)
    out = K().gemm(a.cuda(), b.cuda(), M, N, Kd, bias=bias.cuda(), epi='f32')
    ref = a.float() @ b.float().t() + bias
    assert rel_err(out.cpu(), ref) < 1e-5
    # weight-gradient form: dW[N, Kd] = dY[M, N]^T X[M, Kd], both operands MN-major, split-K
    dy = rn((M, N), 73).bfloat16()
    dw = K().gemm(dy.cuda(), a.cuda(), N, Kd, M, a_mn=True, b_mn=True, epi='f32', split_ok=True)
    assert rel_err(dw.cpu(), dy.float().t() @ a.float()) < 1e-5
    # data-gradient form: dX[M, Kd] = dY[M, N] W[N, Kd], W read MN-major, fp32 out with an fp32 addend
    aux = rn((M, Kd), 74)
    dx = K().gemm(dy.cuda(), b.cuda(), M, Kd, N, b_mn=True, epi='f32', aux=aux.cuda())
    assert rel_err(dx.cpu(), dy.float() @ b.float() + aux) < 1e-5


# ---- module level ------------------------------------------------------------------------------------------
def build(g):
    from videotransformer_pytorch_b200 import MaskFeat
    kw = dict(g.kwargs)
    for k in ('pool_q_stride_size', 'embed_dim_mul', 'atten_head_mul'):
        if k in kw:
            kw[k] = [list(r) for r in kw[k]]
    m = MaskFeat(**kw)
    m.load_state_dict(g.state(torch.float32), strict=True)
    return m.cuda()


@pytest.mark.parametrize('name', ['maskfeat_s32', 'maskfeat_s64', 'maskfeat_s64_3stage'])
def test_maskfeat_forward_features(maskfeat_golden, name):
    g = maskfeat_golden(name)
    m = build(g).train()
    with torch.no_grad():
        f = m.forward_features(g.x.cuda(), g.mask.cuda())
        f0 = m.forward_features(g.x.cuda())
    assert f.shape == g.feats.shape and f.dtype == torch.float32
    assert rel_err(f.cpu(), g.feats) < 4e-2
    assert rel_err(f0[:, 0].cpu(), g.feats_nomask_cls) < 4e-2


@pytest.mark.parametrize('name', ['maskfeat_s32', 'maskfeat_s64'])
def test_maskfeat_loss_and_gradients(maskfeat_golden, name):
    g = maskfeat_golden(name)
    m = build(g).train()
    pred, loss = m(g.x.cuda(), g.target.cuda(), g.mask.cuda(), g.cube_marker)
    assert pred.shape == g.pred.shape
    assert rel_err(pred.cpu(), g.pred) < 4e-2
    assert abs(loss.item() - g.loss) < 5e-3 * abs(g.loss)
    loss.backward()
    errs = []
    for n, p in m.named_parameters():
        if n.endswith('attn.norm_k.bias'):
            continue                                   # exactly zero in theory (softmax shift invariance)
        assert p.grad is not None, n
        if n in g.grad:
            errs.append((rel_err(p.grad.cpu(), g.grad[n]), n))
        elif n in g.gradsum:
            ref = g.gradsum[n]
            errs.append((abs(p.grad.double().norm().item() - ref[1]) / ref[1], n))
    errs.sort()
    median, worst = errs[len(errs) // 2][0], errs[-1]
    assert median < 5e-2, (median, errs[-5:])
    assert worst[0] < 0.3, errs[-5:]


def test_maskfeat_rejects_cpu_tensors(maskfeat_golden):
    g = maskfeat_golden('maskfeat_s32')
    m = build(g)
    with pytest.raises(RuntimeError):
        m.forward_features(g.x)          # CPU clip: no fallback


def test_maskfeat_step_is_graph_capturable(maskfeat_golden):
    """The whole MaskFeat step (forward + loss + backward) replayed as one CUDA graph gives the eager result."""
    from videotransformer_pytorch_b200.graph import GraphedTrainStep
    g = maskfeat_golden('maskfeat_s32')
    m = build(g).train()
    x, target, mask = g.x.cuda(), g.target.cuda(), g.mask.cuda()
    cmask = m.center_frame_mask(mask, g.cube_marker)

    class Step(torch.nn.Module):
        def __init__(self, net):
            super().__init__()
            self.net = net

        def forward(self, x, target, mask, cmask):
            return self.net.forward_with_center_mask(x, target, mask, cmask)[1]

    step = GraphedTrainStep(Step(m), (x, target, mask, cmask))        # before any eager backward (see graph.py)
    loss_g = float(step(x, target, mask, cmask))
    grads_g = {n: p.grad.clone() for n, p in m.named_parameters()}
    assert step.kernels_per_replay > 500
    for p in m.parameters():
        p.grad = None
    _, loss_e = m(x, target, mask, g.cube_marker)
    loss_e.backward()
    assert abs(loss_g - float(loss_e)) < 1e-5 * abs(float(loss_e))
    for n, p in m.named_parameters():
        if n.endswith('attn.norm_k.bias'):
            continue
        assert rel_err(grads_g[n].cpu(), p.grad.cpu()) < 2e-3, n       # fp32 atomics in dK/dV: order-dependent rounding
