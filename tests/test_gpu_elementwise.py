"""Warp-primitive kernels vs torch.  -m gpu"""
import os

import pytest
import torch

pytestmark = pytest.mark.gpu


def K():
    from videotransformer_pytorch_b200 import _lib
    return _lib.K


def rel(a, b):
    return float((a.double() - b.double()).norm() / (b.double().norm() + 1e-30))


@pytest.mark.parametrize('D', [128, 384, 768, 1024])
@pytest.mark.parametrize('rows', [1, 37, 4096])
def test_layernorm_fwd_bwd(D, rows):
    torch.manual_seed(0)
    R = rows + 11
    x = (torch.randn(R, D) * 2 + 0.5).cuda()
    g, b = (1 + 0.1 * torch.randn(D)).cuda(), (0.1 * torch.randn(D)).cuda()
    in_row = torch.randperm(R)[:rows].to(torch.int32).cuda()
    y, mean, rstd = K().ln_fwd(x, g, b, 1e-5, in_row=in_row, rows=rows, out_fp32=True)
    xs = x[in_row.long()].clone().requires_grad_(True)
    gr, br = g.clone().requires_grad_(True), b.clone().requires_grad_(True)
    yr = torch.nn.functional.layer_norm(xs, (D,), gr, br, 1e-5)
    assert rel(y, yr) < 1e-5
    yb, _, _ = K().ln_fwd(x, g, b, 1e-5, in_row=in_row, rows=rows)
    assert yb.dtype == torch.bfloat16 and rel(yb, yr) < 4e-3
    dy = torch.randn(rows, D).cuda()
    yr.backward(dy)
    dres = torch.randn(R, D).cuda()
    dx = torch.full((R, D), 7.0, device='cuda')
    _, _, dg, db = K().ln_bwd(dy, x, mean, rstd, g, in_row=in_row, out_row=in_row, dres=dres, dx=dx)
    exp = torch.full((R, D), 7.0, device='cuda')
    exp[in_row.long()] = xs.grad + dres[in_row.long()]
    assert rel(dx, exp) < 1e-5
    assert rel(dg, gr.grad) < 1e-4 and rel(db, br.grad) < 1e-4
    # bf16 dy + aux rows (negative out_row)
    out_row = in_row.clone()
    n_aux = min(3, rows)
    out_row[:n_aux] = -(torch.arange(n_aux, dtype=torch.int32, device='cuda')) - 1
    dx2, aux, _, _ = K().ln_bwd(dy.bfloat16(), x, mean, rstd, g, in_row=in_row, out_row=out_row, n_aux=n_aux,
                                dx=torch.zeros(R, D, device='cuda'))
    xs2 = x[in_row.long()].clone().requires_grad_(True)
    torch.nn.functional.layer_norm(xs2, (D,), g, b, 1e-5).backward(dy.bfloat16().float())
    assert rel(aux, xs2.grad[:n_aux]) < 1e-5
    assert rel(dx2[in_row[n_aux:].long()], xs2.grad[n_aux:]) < 1e-5 or rows == n_aux


def test_casts_and_colsum():
    torch.manual_seed(1)
    x = torch.randn(1000, 768).cuda()
    assert torch.equal(K().cast_bf16(x), x.bfloat16())
    y = torch.randn(12345).cuda()
    assert torch.equal(K().cast_bf16(y), y.bfloat16())
    in_row = torch.randint(-1, 1000, (700,)).to(torch.int32).cuda()
    rs = torch.rand(700).cuda()
    g = K().gather_cast(x, in_row=in_row, row_scale=rs, rows=700)
    exp = x[in_row.long().clamp(min=0)] * rs[:, None]
    exp[in_row < 0] = 0
    assert torch.equal(g, exp.bfloat16())
    xb = torch.randn(12552, 3072).cuda().bfloat16()
    assert rel(K().colsum(xb), xb.float().sum(0)) < 1e-5
    xb = torch.randn(77, 136).cuda().bfloat16()
    assert rel(K().colsum(xb), xb.float().sum(0)) < 1e-5


@pytest.mark.parametrize('M,N', [(12544, 768), (12608, 2304), (12552, 3072), (1, 8), (255, 264), (257, 1000), (3000, 96),
                                 (513, 100)])
def test_colsum_shapes_and_views(M, N):
    """bias-gradient column sums, contiguous and as a column slice of a wider buffer; twice in a row (the last-CTA counters
    clean up after themselves)."""
    g = torch.Generator().manual_seed(M + N)
    wide = torch.randn(M, N + 16, generator=g).cuda().bfloat16()
    for x in (wide[:, :N].contiguous(), wide[:, 8:8 + N]):
        ref = x.float().sum(0)
        for _ in range(2):
            assert rel(K().colsum(x), ref) < 1e-5


@pytest.mark.parametrize('tube', [1, 2])
def test_im2col_col2im(tube):
    torch.manual_seed(2)
    B, T, C, H, W = 2, 4, 3, 48, 32
    x = torch.randn(B, T, C, H, W).cuda()
    cols = K().im2col(x, tube, 16, 16)
    Tp, Hp, Wp = T // tube, H // 16, W // 16
    ref = x.reshape(B, Tp, tube, C, Hp, 16, Wp, 16).permute(0, 1, 4, 6, 3, 2, 5, 7).reshape(B * Tp * Hp * Wp, -1)
    assert torch.equal(cols, ref.bfloat16())
    back = K().col2im(ref.contiguous(), (B, T, C, H, W), tube, 16, 16)
    assert torch.equal(back, x)


def test_im2col_u8_normalised():
    from tests.emu_kernels import EmuKernels
    from videotransformer_pytorch_b200 import _lib
    g = torch.Generator().manual_seed(0)
    x = torch.randint(0, 256, (2, 4, 32, 48, 3), dtype=torch.uint8, generator=g)
    scale = torch.tensor([1 / (255 * 0.229), 1 / (255 * 0.224), 1 / (255 * 0.225)])
    shift = torch.tensor([-0.485 / 0.229, -0.456 / 0.224, -0.406 / 0.225])
    for tube in (1, 2):
        ref = EmuKernels(exact=True).im2col_u8(x, scale, shift, tube, 16, 16)
        got = _lib.K.im2col_u8(x.cuda(), scale.cuda(), shift.cuda(), tube, 16, 16)
        assert got.shape == ref.shape
        assert float((got.float().cpu() - ref).abs().max()) < 2e-2          # bf16 rounding of values in [-2.2, 2.7]
        assert float((got.float().cpu() - ref.bfloat16().float()).abs().max()) < 1.6e-2


@pytest.mark.parametrize('rows,D,mapped', [(12544, 768, True), (12608, 768, True), (12552, 768, False), (37, 1024, False),
                                           (1000, 64, True), (5, 8, False)])
def test_gather_cast_with_column_sums(rows, D, mapped):
    """gather_cast + colsum in one kernel: same bf16 rows as the two-kernel form, column sums of exactly those rows."""
    g = torch.Generator().manual_seed(3)
    src = torch.randn(rows + 50, D, generator=g).cuda()
    in_row = scale = None
    if mapped:
        in_row = torch.randint(-1, rows + 50, (rows,), generator=g, dtype=torch.int32).cuda()
        scale = torch.rand(rows, generator=g).cuda()
    ref = K().gather_cast(src, in_row=in_row, row_scale=scale, rows=rows)
    for _ in range(2):                                    # twice: the arrival counter must be left at zero
        out, cs = K().gather_cast_colsum(src, in_row=in_row, row_scale=scale, rows=rows)
        assert torch.equal(out, ref)
        exp = ref.double().sum(0)
        assert float((cs.double() - exp).abs().max()) <= 1e-4 * max(1.0, float(exp.abs().max()))


@pytest.mark.parametrize('M,N', [(12552, 3072), (100, 256), (3, 8192), (777, 1536)])
def test_gelu_backward_with_column_sums(M, N):
    g = torch.Generator().manual_seed(4)
    dh = torch.randn(M, N, generator=g).bfloat16().cuda()
    z = (torch.randn(M, N, generator=g) * 2).bfloat16().cuda()
    ref = K().dgelu(dh, z)
    for _ in range(2):
        out, cs = K().dgelu_colsum(dh, z)
        assert torch.equal(out, ref)
        exp = ref.double().sum(0)
        assert float((cs.double() - exp).abs().max()) <= 1e-4 * max(1.0, float(exp.abs().max()))


@pytest.mark.parametrize('S,n,stride', [(296, 768, 768), (33, 8, 8), (592, 3072, 3072), (1000, 4, 12), (5, 256, 256), (64, 192, 384)])
def test_reduce_rows_tall_and_flat(S, n, stride):
    """out[j] (+)= scale * sum_s in[s * stride + j]: the partial-row sums behind split-K, LayerNorm dgamma / dbeta and the
    producer column sums (tall kernel for S >= 32, flat otherwise)."""
    import ctypes as C
    from videotransformer_pytorch_b200 import _lib
    lib = _lib.load_library()
    g = torch.Generator().manual_seed(9)
    src = torch.randn(S, stride, generator=g).cuda()
    for accumulate in (0, 1):
        out = torch.full((n,), 3.0, device='cuda')
        r = _lib.ReduceParams()
        r.inp, r.out, r.stride, r.S, r.n, r.accumulate, r.scale = src.data_ptr(), out.data_ptr(), stride, S, n, accumulate, 0.5
        assert lib.vt_reduce_rows(C.byref(r), C.c_void_p(torch.cuda.current_stream().cuda_stream)) == 0
        exp = 0.5 * src[:, :n].double().sum(0) + (3.0 if accumulate else 0.0)
        assert float((out.double() - exp).abs().max()) < 1e-4


@pytest.mark.parametrize('B,T,D,S', [(8, 8, 768, 1569), (3, 4, 128, 37), (1, 2, 32, 9)])
def test_cls_rows(B, T, D, S):
    g = torch.Generator().manual_seed(11)
    x = torch.randn(B, S, D, generator=g).cuda()
    extra = torch.randn(B, T, D, generator=g).cuda()
    y = torch.full((B, S, D), 5.0, device='cuda')
    K().cls_rows(y[:, 0], x[:, 0])
    assert torch.equal(y[:, 0], x[:, 0]) and bool((y[:, 1:] == 5.0).all())
    K().cls_rows(y[:, 0], x[:, 0], extra=extra, scale=1.0 / T)
    assert float((y[:, 0] - (x[:, 0] + extra.mean(dim=1))).abs().max()) < 1e-5
    assert bool((y[:, 1:] == 5.0).all())
