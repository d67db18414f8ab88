"""The persistent GEMM walks several tiles per CTA, its shared-memory ring running on across tile boundaries.  -m gpu

set_reserved_sms(64) shrinks the grid to vt_sm_count() - 64 CTAs, so the shapes below give CTAs one to three tiles, some
with more k-blocks than the ring has stages.  Every epilogue is checked across those tile boundaries on edges that are not
multiples of the tile, and the result must not depend on the grid size."""

import pytest
import torch

pytestmark = pytest.mark.gpu

RESERVE = 64


def lib():
    from videotransformer_pytorch_b200 import _lib
    return _lib


def mk(shape, seed, scale=1.0):
    g = torch.Generator(device='cpu').manual_seed(seed)
    return (torch.randn(shape, generator=g) * scale).cuda()


def rel(a, b):
    return float((a.double() - b.double()).norm() / (b.double().norm() + 1e-30))


@pytest.fixture
def reserved():
    lib().set_reserved_sms(RESERVE)
    yield lib().K
    lib().set_reserved_sms(0)


def rows_for(n_tiles_per_cta):
    """M (not a multiple of 128) for which 128-row tiles x 2 n-tiles give about this many tiles per CTA"""
    grid = lib().load_library().vt_sm_count() - RESERVE
    return int(n_tiles_per_cta * grid / 2) * 128 - 40


@pytest.mark.parametrize('bn', [128, 192, 256])
@pytest.mark.parametrize('N', [136, 200])
@pytest.mark.parametrize('form', ['bf16', 'f32res'])
def test_epilogues_across_tiles(form, N, bn, reserved):
    K = reserved
    M, Kd = rows_for(2.5), 72
    a, b = mk((M, Kd), 1, 0.3).bfloat16(), mk((N, Kd), 2, 0.3).bfloat16()
    bias, rs = mk((N,), 3), mk((M,), 4)
    r = a.float() @ b.float().t()
    if form == 'bf16':
        out = K.gemm(a, b, M, N, Kd, epi='bf16', bias=bias, row_scale=rs, force_bn=bn)
        assert rel(out, (r + bias) * rs[:, None]) < 4e-3
    else:
        R = M + 50
        aux = mk((R, N), 5)
        out_row = torch.randperm(R, generator=torch.Generator().manual_seed(0))[:M].to(torch.int32).cuda()
        aux_row = torch.randint(0, R, (M,), generator=torch.Generator().manual_seed(1)).to(torch.int32).cuda()
        out_row[5::97] = -1                  # skipped rows
        aux_row[7::89] = -1                  # rows without an addend
        out = torch.full((R, N), 123.0, device='cuda')
        K.gemm(a, b, M, N, Kd, epi='f32', bias=bias, row_scale=rs, aux=aux, aux_row=aux_row, out=out, out_row=out_row,
               force_bn=bn)
        y = (r + bias) * rs[:, None] + aux[aux_row.long().clamp(min=0)] * (aux_row >= 0)[:, None]
        exp = torch.full((R, N), 123.0, device='cuda')
        ok = out_row >= 0
        exp[out_row[ok].long()] = y[ok]
        assert rel(out, exp) < 1e-5


@pytest.mark.parametrize('bn', [128, 192, 256])
@pytest.mark.parametrize('splits', [2, 3])
def test_splitk_across_tiles(splits, bn, reserved):
    K = reserved
    Mtok, Nout, Kin = 1000, rows_for(1.5 / splits), 200      # 16 k-blocks: 8 or 5 per split, about as many as the ring holds
    dy, x = mk((Mtok, Nout), 7).bfloat16(), mk((Mtok, Kin), 8).bfloat16()
    out = torch.full((Nout, Kin), 7.0, device='cuda')
    K.gemm(dy, x, Nout, Kin, Mtok, a_mn=True, b_mn=True, epi='f32', split_ok=True, force_splits=splits, force_bn=bn, out=out)
    assert rel(out, dy.float().t() @ x.float()) < 1e-5


@pytest.mark.parametrize('B,T,P,D', [(2, 8, 196, 200), (3, 4, 9, 136)])
def test_affine_maps_across_tiles(B, T, P, D, reserved):
    """the temporal and spatial residual scatters (cls replicas to side rows) through the affine map, against torch"""
    from videotransformer_pytorch_b200 import ops
    K = reserved
    maps = ops.token_maps(B, T, P, 'cuda:0')
    aff = ops.affine_row_maps(B, T, P, D)
    S = 1 + P * T
    R = B * S
    Kd = 72
    x2 = mk((R, D), 9)
    w, bias = mk((D, Kd), 10).bfloat16(), mk((D,), 11)
    for name, Mrows, out_rows, out_row, aux_row in (('temporal', B * P * T, R, maps['temporal'], maps['temporal']),
                                                    ('spatial', B * T * (P + 1), R + B * T, maps['sp_out'], maps['sp_aux'])):
        a = mk((Mrows, Kd), 12).bfloat16()
        rs = mk((Mrows,), 13)
        for bn in (128, 192):
            got = torch.full((out_rows, D), -7.0, device='cuda')
            K.gemm(a, w, Mrows, D, Kd, epi='f32', bias=bias, row_scale=rs, aux=x2, aux_row=aux_row, out=got, out_row=out_row,
                   row_map=aff[name], force_bn=bn)
            y = (a.float() @ w.float().t() + bias) * rs[:, None] + x2[aux_row.long().clamp(min=0)] * (aux_row >= 0)[:, None]
            exp = torch.full((out_rows, D), -7.0, device='cuda')
            exp[out_row.long()] = y
            assert rel(got, exp) < 1e-5, (name, bn)


def _bitwise_case(seed):
    M, N, Kd = rows_for(2.5), 200, 264
    a, b = mk((M, Kd), seed, 0.3).bfloat16(), mk((N, Kd), seed + 1, 0.3).bfloat16()
    bias, aux = mk((N,), seed + 2), mk((M, N), seed + 3)
    return M, N, Kd, a, b, bias, aux


@pytest.mark.parametrize('bn', [128, 192, 256])
def test_f32_gelu_h_split_k_bitwise_independent_of_grid_and_run(bn):
    """fixed tile width and split count: identical bits for the full grid, a 64-SM-smaller grid, and a second run"""
    K = lib().K
    M, N, Kd, a, b, bias, aux = _bitwise_case(20)
    dy, x = mk((2000, 384), 30).bfloat16(), mk((2000, 200), 31).bfloat16()

    def run():
        y = K.gemm(a, b, M, N, Kd, epi='f32', bias=bias, aux=aux, force_bn=bn)
        h = K.gemm(a, b, M, N, Kd, epi='gelu_h', bias=bias, force_bn=bn)
        g = K.gemm(dy, x, 384, 200, 2000, a_mn=True, b_mn=True, epi='f32', split_ok=True, force_splits=3, force_bn=bn)
        return [y, h, g]

    try:
        full = run()
        again = run()
        lib().set_reserved_sms(RESERVE)
        small = run()
    finally:
        lib().set_reserved_sms(0)
    for f, s, g in zip(full, again, small):
        assert torch.equal(f, g) and torch.equal(f, s)


def test_graph_replay_matches_eager():
    K = lib().K
    M, N, Kd, a, b, bias, aux = _bitwise_case(40)
    eager = K.gemm(a, b, M, N, Kd, epi='f32', bias=bias, aux=aux)
    out = torch.empty_like(eager)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):                        # warm-up outside the capture
        K.gemm(a, b, M, N, Kd, epi='f32', bias=bias, aux=aux, out=out)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        K.gemm(a, b, M, N, Kd, epi='f32', bias=bias, aux=aux, out=out)
    out.zero_()
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, eager)
