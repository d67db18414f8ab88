"""wgmma GEMM (vt_gemm) vs torch fp32 matmul on the same bf16-rounded operands.  -m gpu"""

import pytest
import torch

pytestmark = pytest.mark.gpu


def K():
    from videotransformer_pytorch_b200 import _lib
    return _lib.K


def mk(shape, seed, scale=1.0):
    g = torch.Generator(device='cpu').manual_seed(seed)
    return (torch.randn(shape, generator=g) * scale).cuda()


def ref_mm(a, b, a_mn, b_mn):
    A = a.float().t() if a_mn else a.float()
    B = b.float() if b_mn else b.float().t()
    return A @ B


def rel(a, b):
    return float((a.double() - b.double()).norm() / (b.double().norm() + 1e-30))


SHAPES = [(128, 128, 64), (128, 256, 64), (256, 256, 128), (384, 512, 192), (200, 136, 72), (1000, 768, 768),
          (12544, 2304, 768)]


@pytest.mark.parametrize('M,N,Kd', SHAPES)
@pytest.mark.parametrize('a_mn,b_mn', [(False, False), (False, True), (True, True), (True, False)])
def test_gemm_plain_f32(M, N, Kd, a_mn, b_mn):
    if (a_mn and M % 8) or (b_mn and N % 8) or Kd % 8:
        pytest.skip('leading dims must be multiples of 8')
    a = mk((Kd, M) if a_mn else (M, Kd), 1).bfloat16()
    b = mk((Kd, N) if b_mn else (N, Kd), 2).bfloat16()
    out = K().gemm(a, b, M, N, Kd, a_mn=a_mn, b_mn=b_mn, epi='f32')
    torch.cuda.synchronize()
    r = ref_mm(a, b, a_mn, b_mn)
    assert rel(out, r) < 1e-5, rel(out, r)


@pytest.mark.parametrize('bn', [128, 192, 256])
def test_gemm_bf16_bias_rowscale(bn):
    M, N, Kd = 640, 512, 256
    a, b = mk((M, Kd), 3).bfloat16(), mk((N, Kd), 4).bfloat16()
    bias, rs = mk((N,), 5), mk((M,), 6).abs()
    out = K().gemm(a, b, M, N, Kd, epi='bf16', bias=bias, row_scale=rs, force_bn=bn)
    r = (ref_mm(a, b, False, False) + bias) * rs[:, None]
    assert out.dtype == torch.bfloat16
    assert rel(out, r) < 4e-3


def test_gemm_f32_residual_rowmaps():
    M, N, Kd, R = 300, 256, 128, 400
    a, b = mk((M, Kd), 7).bfloat16(), mk((N, Kd), 8).bfloat16()
    bias, rs = mk((N,), 9), mk((M,), 10)
    aux = mk((R, N), 11)
    perm = torch.randperm(R, generator=torch.Generator().manual_seed(0))[:M]
    out_row = perm.to(torch.int32).cuda()
    out_row[5] = -1                      # skipped row
    aux_row = torch.randint(0, R, (M,), generator=torch.Generator().manual_seed(1)).to(torch.int32).cuda()
    aux_row[7] = -1                      # no addend
    out = torch.full((R, N), 123.0, device='cuda')
    K().gemm(a, b, M, N, Kd, epi='f32', bias=bias, row_scale=rs, aux=aux, aux_row=aux_row, out=out, out_row=out_row)
    r = (ref_mm(a, b, False, False) + bias) * rs[:, None]
    add = aux[aux_row.long().clamp(min=0)]
    add[7] = 0
    r = r + add
    exp = torch.full((R, N), 123.0, device='cuda')
    ok = out_row >= 0
    exp[out_row[ok].long()] = r[ok]
    assert rel(out, exp) < 1e-5


@pytest.mark.parametrize('bn,staged', [(0, '1'), (128, '0'), (192, '1'), (256, '1')],
                         ids=['auto', 'bn128-register', 'bn192', 'bn256'])
@pytest.mark.parametrize('splits', [2, 5, 16])
def test_gemm_splitk_wgrad(splits, bn, staged, monkeypatch):
    """split-K partial tiles summed from the fp32 workspace into the output: with the planner's tile, and at each forced
    width (the partials take the staged fp32 rows at BN = 128 only, so BN = 128 is also run on the register epilogue)."""
    monkeypatch.setenv('VT_GEMM_STAGED_EPI', staged)
    Mtok, Nout, Kin = 2048 + 64, 384, 256
    dy, x = mk((Mtok, Nout), 16).bfloat16(), mk((Mtok, Kin), 17).bfloat16()
    out = torch.full((Nout, Kin), 7.0, device='cuda')            # stale contents must not leak into the result
    K().gemm(dy, x, Nout, Kin, Mtok, a_mn=True, b_mn=True, epi='f32', split_ok=True, force_splits=splits, force_bn=bn,
             out=out)
    r = dy.float().t() @ x.float()
    assert rel(out, r) < 1e-5


def test_gemm_splitk_odd_tile_edges():
    """split-K on a shape whose tiles hang over both output edges."""
    Mtok, Nout, Kin = 1000, 200, 136
    dy, x = mk((Mtok, Nout), 26).bfloat16(), mk((Mtok, Kin), 27).bfloat16()
    out = K().gemm(dy, x, Nout, Kin, Mtok, a_mn=True, b_mn=True, epi='f32', split_ok=True, force_splits=4)
    assert rel(out, dy.float().t() @ x.float()) < 1e-5


def test_gemm_wgrad_heuristic_split_big():
    Mtok, Nout, Kin = 12552, 768, 3072
    dy, x = mk((Mtok, Nout), 18, 0.1).bfloat16(), mk((Mtok, Kin), 19, 0.1).bfloat16()
    out = K().gemm(dy, x, Nout, Kin, Mtok, a_mn=True, b_mn=True, epi='f32', split_ok=True)
    r = dy.float().t() @ x.float()
    assert rel(out, r) < 1e-5


def test_gemm_rejects_bad_args():
    a, b = mk((64, 64), 1).bfloat16(), mk((64, 64), 2).bfloat16()
    with pytest.raises(RuntimeError):
        K().gemm(a.float(), b, 64, 64, 64)
    with pytest.raises(RuntimeError):
        K().gemm(a, b, 64, 60, 64)        # N not a multiple of 8 / shape mismatch
    with pytest.raises(RuntimeError, match="'bf16', 'f32', 'gelu_h'"):
        K().gemm(a, b, 64, 64, 64, epi='gelu')
    with pytest.raises(RuntimeError, match='fp32 epilogue only'):
        K().gemm(a, b, 64, 64, 64, epi='bf16', aux=a)


def test_vt_gemm_refuses_retired_epilogues_and_bf16_addend():
    """The C entry point refuses epilogue values 2 and 3 (the retired GELU / dGELU forms) and an addend with an epilogue
    other than fp32, which no bf16 form reads: each call returns an error, launches nothing and leaves the output as it
    was.  The same parameters with the plain bf16 epilogue and no addend run."""
    import ctypes as C
    from videotransformer_pytorch_b200 import _lib
    lib = _lib.load_library()
    M, N, Kd = 256, 256, 128
    a, b = mk((M, Kd), 12, 0.3).bfloat16(), mk((N, Kd), 13, 0.3).bfloat16()
    out = torch.full((M, N), 3.0, device='cuda', dtype=torch.bfloat16)
    other = mk((M, N), 14).bfloat16()

    def params(epilogue, out2=None, aux=None):
        p = _lib.GemmParams()
        p.a, p.b, p.lda, p.ldb = a.data_ptr(), b.data_ptr(), a.stride(0), b.stride(0)
        p.M, p.N, p.K, p.epilogue = M, N, Kd, epilogue
        p.out, p.ldo = out.data_ptr(), out.stride(0)
        if out2 is not None:
            p.out2, p.ldo2 = out2.data_ptr(), out2.stride(0)
        if aux is not None:
            p.aux, p.ldaux = aux.data_ptr(), aux.stride(0)
        p.map_special_base = -1
        return p

    for what, p, msg in (('epilogue 2', params(2, out2=other.clone()), 'bad epilogue 2'),
                         ('epilogue 3', params(3, aux=other), 'bad epilogue 3'),
                         ('bf16 with aux', params(_lib.EPI['bf16'], aux=other), 'aux'),
                         ('gelu_h with aux', params(_lib.EPI['gelu_h'], aux=other), 'aux')):
        torch.cuda.synchronize()
        n0 = _lib.launch_count()
        rc = lib.vt_gemm(C.byref(p), _lib._stream())
        torch.cuda.synchronize()
        err = C.create_string_buffer(512)
        lib.vt_last_error(err, 512)
        assert rc != 0, what
        assert msg in err.value.decode(), (what, err.value)
        assert _lib.launch_count() == n0, what
        assert bool((out == 3.0).all()), what
    n0 = _lib.launch_count()
    assert lib.vt_gemm(C.byref(params(_lib.EPI['bf16'])), _lib._stream()) == 0
    torch.cuda.synchronize()
    assert _lib.launch_count() == n0 + 1
    assert rel(out, ref_mm(a, b, False, False)) < 4e-3


@pytest.mark.parametrize('M,N,Kd', [(12552, 768, 3072), (12608, 2304, 768), (1000, 576, 192)])
def test_gemm_bn192_and_auto_config(M, N, Kd):
    a, b = mk((M, Kd), 21, 0.2).bfloat16(), mk((N, Kd), 22, 0.2).bfloat16()
    r = ref_mm(a, b, False, False)
    for bn in (0, 192):
        out = K().gemm(a, b, M, N, Kd, epi='f32', force_bn=bn)
        assert rel(out, r) < 1e-5, bn


@pytest.mark.parametrize('shape', [(1000, 3072), (12552, 3072), (2344, 3072), (5, 8), (1, 8)])
def test_gelu_kernels(shape):
    """sizes below, between and above one / two grid strides (the kernels take two vectors per thread per iteration)"""
    torch.manual_seed(3)
    z = (torch.randn(*shape) * 1.5).cuda().bfloat16()
    h = K().gelu(z)
    zf = z.float().requires_grad_(True)
    ref = torch.nn.functional.gelu(zf)
    assert rel(h, ref) < 3e-3
    dh = torch.randn(*shape).cuda().bfloat16()
    ref.backward(dh.float())
    assert rel(K().dgelu(dh, z), zf.grad) < 3e-3


@pytest.mark.parametrize('bn', [0, 128, 192, 256])
@pytest.mark.parametrize('M,N,Kd,a_mn,b_mn', [(128, 256, 128, False, False), (100, 128, 64, False, False),
                                              (1000, 768, 768, False, False), (12544, 768, 768, False, True),
                                              (12552, 3072, 768, False, False), (12608, 768, 768, False, True),
                                              (2304, 768, 12544, True, True), (640, 576, 320, True, True),
                                              (640, 384, 320, True, False)])
def test_gemm_forced_tile_widths(M, N, Kd, a_mn, b_mn, bn):
    """every operand layout at the planner's tile width (bn = 0) and at each forced one"""
    a = mk((Kd, M) if a_mn else (M, Kd), 31, 0.3).bfloat16()
    b = mk((Kd, N) if b_mn else (N, Kd), 32, 0.3).bfloat16()
    out = K().gemm(a, b, M, N, Kd, a_mn=a_mn, b_mn=b_mn, epi='f32', force_bn=bn, split_ok=a_mn and b_mn)
    torch.cuda.synchronize()
    assert rel(out, ref_mm(a, b, a_mn, b_mn)) < 1e-5


@pytest.mark.parametrize('epi', ['bf16', 'f32res'])
def test_gemm_epilogues_partial_last_tile(epi):
    """every epilogue with M = 1000: the last row of tiles holds 104 valid rows"""
    M, N, Kd = 1000, 512, 256
    a, b = mk((M, Kd), 41, 0.3).bfloat16(), mk((N, Kd), 42, 0.3).bfloat16()
    bias = mk((N,), 43)
    r = ref_mm(a, b, False, False)
    if epi == 'bf16':
        out = K().gemm(a, b, M, N, Kd, epi='bf16', bias=bias)
        assert rel(out, r + bias) < 4e-3
    elif epi == 'f32res':
        aux = mk((M, N), 44)
        perm = torch.randperm(M).to(torch.int32).cuda()
        out = torch.zeros(M, N, device='cuda')
        K().gemm(a, b, M, N, Kd, epi='f32', bias=bias, aux=aux, aux_row=perm, out_row=perm, out=out)
        exp = torch.zeros(M, N, device='cuda')
        exp[perm.long()] = r + bias + aux[perm.long()]
        assert rel(out, exp) < 1e-5


# ---- fp32 residual epilogue with plain rows and affine row maps, short last row tiles ---------------------------------
def _ops():
    from videotransformer_pytorch_b200 import ops
    return ops


@pytest.mark.parametrize('bn', [0, 128, 192, 256])
@pytest.mark.parametrize('M,N,Kd', [(1000, 768, 256), (12552, 768, 768), (130, 96, 192), (4096, 256, 64),
                                    (12544, 768, 3072), (1568, 384, 128), (200, 136, 72)])
def test_residual_epilogue_plain_rows_deterministic(M, N, Kd, bn):
    """y = s(m) (A B^T + bias) + aux without row maps (FC2, joint proj) against torch, with full and partial row and column
    tiles; a second call into a fresh output gives the same bits."""
    a, b = mk((M, Kd), 30).bfloat16(), mk((N, Kd), 31).bfloat16()
    bias, rs, aux = mk((N,), 32), mk((M,), 33), mk((M, N), 34)
    out = torch.full((M, N), 55.0, device='cuda')
    K().gemm(a, b, M, N, Kd, epi='f32', bias=bias, row_scale=rs, aux=aux, out=out, force_bn=bn)
    r = (ref_mm(a, b, False, False) + bias) * rs[:, None] + aux
    assert rel(out, r) < 1e-5
    again = torch.empty_like(out)
    K().gemm(a, b, M, N, Kd, epi='f32', bias=bias, row_scale=rs, aux=aux, out=again, force_bn=bn)
    assert torch.equal(out, again)


@pytest.mark.parametrize('staged', ['0', '1'], ids=['register', 'staged'])
@pytest.mark.parametrize('B,T,P,D', [(2, 8, 196, 768), (3, 4, 9, 128), (1, 2, 50, 256), (2, 8, 196, 96)])
def test_residual_epilogue_affine_maps_match_index_arrays(B, T, P, D, staged, monkeypatch):
    """The divided space-time scatters given as affine row maps (temporal '(b p) t', spatial '(b t) (1+p)' with the
    per-frame cls replicas going to side rows) against the same GEMM driven by the out_row / aux_row arrays alone, on the
    register and on the staged fp32 epilogue."""
    monkeypatch.setenv('VT_GEMM_STAGED_EPI', staged)
    ops = _ops()
    maps = ops.token_maps(B, T, P, 'cuda:0')
    aff = ops.affine_row_maps(B, T, P, D)
    S = 1 + P * T
    R = B * S
    Kd = 128
    x2 = mk((R, D), 40)
    w, bias = mk((D, Kd), 41).bfloat16(), mk((D,), 42)
    for name, Mrows, out_rows, out_row, aux_row in (('temporal', B * P * T, R, maps['temporal'], maps['temporal']),
                                                    ('spatial', B * T * (P + 1), R + B * T, maps['sp_out'], maps['sp_aux'])):
        a = mk((Mrows, Kd), 43).bfloat16()
        rs = mk((Mrows,), 44)
        got = torch.full((out_rows, D), -7.0, device='cuda')
        K().gemm(a, w, Mrows, D, Kd, epi='f32', bias=bias, row_scale=rs, aux=x2, aux_row=aux_row, out=got, out_row=out_row,
                 row_map=aff[name])
        exp = torch.full((out_rows, D), -7.0, device='cuda')
        K().gemm(a, w, Mrows, D, Kd, epi='f32', bias=bias, row_scale=rs, aux=x2, aux_row=aux_row, out=exp, out_row=out_row)
        assert rel(got, exp) < 1e-6, name
        # rows the map never names (the cls row of every sample) keep their old contents
        assert bool((got[torch.arange(B, device='cuda') * S] == -7.0).all()), name
        r = (a.float() @ w.float().t() + bias) * rs[:, None]
        add = x2[aux_row.long().clamp(min=0)] * (aux_row >= 0)[:, None]
        full = torch.full((out_rows, D), -7.0, device='cuda')
        full[out_row.long()] = r + add
        assert rel(got, full) < 1e-5, name


@pytest.mark.parametrize('M,N,Kd', [(12552, 768, 768), (12608, 2304, 256), (12552, 3072, 128), (136, 512, 192), (264, 256, 64)])
@pytest.mark.parametrize('form', ['fwd_bf16', 'dgrad_bf16', 'fwd_f32_residual'])
@pytest.mark.parametrize('bn', [0, 128, 192, 256])
def test_short_last_row_tile_deterministic(bn, M, N, Kd, form):
    """A last row of tiles with <= 64 valid rows (M = 12552 / 12608 of the FFN / spatial pass), at the planner's tile width
    (bn = 0) and at each forced one: against fp32 torch, and a second call gives the same bits."""
    a = mk((M, Kd), 50).bfloat16()
    bias, rs = mk((N,), 51), mk((M,), 52)
    if form == 'dgrad_bf16':
        b = mk((Kd, N), 53).bfloat16()                       # W [n_out = Kd, k_in = N] read MN-major
        kw = dict(b_mn=True, epi='bf16', row_scale=rs)
        r = (a.float() @ b.float()) * rs[:, None]
    elif form == 'fwd_bf16':
        b = mk((N, Kd), 53).bfloat16()
        kw = dict(epi='bf16', bias=bias)
        r = a.float() @ b.float().t() + bias
    else:
        b = mk((N, Kd), 53).bfloat16()
        aux = mk((M, N), 54)
        kw = dict(epi='f32', bias=bias, row_scale=rs, aux=aux)
        r = (a.float() @ b.float().t() + bias) * rs[:, None] + aux
    got = K().gemm(a, b, M, N, Kd, force_bn=bn, **kw)
    again = K().gemm(a, b, M, N, Kd, force_bn=bn, **kw)
    tol = 1e-5 if form == 'fwd_f32_residual' else 4e-3
    assert rel(got, r) < tol
    assert torch.equal(got, again)


@pytest.mark.parametrize('staged', ['0', '1'], ids=['register', 'staged'])
@pytest.mark.parametrize('M,N,Kd', [(12544, 768, 768), (1000, 256, 64), (12552, 768, 3072)])
def test_second_bias_after_row_scale(M, N, Kd, staged, monkeypatch):
    """out = s(m) (A B^T + bias) + bias2 + aux: the bias of a second linear layer folded into the GEMM (merged proj +
    temporal_fc), on the register and on the staged fp32 epilogue."""
    monkeypatch.setenv('VT_GEMM_STAGED_EPI', staged)
    a, b = mk((M, Kd), 70).bfloat16(), mk((N, Kd), 71).bfloat16()
    bias, bias2, rs, aux = mk((N,), 72), mk((N,), 73), mk((M,), 74), mk((M, N), 75)
    out = K().gemm(a, b, M, N, Kd, epi='f32', bias=bias, bias2=bias2, row_scale=rs, aux=aux)
    r = (ref_mm(a, b, False, False) + bias) * rs[:, None] + bias2 + aux
    assert rel(out, r) < 1e-5


@pytest.mark.parametrize('init', [9.0, 0.0], ids=['stale', 'zeroed'])
@pytest.mark.parametrize('M,N,Kd', [(768, 768, 12544), (2304, 768, 12608), (96, 448, 20000)])
def test_split_k_into_a_prezeroed_output(M, N, Kd, init):
    """Weight-gradient form (both operands MN-major, split-K): the output is written in full, so a stale-filled and a
    zero-filled output both end up equal to the product."""
    a, b = mk((Kd, M), 80).bfloat16(), mk((Kd, N), 81).bfloat16()
    r = a.float().t() @ b.float()
    out = torch.full((M, N), init, device='cuda')
    K().gemm(a, b, M, N, Kd, a_mn=True, b_mn=True, epi='f32', split_ok=True, out=out)
    assert rel(out, r) < 1e-5
