"""Attention kernels row by row against fp64 at the tile edges.  -m gpu

Every output is compared one row at a time (tests/attn_mma_emu.row_errors) with closed-form fp64 attention on the same bf16
inputs.  The budget is the error of the CPU model of the same kernel on the same inputs (attn_mma_emu: 'bf16' for the
tensor-core kernels, 'bf16_out' for the CUDA-core ones) times the factors fixed in attn_mma_emu, and the tensor-core kernels
must also stay close to their model directly.  The kernels are driven through ctypes with outputs of the test's own:
pre-filled with NaN and placed between NaN guard rows, with k / v / q read from buffers whose rows past the end hold NaN, so a
missing store, a store past Nq / Nk or a read of a row past the end shows.
"""
import ctypes as C

import pytest
import torch

from tests import attn_mma_emu as AE

pytestmark = pytest.mark.gpu

AUTO, SIMT, TC, WARP8 = 0, 1, 2, 3
G = 16                       # guard rows on either side of every output
PAD = 8                      # rows past the end of every input, NaN
NAN16, NAN32 = torch.tensor(float('nan'), dtype=torch.bfloat16).view(torch.int16), torch.tensor(float('nan')).view(torch.int32)


def _lib():
    from videotransformer_pytorch_b200 import _lib
    return _lib, _lib.load_library()


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _call(fn, p, what):
    _lib_, lib = _lib()
    _lib_._check(getattr(lib, fn)(C.byref(p), _stream()), what)


class Guarded:
    """`rows` x `width` output between G NaN guard rows on each side; the rows themselves start as NaN too"""

    def __init__(self, rows, width, dtype):
        self.buf = torch.full(((rows + 2 * G) * width,), float('nan'), dtype=dtype, device='cuda')
        self.rows, self.width = rows, width
        self.inner = self.buf[G * width:(G + rows) * width]

    def check(self, name, cols=None):
        """every element of the rows (of columns `cols` only, if given) written and finite; guards keep their NaN bits"""
        torch.cuda.synchronize()
        bits = NAN16 if self.buf.dtype == torch.bfloat16 else NAN32
        idt = torch.int16 if self.buf.dtype == torch.bfloat16 else torch.int32
        w = self.width
        guard = torch.cat([self.buf[:G * w], self.buf[-G * w:]]).view(idt)
        assert bool((guard == bits.to(guard.device)).all()), f'{name}: store outside the output'
        inner = self.inner.view(self.rows, w)
        part = inner if cols is None else inner[:, cols]
        bad = ~torch.isfinite(part.float())
        assert not bool(bad.any()), f'{name}: {int(bad.sum())} elements not written or not finite, first at {bad.nonzero()[0].tolist()}'
        if cols is not None:
            rest = torch.ones(w, dtype=torch.bool)
            rest[cols] = False
            assert bool((inner[:, rest.nonzero()[:, 0].cuda()].view(idt) == bits.to(inner.device)).all()), \
                f'{name}: store into a neighbouring slot'


def _bf16_cuda(x):
    return x.to(torch.bfloat16).cuda()


# ---- vt_xattn_* driver -----------------------------------------------------------------------------------------------
def run_xattn(q, k, v, do, scale, impl=TC, layout='head'):
    """q, do [B, H, Nq, hd], k, v [B, H, Nk, hd] (bf16-valued fp64, CPU) through vt_xattn_fwd / vt_xattn_bwd.
    layout: 'head'   q / k / v head-major [B, H, N, hd] with NaN rows past N, dq head-major;
            'packed' q / k / v token-major slots of one [B * N, 3, H, hd] projection (Nq == Nk), dq into slot 0 of a gradient
                     buffer of the same shape;
            'mvit'   q token-major slot 0 of a [B * Nq, 3, H, hd] projection (k / v slots NaN), k / v head-major, dq into
                     slot 0.
    -> dict of CPU fp64 o [B, H, Nq, hd], lse [B, H, Nq], delta, dq, dk, dv (fp32 [B, H, Nk, hd])"""
    lib_, _ = _lib()
    B, H, Nq, hd = q.shape
    Nk = k.shape[2]
    d = H * hd

    def head_major(x):
        n = x.shape[2]
        buf = torch.full((B, H, n + PAD, hd), float('nan'), dtype=torch.bfloat16, device='cuda')
        buf[:, :, :n] = _bf16_cuda(x)
        return buf, (buf.data_ptr(), H * (n + PAD) * hd, (n + PAD) * hd, hd)

    def token_major(xs, n):
        buf = torch.full((B * n + PAD, 3, H, hd), float('nan'), dtype=torch.bfloat16, device='cuda')
        for s, x in enumerate(xs):
            if x is not None:
                buf[:B * n, s] = _bf16_cuda(x.permute(0, 2, 1, 3).reshape(B * n, H, hd))
        return buf, [(buf.data_ptr() + s * d * 2, n * 3 * d, hd, 3 * d) for s in range(3)]

    keep = []
    if layout == 'head':
        (qb, qd), (kb, kd), (vb, vd) = head_major(q), head_major(k), head_major(v)
        keep += [qb, kb, vb]
    elif layout == 'packed':
        assert Nq == Nk
        buf, (qd, kd, vd) = token_major((q, k, v), Nq)
        keep.append(buf)
    else:
        buf, (qd, _, _) = token_major((q, None, None), Nq)
        (kb, kd), (vb, vd) = head_major(k), head_major(v)
        keep += [buf, kb, vb]
    o = Guarded(B * Nq, d, torch.bfloat16)
    lse = Guarded(B * H, Nq, torch.float32)
    p = lib_.XattnFwdParams()
    p.q, p.q_bs, p.q_hs, p.q_rs = qd
    p.k, p.k_bs, p.k_hs, p.k_rs = kd
    p.v, p.v_bs, p.v_hs, p.v_rs = vd
    p.o, p.o_bs, p.o_hs, p.o_rs = o.inner.data_ptr(), Nq * d, hd, d
    p.lse = lse.inner.data_ptr()
    p.B, p.H, p.Nq, p.Nk, p.hd, p.scale, p.impl = B, H, Nq, Nk, hd, scale, impl
    _call('vt_xattn_fwd', p, 'vt_xattn_fwd')
    o.check('o')
    lse.check('lse')
    dout = _bf16_cuda(do.permute(0, 2, 1, 3).reshape(B * Nq, d))
    delta = Guarded(B * H, Nq, torch.float32)
    dk, dv = Guarded(B * H * Nk, hd, torch.float32), Guarded(B * H * Nk, hd, torch.float32)
    if layout == 'head':
        dq = Guarded(B * H * Nq, hd, torch.bfloat16)
        dqd = (dq.inner.data_ptr(), H * Nq * hd, Nq * hd, hd)
    else:
        dq = Guarded(B * Nq, 3 * d, torch.bfloat16)
        dqd = (dq.inner.data_ptr(), Nq * 3 * d, hd, 3 * d)
    pb = lib_.XattnBwdParams()
    pb.q, pb.q_bs, pb.q_hs, pb.q_rs = qd
    pb.k, pb.k_bs, pb.k_hs, pb.k_rs = kd
    pb.v, pb.v_bs, pb.v_hs, pb.v_rs = vd
    pb.o, pb.dout = o.inner.data_ptr(), dout.data_ptr()
    pb.o_bs, pb.o_hs, pb.o_rs = Nq * d, hd, d
    pb.dq, pb.dq_bs, pb.dq_hs, pb.dq_rs = dqd
    pb.lse, pb.delta, pb.dk, pb.dv = lse.inner.data_ptr(), delta.inner.data_ptr(), dk.inner.data_ptr(), dv.inner.data_ptr()
    pb.B, pb.H, pb.Nq, pb.Nk, pb.hd, pb.scale, pb.impl = B, H, Nq, Nk, hd, scale, impl
    _call('vt_xattn_bwd', pb, 'vt_xattn_bwd')
    delta.check('delta')
    dk.check('dk')
    dv.check('dv')
    if layout == 'head':
        dq.check('dq')
        dq_t = dq.inner.view(B, H, Nq, hd)
    else:
        dq.check('dq', cols=torch.arange(d))                           # slot 0 written, k / v slots untouched
        dq_t = dq.inner.view(B, Nq, 3, H, hd)[:, :, 0].permute(0, 2, 1, 3)
    f = lambda t: t.double().cpu()
    return dict(o=f(o.inner.view(B, Nq, H, hd).permute(0, 2, 1, 3)), lse=f(lse.inner.view(B, H, Nq)),
                delta=f(delta.inner.view(B, H, Nq)), dq=f(dq_t), dk=f(dk.inner.view(B, H, Nk, hd)),
                dv=f(dv.inner.view(B, H, Nk, hd)))


# ---- vt_attn_* driver (packed qkv [Bp, N, 3, H, 64]) --------------------------------------------------------------------
def run_attn(q, k, v, do, scale, impl):
    """q, k, v, do [Bp, H, N, 64] (bf16-valued fp64, CPU) through vt_attn_fwd / vt_attn_bwd with a guarded qkv buffer and
    guarded outputs -> dict of CPU fp64 o, lse, dq, dk, dv ([Bp, H, N, hd] / [Bp, H, N])"""
    lib_, _ = _lib()
    Bp, H, N, hd = q.shape
    d = H * hd
    qkv = Guarded(Bp * N, 3 * d, torch.bfloat16)
    qkv.inner.view(Bp * N, 3, H, hd).copy_(torch.stack([x.permute(0, 2, 1, 3).reshape(Bp * N, H, hd) for x in (q, k, v)], 1)
                                          .to(torch.bfloat16).cuda())
    ctx, lse = Guarded(Bp * N, d, torch.bfloat16), Guarded(Bp * H, N, torch.float32)
    p = lib_.AttnFwdParams()
    p.qkv, p.ctx, p.lse, p.probs = qkv.inner.data_ptr(), ctx.inner.data_ptr(), lse.inner.data_ptr(), None
    p.Bp, p.N, p.H, p.hd, p.scale, p.impl = Bp, N, H, hd, scale, impl
    _call('vt_attn_fwd', p, 'vt_attn_fwd')
    ctx.check('ctx')
    lse.check('lse')
    dctx = _bf16_cuda(do.permute(0, 2, 1, 3).reshape(Bp * N, d))
    dqkv = Guarded(Bp * N, 3 * d, torch.bfloat16)
    pb = lib_.AttnBwdParams()
    pb.qkv, pb.ctx, pb.dctx, pb.lse, pb.dqkv = qkv.inner.data_ptr(), ctx.inner.data_ptr(), dctx.data_ptr(), lse.inner.data_ptr(), \
        dqkv.inner.data_ptr()
    pb.Bp, pb.N, pb.H, pb.hd, pb.scale, pb.impl = Bp, N, H, hd, scale, impl
    _call('vt_attn_bwd', pb, 'vt_attn_bwd')
    dqkv.check('dqkv')
    g = dqkv.inner.view(Bp, N, 3, H, hd).permute(2, 0, 3, 1, 4).double().cpu()
    return dict(o=ctx.inner.view(Bp, N, H, hd).permute(0, 2, 1, 3).double().cpu(), lse=lse.inner.view(Bp, H, N).double().cpu(),
                dq=g[0], dk=g[1], dv=g[2])


# ---- checks ------------------------------------------------------------------------------------------------------------
def flat(x):
    return x.reshape(-1, *x.shape[2:])


def check_against_fp64(tag, got, q, k, v, do, scale, mode, dkv_bf16, sample=None):
    """got: kernel outputs of the whole batch; the fp64 reference and the model run on the (b, h) problems in `sample` (flat
    indices; all if None).  mode: the model of the kernel ('bf16' tensor cores, 'bf16_out' CUDA cores)."""
    B, H = q.shape[:2]
    idx = torch.arange(B * H) if sample is None else torch.tensor(sample)
    sel = lambda x: flat(x)[idx]
    qs, ks, vs, dos = sel(q), sel(k), sel(v), sel(do)
    r_o, r_lse, r_dq, r_dk, r_dv = AE.reference(qs, ks, vs, dos, scale)
    m_o, m_lse = AE.fwd(qs, ks, vs, scale, mode)                       # the model's own chain: the budget
    m_dq, m_dk, m_dv = AE.bwd(qs, ks, vs, m_o, dos, m_lse, scale, mode, dkv_bf16=dkv_bf16)
    g = {n: sel(got[n]) for n in ('o', 'lse', 'dq', 'dk', 'dv')}
    if mode == 'bf16':                                                 # the model fed the kernel's own o / lse: direct gate
        d_o = m_o
        d_dq, d_dk, d_dv = AE.bwd(qs, ks, vs, g['o'], dos, g['lse'], scale, mode, dkv_bf16=dkv_bf16)
    e_lse, i = AE.lse_error(g['lse'], r_lse)
    Nq = q.shape[2]
    assert e_lse <= AE.LSE_TOL, f'{tag} lse: {e_lse:.3e} at problem {int(idx[i // Nq])} row {i % Nq}'
    one_key = k.shape[2] == 1
    report = []
    for n, ref, model in (('o', r_o, m_o), ('dq', r_dq, m_dq), ('dk', r_dk, m_dk), ('dv', r_dv, m_dv)):
        if one_key and n in ('dq', 'dk'):                              # exactly zero; o = v rounds to v, so only noise
            assert float(g[n].abs().max()) < 1e-3, (tag, n, float(g[n].abs().max()))
            continue
        ok, e, m = AE.within_budget(g[n], ref, model)
        budget = AE.C_ROW * m.worst + AE.ABS_FLOOR
        report.append(f'{n} {e.worst:.2e}/{budget:.2e}')
        where = (int(idx[e.where[0]]) // H, int(idx[e.where[0]]) % H, e.where[2])
        assert ok, (f'{tag} {n}: worst row {e.worst:.3e} at (b, h, row) {where} against {budget:.3e}; '
                    f'global {e.glob:.3e} against {AE.C_GLOB * m.glob + AE.ABS_FLOOR:.3e}')
        if mode == 'bf16':
            direct = {'o': d_o, 'dq': d_dq, 'dk': d_dk, 'dv': d_dv}[n]
            dist = float((g[n] - direct).norm() / ref.norm().clamp(min=1e-300)) if float(ref.norm()) > 0 else 0.0
            assert dist <= AE.D_GLOB * m.glob + AE.ABS_FLOOR, f'{tag} {n}: {dist:.3e} from the model of the kernel'
    print(f'[attn-edges] {tag}: ' + ', '.join(report))


def inputs(B, H, Nq, Nk, hd, scale, regime='benign', seed=0):
    q, k, v, do = AE.make_inputs(B * H, Nq, Nk, hd, scale, regime, seed)
    return tuple(t.view(B, H, *t.shape[1:]) for t in (q, k, v, do))


# ---- tensor-core strided attention (vt_xattn_*, impl 2) ---------------------------------------------------------------
EDGE = [(1, 1), (1, 393), (17, 393), (393, 17), (393, 1), (63, 65), (64, 64), (65, 64), (65, 129), (128, 129), (129, 63),
        (129, 128), (197, 197), (17, 63)]


@pytest.mark.parametrize('hd', [64, 96])
@pytest.mark.parametrize('Nq,Nk', EDGE)
def test_xattn_tensor_core_tile_edges(Nq, Nk, hd):
    layout = 'packed' if Nq == Nk else ('mvit' if (Nq + Nk) % 2 else 'head')
    scale = hd ** -0.5
    q, k, v, do = inputs(2, 2, Nq, Nk, hd, scale, seed=Nq * 7 + Nk)
    got = run_xattn(q, k, v, do, scale, TC, layout)
    check_against_fp64(f'xattn tc hd{hd} {Nq}x{Nk} {layout}', got, q, k, v, do, scale, 'bf16', False)


@pytest.mark.parametrize('hd', [64, 96])
@pytest.mark.parametrize('scale', ['hd', 1.0, 0.05])
@pytest.mark.parametrize('regime', AE.REGIMES)
def test_xattn_tensor_core_logit_regimes(regime, scale, hd):
    """Nq = 129, Nk = 197: partial last query and key tiles (1 and 5 rows); each regime at three scales, so a kernel that
    hard-codes 1/sqrt(hd) in the forward, dQ or dK / dV pass fails."""
    scale = hd ** -0.5 if scale == 'hd' else scale
    q, k, v, do = inputs(2, 2, 129, 197, hd, scale, regime, seed=hd)
    got = run_xattn(q, k, v, do, scale, TC, 'head')
    check_against_fp64(f'xattn tc hd{hd} {regime} scale {scale:.3f}', got, q, k, v, do, scale, 'bf16', False)


@pytest.mark.parametrize('B,H,Nq,Nk,hd,layout,sample', [
    (2, 12, 1569, 1569, 64, 'packed', [0, 13, 23]),            # TimeSformer joint space-time pass
    (2, 1, 25088, 393, 96, 'mvit', [0, 1]),                    # MViT-B stage 1 pooling attention
])
def test_xattn_tensor_core_real_shapes(B, H, Nq, Nk, hd, layout, sample):
    scale = hd ** -0.5
    q, k, v, do = inputs(B, H, Nq, Nk, hd, scale, seed=Nq)
    got = run_xattn(q, k, v, do, scale, TC, layout)
    check_against_fp64(f'xattn tc hd{hd} {Nq}x{Nk} {layout}', got, q, k, v, do, scale, 'bf16', False, sample=sample)


@pytest.mark.parametrize('hd', [64, 96])
def test_xattn_cuda_core_and_tensor_core_kernels_agree(hd):
    """The CUDA-core kernels (impl 1) and the tensor-core kernels on the same inputs, each within its own budget."""
    scale = hd ** -0.5
    q, k, v, do = inputs(2, 2, 197, 129, hd, scale, seed=5)
    for impl, mode in ((SIMT, 'bf16_out'), (TC, 'bf16')):
        got = run_xattn(q, k, v, do, scale, impl, 'head')
        check_against_fp64(f'xattn impl{impl} hd{hd} 197x129', got, q, k, v, do, scale, mode, False)


def test_xattn_delta_is_rowsum_of_do_times_o():
    q, k, v, do = inputs(1, 2, 129, 65, 96, 0.1, seed=6)
    got = run_xattn(q, k, v, do, 0.1, TC, 'head')
    ref = (do * got['o']).sum(-1)
    assert float((got['delta'] - ref).abs().max()) < 1e-4 * float(ref.abs().max())


# ---- packed-qkv attention (vt_attn_*): every implementation, dispatch thresholds ----------------------------------------
ATTN_N = [8, 9, 32, 33, 63, 64, 65, 128, 129, 197, 255, 256, 257, 289]


def picked(N):
    return WARP8 if N == 8 else (TC if N > 32 else SIMT)


@pytest.mark.parametrize('impl', [SIMT, TC, WARP8])
@pytest.mark.parametrize('N', ATTN_N)
def test_attn_packed_each_implementation(N, impl):
    if impl == WARP8 and N != 8:
        pytest.skip('the warp-per-problem kernel takes N = 8 only (refusal checked below)')
    if impl == SIMT and N > 256:
        pytest.skip('the generic kernel takes N <= 256 only (refusal checked below)')
    scale = 0.125
    q, k, v, do = inputs(2, 3, N, N, 64, scale, seed=N + impl)
    got = run_attn(q, k, v, do, scale, impl)
    check_against_fp64(f'attn impl{impl} N{N}', got, q, k, v, do, scale, 'bf16' if impl == TC else 'bf16_out', True)


@pytest.mark.parametrize('N', ATTN_N)
def test_attn_packed_auto_dispatch(N):
    """impl 0 picks warp8 at N = 8, the tensor-core kernel for N > 32 and the generic kernel otherwise: bitwise the same
    results as the implementation asked for by name."""
    q, k, v, do = inputs(2, 3, N, N, 64, 0.125, seed=N)
    a, b = run_attn(q, k, v, do, 0.125, AUTO), run_attn(q, k, v, do, 0.125, picked(N))
    for n in a:
        assert torch.equal(a[n], b[n]), (N, n)


def test_attn_packed_refusals_at_kernel_limits():
    q, k, v, do = inputs(1, 1, 257, 257, 64, 0.125)
    with pytest.raises(RuntimeError, match='N=257 unsupported'):
        run_attn(q, k, v, do, 0.125, SIMT)
    for n in (9, 257):
        q, k, v, do = inputs(1, 1, n, n, 64, 0.125)
        with pytest.raises(RuntimeError, match='warp8 kernel needs N == 8'):
            run_attn(q, k, v, do, 0.125, WARP8)


@pytest.mark.parametrize('scale', [1.0, 0.05])
@pytest.mark.parametrize('regime', ['max_last', 'max_first', 'uniform'])
def test_attn_packed_tensor_core_logit_regimes(regime, scale):
    q, k, v, do = inputs(2, 2, 197, 197, 64, scale, regime, seed=11)
    got = run_attn(q, k, v, do, scale, TC)
    check_against_fp64(f'attn tc {regime} scale {scale}', got, q, k, v, do, scale, 'bf16', True)


# ---- determinism, batch independence, grid limits -----------------------------------------------------------------------
@pytest.mark.parametrize('hd', [64, 96])
def test_tensor_core_results_are_deterministic_and_per_problem(hd):
    """Two runs are bitwise equal (no atomics, every dK / dV element written once), and problem 1's results do not change when
    every other problem of the batch is scaled by 50."""
    scale = hd ** -0.5
    q, k, v, do = inputs(3, 2, 193, 135, hd, scale, seed=12)
    a, b = run_xattn(q, k, v, do, scale, TC, 'head'), run_xattn(q, k, v, do, scale, TC, 'head')
    for n in a:
        assert torch.equal(a[n], b[n]), n
    wild = [x.clone() for x in (q, k, v, do)]
    for x in wild:
        x[0] *= 50
        x[2] *= 50
    c = run_xattn(*wild, scale, TC, 'head')
    for n in a:
        assert torch.equal(a[n][1], c[n][1]), n
    if hd == 64:
        qp, kp, vp, dop = inputs(2, 3, 197, 197, 64, 0.125, seed=13)
        x, y = run_attn(qp, kp, vp, dop, 0.125, TC), run_attn(qp, kp, vp, dop, 0.125, TC)
        for n in x:
            assert torch.equal(x[n], y[n]), n


def test_grid_limit_on_problems():
    """B * H = 65 535 problems (one grid dimension) are accepted with Nq = Nk = 1 and computed right; 65 536 are refused."""
    B, hd, scale = 65535, 64, 0.125
    q, k, v, do = inputs(B, 1, 1, 1, hd, scale, seed=14)
    got = run_xattn(q, k, v, do, scale, TC, 'head')
    assert torch.equal(got['o'], v)                                    # one key: P = 1, o = v
    assert torch.equal(got['dv'], do)
    lse = (q * k).sum(-1) * scale
    assert float(((got['lse'] - lse).abs() / (1 + lse.abs())).max()) < AE.LSE_TOL
    assert float(got['dq'].abs().max()) < 1e-3 and float(got['dk'].abs().max()) < 1e-3
    att = run_attn(q.view(B, 1, 1, hd), k.view(B, 1, 1, hd), v.view(B, 1, 1, hd), do.view(B, 1, 1, hd), scale, TC)
    assert torch.equal(att['o'], v)
    q, k, v, do = inputs(65536, 1, 1, 1, hd, scale, seed=15)
    with pytest.raises(RuntimeError, match='bad dims'):
        run_xattn(q, k, v, do, scale, TC, 'head')
    with pytest.raises(RuntimeError, match='B\\*H too large'):
        run_attn(q, k, v, do, scale, TC)
