"""vt_gemm element by element.

A. Exact regime (tests/gemm_exact.py): integer operands and dyadic epilogue operands make every fp32 step exact, so each
   output must equal the float64 result rounded once, bit for bit: every form, both epilogue paths, every tile width and
   operand layout, tile / k-block edges, split-K, the persistent walk on reduced grids and M a few rows past a tile.
   Which kernel each configuration reaches is read from torch.profiler, in one session in a child process
   (test_dispatch_reaches_every_register_and_staged_cell): a profiler session per case, in the process that runs the
   suite, left the later sessions of that process without records of kernels that had already run, and so blinded the
   profiler checks of other modules.
B. Every operand is a view into a NaN-filled allocation (padded pitch, rows past K / M / N), and every output lives in a
   sentinel-filled buffer with a padded pitch, so a read the tensor maps should have clipped turns
   outputs into NaN, and a stray write changes a sentinel.
C. GELU over all 65 536 bf16 inputs: the stand-alone kernels against the float64 GELU within the derived per-element
   bound of tests/gemm_exact.py, and the forward-only gelu_h epilogue bit for bit against the stand-alone kernel.
D. Gaussian operands at the model's shapes against float64 within K 2^-23 (|A||B|)_mn plus the epilogue's roundings.
E. Host checks of the reference arithmetic (no GPU).
"""

import math
import re

import numpy as np
import pytest
import torch

from tests import gemm_exact as X

FORMS = ('bf16', 'f32', 'gelu_h')
SENT16 = 0x7FAB                          # bf16 NaN payload no kernel writes
SENT32 = 0x7FC0DEAD                      # fp32 NaN payload no kernel writes


def K():
    from videotransformer_pytorch_b200 import _lib
    return _lib.K


def lib():
    from videotransformer_pytorch_b200 import _lib
    return _lib


# ---- buffers --------------------------------------------------------------------------------------------------------
def _ld(cols, pad, align):
    ld = cols + pad
    return ld + (-ld) % align


def nan_view(t, pad, dtype=torch.bfloat16, align=8):
    """t copied into the top-left of a NaN-filled [rows + pad, ld] allocation (ld >= cols + pad, a multiple of align)"""
    rows, cols = t.shape
    buf = torch.full((rows + pad, _ld(cols, pad, align)), float('nan'), dtype=dtype, device='cuda')
    buf[:rows, :cols] = t.to(device='cuda', dtype=dtype)
    return buf[:rows, :cols]


class Out:
    """a sentinel-filled output buffer with padded pitch and extra rows; .view is the [rows, cols] operand"""

    def __init__(self, rows, cols, dtype, pad):
        self.dtype, self.rows, self.cols = dtype, rows, cols
        ib = torch.int16 if dtype == torch.bfloat16 else torch.int32
        self.buf = torch.full((rows + pad, _ld(cols, pad, 8)), SENT16 if ib == torch.int16 else SENT32, dtype=ib,
                              device='cuda')
        self.view = self.buf.view(dtype)[:rows, :cols]

    def expected(self, rows, values):
        """the whole buffer's bits with `values` [len(rows), cols] written at `rows` and sentinels elsewhere"""
        ib = self.buf.dtype
        full = torch.full_like(self.buf, SENT16 if ib == torch.int16 else SENT32)
        full[rows, :self.cols] = values.to(self.dtype).contiguous().view(ib)
        return full

    def check(self, exp, tag):
        got = self.buf
        bad = got != exp
        if bool(bad.any()):
            i = bad.nonzero()[0].tolist()
            g, e = got[i[0], i[1]].item(), exp[i[0], i[1]].item()
            raise AssertionError(f'{tag}: {int(bad.sum())} of {bad.numel()} elements differ; first at {i}: '
                                 f'got bits {g & 0xFFFFFFFF:#x}, expected {e & 0xFFFFFFFF:#x}')


def parse_cell(name):
    """kernel name -> its (kernel, SE, BN, TA, TB) cell, or None for a kernel that is not a GEMM"""
    m = re.search(r'gemm_wgmma_kernel<(\d+), ?(\d+), ?(\d+), ?(\d+)>', name)
    if m:
        bn, ta, tb, se = map(int, m.groups())
        return ('wgmma', se, bn, ta, tb)
    m = re.search(r'gemm_f32_kernel<(\d+), ?(\d+), ?(\d+)>', name)
    if m:
        bn, ta, tb = map(int, m.groups())
        return ('f32', 3, bn, ta, tb)
    return None


def expected_cell(form, staged, bn, ta, tb):
    if not staged:
        return ('wgmma', 0, bn, ta, tb)
    if form in ('bf16', 'gelu_h'):
        return ('wgmma', 1, bn, ta, tb)
    return ('wgmma', 0, bn, ta, tb) if bn == 256 else ('f32', 3, bn, ta, tb)


# ---- one exact-regime call --------------------------------------------------------------------------------------------
def int_operands(M, N, Kd, ta, tb, seed, pad):
    """A [M, K], B [N, K] integer matrices (CPU) and the NaN-padded bf16 operands in the requested layouts"""
    A, B = X.int_operand((M, Kd), seed), X.int_operand((N, Kd), seed + 1)
    a = nan_view(A.t() if ta else A, pad)
    b = nan_view(B.t() if tb else B, pad)
    return A, B, a, b


def run_exact(form, M, N, Kd, *, ta=0, tb=0, bn=0, seed=0, pad=8, bias=False, rs=False, aux=False, bias2=False,
              rowmap=False, tag=''):
    """one vt_gemm call in the exact regime, checked bit for bit over its whole output buffers"""
    A, B, a, b = int_operands(M, N, Kd, ta, tb, seed, pad)
    g = seed * 7 + 3
    bias_t = X.quarter_values((N,), g) if bias else None
    rs_t = X.pow2_scale(M, g + 1) if rs else None
    Raux = M + 5
    aux_t = X.quarter_values((Raux, N), g + 2) if aux and form == 'f32' else None
    bias2_t = X.quarter_values((N,), g + 3) if bias2 and aux_t is not None else None
    X.exact_premise(Kd, bias=bias_t, bias2=bias2_t, aux=aux_t, row_scale=rs_t)
    kw = dict(a_mn=bool(ta), b_mn=bool(tb), epi=form, force_bn=bn)
    if bias_t is not None:
        kw['bias'] = nan_view(bias_t[None], 4, torch.float32, 4)[0]
    if rs_t is not None:
        kw['row_scale'] = nan_view(rs_t[None], 4, torch.float32, 4)[0]
    if bias2_t is not None:
        kw['bias2'] = nan_view(bias2_t[None], 4, torch.float32, 4)[0]
    gen = torch.Generator(device='cpu').manual_seed(g + 4)
    R = M
    rows = torch.arange(M)
    if rowmap:
        R = M + 3
        rows = torch.randperm(R, generator=gen)[:M]
        rows[torch.rand(M, generator=gen) < 0.15] = -1
        kw['out_row'] = rows.int().cuda()
        kw['out_rows'] = R
    arow = torch.arange(M)
    if aux_t is not None:
        if rowmap:
            arow = torch.randperm(Raux, generator=gen)[:M]
            arow[torch.rand(M, generator=gen) < 0.15] = -1
            kw['aux_row'] = arow.int().cuda()
        kw['aux'] = nan_view(aux_t, 2, torch.float32, 4)
    odt = torch.float32 if form == 'f32' else torch.bfloat16
    out = Out(R, N, odt, 3)
    kw['out'] = out.view
    K().gemm(a, b, M, N, Kd, **kw)

    v = A.double().cuda() @ B.double().cuda().t()
    if bias_t is not None:
        v = v + bias_t.double().cuda()
    if rs_t is not None:
        v = v * rs_t.double().cuda()[:, None]
    if form == 'f32':
        v = v + 0.0                                    # the addend is +0 where there is none: -0 comes out +0
        if aux_t is not None:
            add = aux_t.double().cuda()[arow.clamp(min=0)] * (arow >= 0).double().cuda()[:, None]
            v = v + add
        if bias2_t is not None:
            v = v + bias2_t.double().cuda()
    keep = rows >= 0
    dst = rows[keep].cuda()
    tag = f'{tag} {form} M={M} N={N} K={Kd} ta={ta} tb={tb} bn={bn} bias={bias} rs={rs} aux={aux} bias2={bias2} map={rowmap}'
    if form == 'f32':
        out.check(out.expected(dst, X.round_once(v, torch.float32)[keep.cuda()]), tag)
    elif form == 'bf16':
        out.check(out.expected(dst, X.round_once(v, torch.bfloat16)[keep.cuda()]), tag)
    else:  # gelu_h
        h = K().gelu(X.round_once(v, torch.bfloat16).contiguous())
        out.check(out.expected(dst, h[keep.cuda()]), tag)


def variants(form):
    if form in ('bf16', 'gelu_h'):
        return [{}, dict(bias=True), dict(rs=True), dict(bias=True, rs=True), dict(bias=True, rs=True, rowmap=True)]
    return [{}, dict(bias=True), dict(rs=True), dict(aux=True), dict(aux=True, bias2=True),
            dict(bias=True, rs=True, aux=True, bias2=True), dict(bias=True, rs=True, aux=True, bias2=True, rowmap=True),
            dict(bias=True, rowmap=True)]


# M, N, K: partial row and column tiles, one row, below one k-block, partial last k-blocks, several n-tiles
CELL_SHAPES = ((129, 200, 136), (1, 8, 8), (8, 72, 40), (127, 776, 72))


# ---- A / B: the kernel cells ----------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize('tb', [0, 1])
@pytest.mark.parametrize('ta', [0, 1])
@pytest.mark.parametrize('bn', [128, 192, 256, 0])
@pytest.mark.parametrize('staged', [0, 1])
@pytest.mark.parametrize('form', FORMS)
def test_exact_cell(form, staged, bn, ta, tb, monkeypatch):
    """every form x epilogue path x tile width x operand layout on small edge shapes, bit for bit (the kernel each of
    these configurations reaches: test_dispatch_reaches_every_register_and_staged_cell)"""
    monkeypatch.setenv('VT_GEMM_STAGED_EPI', str(staged))
    for i, (M, N, Kd) in enumerate(CELL_SHAPES):
        for j, var in enumerate(variants(form)):
            run_exact(form, M, N, Kd, ta=ta, tb=tb, bn=bn, seed=100 * i + j, pad=8 * (1 + (i + j) % 2), **var)


def dispatch_probe():
    """Body of the child process of test_dispatch_reaches_every_register_and_staged_cell: one vt_gemm call per
    configuration of test_exact_cell (shape 129 x 200 x 136), all inside one torch.profiler session, with every operand
    allocated before it.  Prints one JSON line: the configurations in call order and the cells of the GEMM kernels in
    launch order."""
    import itertools
    import json
    import os
    from torch.profiler import ProfilerActivity, profile
    M, N, Kd = 129, 200, 136
    calls = []
    for form, staged, bn, ta, tb in itertools.product(FORMS, (0, 1), (128, 192, 256, 0), (0, 1), (0, 1)):
        _, _, a, b = int_operands(M, N, Kd, ta, tb, seed=1, pad=8)
        kw = dict(a_mn=bool(ta), b_mn=bool(tb), epi=form, force_bn=bn,
                  out=torch.empty((M, N), dtype=torch.float32 if form == 'f32' else torch.bfloat16, device='cuda'))
        calls.append(([form, staged, bn, ta, tb], {'VT_GEMM_STAGED_EPI': str(staged)}, (a, b, M, N, Kd), kw))
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _, env, args, kw in calls:
            os.environ.update(env)
            K().gemm(*args, **kw)
        torch.cuda.synchronize()
    launched = sorted((e.time_range.start, parse_cell(e.name)) for e in prof.events()
                      if e.device_type == torch.autograd.DeviceType.CUDA and parse_cell(e.name))
    print(json.dumps(dict(configs=[c[0] for c in calls], kernels=[list(c) for _, c in launched])))


@pytest.mark.gpu
def test_dispatch_reaches_every_register_and_staged_cell():
    """The kernel cell each configuration of test_exact_cell reaches: every (kernel, SE, BN, TA, TB) cell of the bf16
    wgmma GEMM that the dispatch can reach.  Calls run in order on one stream, so the i-th GEMM kernel launched belongs
    to the i-th call."""
    import json
    import os
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    cmd = [sys.executable] + (['-s'] if sys.flags.no_user_site else []) + \
        ['-c', 'from tests.test_gpu_gemm_exact import dispatch_probe; dispatch_probe()']
    res = subprocess.run(cmd, cwd=root, capture_output=True, text=True, timeout=600)
    assert res.returncode == 0, res.stdout[-2000:] + res.stderr[-4000:]
    out = json.loads(res.stdout.strip().splitlines()[-1])
    configs, kernels = out['configs'], [tuple(k) for k in out['kernels']]
    assert len(kernels) == len(configs), (len(kernels), len(configs))
    reached = {}
    for cfg, cell in zip(configs, kernels):
        form, staged, bn, ta, tb = cfg
        want = expected_cell(form, staged, bn, ta, tb) if bn else (cell[0], cell[1], cell[2], ta, tb)
        assert cell == want, (cfg, cell, want)
        reached.setdefault(cell, []).append(cfg)
    want_cells = {('wgmma', se, bn, ta, tb) for se in (0, 1) for bn in (128, 192, 256) for ta in (0, 1) for tb in (0, 1)}
    want_cells |= {('f32', 3, bn, ta, tb) for bn in (128, 192) for ta in (0, 1) for tb in (0, 1)}
    assert want_cells <= set(reached), sorted(want_cells - set(reached))
    for cell in sorted(reached):
        print(cell, '<-', reached[cell][:3], f'({len(reached[cell])} configurations)')


@pytest.mark.gpu
@pytest.mark.parametrize('form,M,N,Kd,tb', [('bf16', 12552, 2304, 768, 0), ('bf16', 12552, 768, 2304, 1),
                                            ('f32', 12552, 768, 3072, 0), ('gelu_h', 12552, 3072, 768, 0)])
def test_exact_persistent_walk(form, M, N, Kd, tb, monkeypatch):
    """the model's shapes with every SM, one fewer and 64 fewer: many tiles per CTA, each CTA's ring and staging buffers
    reused across tiles of different row and column blocks"""
    var = dict(bias=True, rs=True, aux=True, bias2=True) if form == 'f32' else dict(bias=True, rs=True)
    try:
        for reserve in (0, 1, 64):
            lib().set_reserved_sms(reserve)
            for staged in (0, 1):
                monkeypatch.setenv('VT_GEMM_STAGED_EPI', str(staged))
                run_exact(form, M, N, Kd, tb=tb, seed=7, pad=8, tag=f'reserve={reserve} staged={staged}', **var)
    finally:
        lib().set_reserved_sms(0)


@pytest.mark.gpu
@pytest.mark.parametrize('bn', [128, 192, 256])
@pytest.mark.parametrize('zeroed', [False, True], ids=['sentinel', 'zeroed'])
def test_exact_split_k(zeroed, bn, monkeypatch):
    """weight-gradient form (both operands MN-major) with forced splits that do not divide the k-block count: partials
    through the workspace, summed into a sentinel-filled output and into a zeroed one: prior contents never matter.  The
    kernels these calls take are the cells of test_exact_cell with one split; test_gpu_gemm_staged_f32 checks which one a
    split call picks."""
    for M, N, Kd, splits in ((776, 200, 12552, (2, 5, 16)), (768, 768, 3072, (5, 7)), (136, 72, 584, (3,))):
        A, B, a, b = int_operands(M, N, Kd, 1, 1, seed=M + Kd, pad=8)
        X.exact_premise(Kd)
        ref = X.round_once(A.double().cuda() @ B.double().cuda().t(), torch.float32)
        kb = (Kd + 63) // 64
        for sp in splits:
            assert kb % sp, (kb, sp)
            for staged in (0, 1):
                monkeypatch.setenv('VT_GEMM_STAGED_EPI', str(staged))
                buf = torch.zeros((M + 3, N), device='cuda') if zeroed else \
                    torch.full((M + 3, N), SENT32, dtype=torch.int32, device='cuda').view(torch.float32)
                tail = buf[M:].clone()
                K().gemm(a, b, M, N, Kd, a_mn=True, b_mn=True, epi='f32', split_ok=True, force_splits=sp,
                         force_bn=bn, out=buf[:M])
                tag = (M, N, Kd, sp, bn, staged, zeroed)
                assert torch.equal(buf[:M].view(torch.int32), ref.view(torch.int32)), tag
                assert torch.equal(buf[M:].view(torch.int32), tail.view(torch.int32)), tag


@pytest.mark.gpu
@pytest.mark.parametrize('M,N,Kd,tb', [(1032, 200, 2048, 0), (1040, 768, 2048, 1), (1032, 1024, 2048, 1),
                                      (12552, 768, 3072, 0), (12552, 768, 3072, 1), (1025, 768, 2304, 0),
                                      (1025, 768, 2304, 1), (1040, 384, 4096, 0), (1040, 384, 4096, 1)])
def test_exact_remainder_rows(M, N, Kd, tb):
    """M 1 to 16 rows past a multiple of 128 with long K: a last row of tiles that is nearly all padding, with every
    epilogue operand of the bf16 and fp32 forms"""
    for form, var in (('bf16', dict(bias=True, rs=True)), ('f32', dict(bias=True, rs=True, aux=True, bias2=True)),
                      ('f32', dict(aux=True)), ('bf16', {})):
        run_exact(form, M, N, Kd, tb=tb, seed=N, pad=8, **var)


@pytest.mark.gpu
@pytest.mark.parametrize('shape', [(3, 4, 9, 136), (2, 8, 196, 768)])
@pytest.mark.parametrize('bn', [0, 128, 192, 256])
def test_exact_affine_maps(shape, bn, monkeypatch):
    """the residual stream regrouped in place by the affine row maps (temporal, and spatial with the cls replicas going
    to the side rows), against the index-array definition of the same maps"""
    from videotransformer_pytorch_b200 import ops
    B, T, P, D = shape
    S = 1 + P * T
    maps, aff = ops.token_maps(B, T, P, 'cuda'), ops.affine_row_maps(B, T, P, D)
    stream = X.quarter_values((B * S + B * T, D), D).cuda()
    w = X.int_operand((D, D), 1)
    bias, bias2 = X.quarter_values((D,), 2), X.quarter_values((D,), 3)
    for kind in ('temporal', 'spatial'):
        M = B * P * T if kind == 'temporal' else B * T * (P + 1)
        x = X.int_operand((M, D), 4)
        rs = X.pow2_scale(M, 5)
        X.exact_premise(D, bias=bias, bias2=bias2, aux=stream, row_scale=rs)
        out_row = maps['temporal'] if kind == 'temporal' else maps['sp_out']
        aux_row = maps['temporal'] if kind == 'temporal' else maps['sp_aux']
        v = (x.double() @ w.double().t() + bias.double()) * rs.double()[:, None] + bias2.double()
        v = v.cuda() + stream.double()[aux_row.long().clamp(min=0)] * (aux_row >= 0).double()[:, None]
        exp = stream.clone()
        exp[out_row.long()] = X.round_once(v, torch.float32)
        for staged in (0, 1):
            monkeypatch.setenv('VT_GEMM_STAGED_EPI', str(staged))
            buf = stream.clone()
            K().gemm(nan_view(x, 8), nan_view(w, 8), M, D, D, epi='f32', aux=buf, out=buf, aux_row=aux_row,
                     out_row=out_row, row_map=aff[kind], bias=bias.cuda(), bias2=bias2.cuda(), row_scale=rs.cuda(),
                     force_bn=bn)
            assert torch.equal(buf.view(torch.int32), exp.view(torch.int32)), (shape, kind, bn, staged)


# ---- C: GELU over every bf16 input ---------------------------------------------------------------------------------
def all_bf16():
    """the 65 536 bf16 bit patterns as a [256, 256] int16 matrix, pattern i at row i // 256, column i % 256"""
    return torch.arange(-32768, 32768, dtype=torch.int32).to(torch.int16).reshape(256, 256)


REGIONS = (('negative tail z < -4', lambda z: z < -4), ('-4 <= z <= -1', lambda z: (z >= -4) & (z <= -1)),
           ('|z| < 1', lambda z: np.abs(z) < 1), ('2 <= |z| <= 4', lambda z: (np.abs(z) >= 2) & (np.abs(z) <= 4)),
           ('positive z > 4', lambda z: z > 4))


def ratio_report(name, z, got, ref, bound):
    ratio = np.abs(got - ref) / bound
    lines = [f'{name}: max |got - ref| / bound']
    for rn, sel in REGIONS:
        m = sel(z)
        k = int(np.argmax(np.where(m, ratio, -1)))
        lines.append(f'  {rn:>22}: {float(ratio[m].max()):.3f} at z = {z[k]:.6g} (got {got[k]:.6g}, fp64 {ref[k]:.6g})')
    print('\n'.join(lines))
    return ratio


@pytest.mark.gpu
def test_gelu_every_bf16_input():
    """K.gelu and K.dgelu (dh = 1) on every bf16 pattern: finite inputs within the derived bound of the fp64 GELU, NaN to
    NaN, and the current results at +-inf pinned (torch gives NaN for gelu'(+-inf) and gelu(-inf) too)"""
    bits = all_bf16().cuda()
    zb = bits.view(torch.bfloat16)
    h = K().gelu(zb).float().cpu().double().numpy().ravel()
    d = K().dgelu(torch.ones_like(zb), zb).float().cpu().double().numpy().ravel()
    z = zb.float().cpu().double().numpy().ravel()
    fin = np.isfinite(z)
    assert np.isnan(h[np.isnan(z)]).all() and np.isnan(d[np.isnan(z)]).all()
    pinf, ninf = z == np.inf, z == -np.inf
    assert (h[pinf] == np.inf).all() and np.isnan(h[ninf]).all(), (h[pinf], h[ninf])
    assert np.isnan(d[pinf]).all() and np.isnan(d[ninf]).all(), (d[pinf], d[ninf])
    zf = z[fin]
    for name, got, ref, bound in (('gelu', h[fin], X.gelu64(zf), X.gelu_bound(zf)),
                                  ('gelu\'', d[fin], X.dgelu64(zf), X.dgelu_bound(zf))):
        assert np.isfinite(got).all(), name
        ratio = ratio_report(name, zf, got, ref, bound)
        worst = int(np.argmax(ratio))
        assert ratio[worst] <= 1.0, (name, zf[worst], got[worst], ref[worst], bound[worst])


@pytest.mark.gpu
@pytest.mark.parametrize('staged', [0, 1])
@pytest.mark.parametrize('bn', [0, 128, 256])
def test_gelu_h_epilogue_every_bf16_input(bn, staged, monkeypatch):
    """the same patterns as GEMM outputs (a = the pattern matrix, b = identity): gelu_h's output must equal the
    stand-alone kernel's result bit for bit.  Non-finite patterns cannot pass through the MMA (NaN / inf times the
    identity's zeros spoils the row) and neither can -0 (the zeros of the other products make it +0): those enter a as 0
    and are checked by the stand-alone test."""
    monkeypatch.setenv('VT_GEMM_STAGED_EPI', str(staged))
    bits = all_bf16().cuda()
    pat = bits.view(torch.bfloat16)
    ok = torch.isfinite(pat) & (bits != -0x8000)
    a = torch.where(ok, pat, torch.zeros_like(pat))
    eye = torch.eye(256, device='cuda').bfloat16()
    table_h = K().gelu(a)
    h = K().gemm(nan_view(a, 8), nan_view(eye, 8), 256, 256, 256, epi='gelu_h', force_bn=bn)
    assert torch.equal(h.contiguous().view(torch.int16), table_h.view(torch.int16))


# ---- D: random operands against the fp64 bound --------------------------------------------------------------------
def gauss(shape, seed):
    g = torch.Generator(device='cpu').manual_seed(seed)
    return torch.randn(shape, generator=g)


D_CASES = [  # name, M, N, K, ta, tb, form, epilogue operands, extra gemm arguments
    ('qkv', 12552, 2304, 768, 0, 0, 'bf16', ('bias',), {}),
    ('proj+res', 12552, 768, 768, 0, 0, 'f32', ('bias', 'rs', 'aux', 'bias2'), {}),
    ('fc1', 12552, 3072, 768, 0, 0, 'bf16', ('bias',), {}),
    ('fc2+res', 12552, 768, 3072, 0, 0, 'f32', ('bias', 'aux'), {}),
    ('fc2+res rs bias2', 12552, 768, 3072, 0, 0, 'f32', ('bias', 'rs', 'aux', 'bias2'), {}),
    ('fc1 dgrad', 12552, 768, 3072, 0, 1, 'bf16', ('rs',), {}),
    ('qkv dgrad', 12552, 768, 2304, 0, 1, 'f32', (), {}),
    ('fc2 dgrad', 12552, 3072, 768, 0, 1, 'bf16', (), {}),
    ('fc1 wgrad split', 3072, 768, 12552, 1, 1, 'f32', (), dict(split_ok=True)),
    ('fc2 wgrad split 5', 768, 3072, 12552, 1, 1, 'f32', (), dict(split_ok=True, force_splits=5)),
    ('mvit s1 fc2', 50184, 96, 384, 0, 0, 'f32', ('bias', 'aux'), {}),
]


@pytest.mark.gpu
@pytest.mark.parametrize('case', D_CASES, ids=[c[0] for c in D_CASES])
def test_random_operands_within_fp64_bound(case):
    name, M, N, Kd, ta, tb, form, epi_ops, extra = case
    A, B = gauss((M, Kd), M + N).bfloat16().double(), gauss((N, Kd), Kd).bfloat16().double()
    a = (A.t() if ta else A).contiguous().bfloat16().cuda()
    b = (B.t() if tb else B).contiguous().bfloat16().cuda()
    kw = dict(a_mn=bool(ta), b_mn=bool(tb), epi=form, **extra)
    bias = gauss((N,), 1).cuda() if 'bias' in epi_ops else None
    rs = (gauss((M,), 2).abs() + 0.5).cuda() if 'rs' in epi_ops else None
    aux = gauss((M, N), 3).cuda() * 4 if 'aux' in epi_ops else None
    bias2 = gauss((N,), 4).cuda() if 'bias2' in epi_ops else None
    for k, t in (('bias', bias), ('row_scale', rs), ('aux', aux), ('bias2', bias2)):
        if t is not None:
            kw[k] = t
    got = K().gemm(a, b, M, N, Kd, **kw).double()
    Ad, Bd = A.cuda(), B.cuda()
    ref = Ad @ Bd.t()
    absprod = Ad.abs() @ Bd.abs().t()
    del Ad, Bd
    T = absprod.clone()
    if bias is not None:
        ref += bias.double()
        T += bias.double().abs()
    s = None
    if rs is not None:
        s = rs.double()[:, None]
        ref *= s
        T *= s
    if aux is not None:
        ref += aux.double()
        T += aux.double().abs()
    if bias2 is not None:
        ref += bias2.double()
        T += bias2.double().abs()
    splits = extra.get('force_splits', 16 if extra.get('split_ok') else 1)
    bound = X.accumulation_bound(Kd, absprod, scale=s, epi_terms=T, splits=splits,
                                 bf16_ref=ref.abs() if form == 'bf16' else None)
    ratio = ((got - ref).abs() / bound)
    worst = float(ratio.max())
    print(f'{name} {M}x{N}x{Kd} {form}: max |got - ref| / bound = {worst:.3e}')
    assert torch.isfinite(got).all() and worst <= 1.0, (name, worst)


# ---- E: host checks of the reference arithmetic ----------------------------------------------------------------------
def test_generators_satisfy_exactness_premise():
    a = X.int_operand((64, 300), 1)
    assert bool((a == a.round()).all()) and int(a.abs().max()) == 3 and set(a.unique().tolist()) == set(range(-3, 4))
    assert torch.equal(a.bfloat16().float(), a)
    q = X.quarter_values((4096,), 2, limit=X.QUARTER_LIMIT)
    assert bool(((q * 4) == (q * 4).round()).all()) and float(q.abs().max()) < X.QUARTER_LIMIT
    s = X.pow2_scale(4096, 3)
    assert set(s.abs().log2().round().int().unique().tolist()) == set(range(X.SCALE_EXP[0], X.SCALE_EXP[1] + 1))
    assert bool((s > 0).any()) and bool((s < 0).any())
    bits = X.exact_premise(4096, bias=q, bias2=q, aux=q[None].expand(3, -1), row_scale=s)
    assert bits < 24
    X.exact_premise(12552)                                            # split-K sums over the token count
    with pytest.raises(AssertionError):
        X.exact_premise(2 ** 21)                                      # 9 K >= 2^24
    with pytest.raises(AssertionError):
        X.exact_premise(64, bias=torch.tensor([0.125]))               # not a multiple of 1/4
    with pytest.raises(AssertionError):
        X.exact_premise(64, row_scale=torch.tensor([3.0]))            # not a power of two
    with pytest.raises(AssertionError):
        X.exact_premise(2 ** 20, bias=torch.tensor([0.25]))          # 9 K + bias over a resolution of 1/4 >= 2^24


def test_gelu_reference_against_known_values():
    from scipy.special import erf
    z = np.array([-6.0, -3.0, -1.0, -0.5, 0.0, 0.5, 1.0, 2.0, 3.0, 6.0])
    phi = 0.5 * (1 + erf(z / math.sqrt(2)))
    assert np.allclose(X.gelu64(z), z * phi, rtol=1e-15, atol=0)
    assert X.gelu64(np.array([1.0]))[0] == pytest.approx(0.8413447460685429, rel=1e-15)
    assert X.gelu64(np.array([-1.0]))[0] == pytest.approx(-0.15865525393145707, rel=1e-15)
    assert X.dgelu64(np.array([0.0]))[0] == 0.5
    zz = np.linspace(-5, 5, 101)
    hstep = 1e-6
    fd = (X.gelu64(zz + hstep) - X.gelu64(zz - hstep)) / (2 * hstep)
    assert np.allclose(X.dgelu64(zz), fd, atol=1e-8)


def test_bf16_rounding_is_nearest_even():
    def rne(vals):
        return X.bf16_rne_bits(torch.tensor(vals, dtype=torch.float32)).view(torch.bfloat16).float().tolist()
    # exact ties: 1 + 2^-8 lies between 1 and 1 + 2^-7; 257 between 256 and 258; 259 between 258 and 260
    assert rne([1 + 2 ** -8, 1 + 3 * 2 ** -8, 257.0, 259.0, -257.0, -259.0]) == [1.0, 1 + 2 ** -6, 256.0, 260.0, -256.0, -260.0]
    assert rne([1 + 2 ** -8 + 2 ** -20, 257.0 + 2 ** -10]) == [1 + 2 ** -7, 258.0]    # above the tie: up
    assert rne([3.3895313892515355e38, 3.4e38]) == [3.3895313892515355e38, math.inf]     # max bf16 stays, above rounds to inf
    assert math.isnan(rne([math.nan])[0]) and rne([math.inf, -math.inf, -0.0]) == [math.inf, -math.inf, -0.0]
    assert X.bf16_rne_bits(torch.tensor([-0.0]))[0] == -0x8000
    x = torch.randn(1 << 16, generator=torch.Generator().manual_seed(0)) * torch.exp2(torch.randint(-130, 120, (1 << 16,)).float())
    assert torch.equal(X.bf16_rne_bits(x), x.bfloat16().view(torch.int16))    # torch's conversion rounds to nearest even
    ints = torch.arange(256, 1 << 14, dtype=torch.float32)
    r = X.bf16_rne_bits(ints).view(torch.bfloat16).float()
    tie = (ints % 2 == 1) & (ints < 512)                            # odd integers in [256, 512) are exact ties
    assert bool(((r[tie] / 2) % 2 == 0).all())                      # ... and go to the even neighbour
    assert torch.equal(X.round_once(torch.tensor([257.0], dtype=torch.float64), torch.bfloat16).float(), torch.tensor([256.0]))
    with pytest.raises(AssertionError):
        X.round_once(torch.tensor([1 + 2.0 ** -30], dtype=torch.float64), torch.float32)


def test_bounds_are_monotone():
    z = np.linspace(-12, 12, 2001)
    for f in (X.gelu_bound, X.dgelu_bound):
        lo, hi = f(z, as_err=1e-7), f(z, as_err=2e-7)
        assert (hi >= lo).all()
        assert (f(z) > 0).all() and np.isfinite(f(z)).all()
    e = X.erf_fast_error(z)
    assert (e >= X.AS_ERR).all()
    hu = X.bf16_half_ulp(np.logspace(-40, 38, 5000))
    assert (np.diff(hu) >= 0).all()
    assert X.bf16_half_ulp(np.array([1.0, 1.99, 2.0]))[0] == 2.0 ** -8 and X.bf16_half_ulp(np.array([2.0]))[0] == 2.0 ** -7
    ht = X.bf16_half_ulp(torch.tensor([1.0, 1.99, 2.0, 0.0], dtype=torch.float64))
    assert ht.tolist() == [2.0 ** -8, 2.0 ** -8, 2.0 ** -7, 2.0 ** -134]
    G = torch.tensor([0.5, 1.0, 4.0], dtype=torch.float64)
    base = X.accumulation_bound(768, G, epi_terms=G + 1)
    assert bool((X.accumulation_bound(3072, G, epi_terms=G + 1) >= base).all())
    assert bool((X.accumulation_bound(768, G * 2, epi_terms=G + 1) >= base).all())
    assert bool((X.accumulation_bound(768, G, epi_terms=G + 2) >= base).all())
    assert bool((X.accumulation_bound(768, G, epi_terms=G + 1, splits=5) >= base).all())
    assert bool((X.accumulation_bound(768, G, epi_terms=G + 1, bf16_ref=G) >= base).all())
    assert bool((torch.diff(X.accumulation_bound(768, G)) >= 0).all())
