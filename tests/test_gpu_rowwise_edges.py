"""The row-wise kernels between the GEMMs element by element against fp64: LayerNorm forward / backward at every width the
entry points take (both backward generations), the dY producers with column sums, colsum, reduce_rows and cls_rows.  -m gpu

Every output is checked per element against the bounds of tests/rowwise_ref.py (shown to hold for an fp32 model and to
reject seeded defects in tests/test_rowwise_bounds.py).  The kernels are driven through ctypes: every output sits between
NaN guard rows and starts as NaN; x is a window of a NaN-filled wider buffer (ldx > D, 16 bytes into its row) whose rows
no in_row entry names are NaN; dx has a pitch wider than D, its rows out_row does not reach start as a sentinel and must
keep its bits; the partial-sum workspaces start as NaN, so a CTA that does not write its partial row shows.  Row counts
reach past the CTA cap (4 per SM, read from vt_sm_count()), where warps walk several rows.
"""
import pytest
import torch

from tests import rowwise_ref as R
from tests.test_gpu_attention_edges import Guarded, _call, _lib

pytestmark = pytest.mark.gpu

PAD = 8                      # rows past the end of every input, NaN
SENTINEL = 1234.5
NAN = float('nan')


def _sm():
    return _lib()[1].vt_sm_count()


def _bits(t):
    return t.contiguous().view(torch.int16 if t.dtype == torch.bfloat16 else torch.int32)


def _nan_rows(rows, width, dtype=torch.float32):
    return torch.full((rows + PAD, width), NAN, dtype=dtype, device='cuda')


def _reduce(partials, S, n, out, accumulate=0, scale=1.0, stride=None):
    lib_, lib = _lib()
    r = lib_.ReduceParams()
    r.inp, r.out, r.stride, r.S, r.n, r.accumulate, r.scale = partials.data_ptr(), out.data_ptr(), stride or n, S, n, accumulate, scale
    _call('vt_reduce_rows', r, 'vt_reduce_rows')


class LnRun:
    """one LayerNorm problem: x fp32 [R, D] (CPU) placed 16 bytes into the rows of a NaN-filled [R + PAD, D + 8] buffer;
    rows no in_row entry names are NaN"""

    def __init__(self, x, in_row, rows, gam, bet):
        self.R, self.D = x.shape
        self.rows, self.ldx = rows, self.D + 8
        self.buf = _nan_rows(self.R, self.ldx)
        named = torch.ones(self.R, dtype=torch.bool) if in_row is None else torch.zeros(self.R, dtype=torch.bool)
        if in_row is not None:
            named[in_row.long()] = True
        self.buf[:self.R, 4:4 + self.D] = torch.where(named[:, None], x, torch.full_like(x, NAN)).cuda()
        self.x = self.buf.data_ptr() + 16
        self.in_row = None if in_row is None else in_row.cuda()
        self.gam, self.bet = gam.cuda(), bet.cuda()

    def fwd(self, eps, y_fp32, stats=True):
        lib_, _ = _lib()
        y = Guarded(self.rows, self.D, torch.float32 if y_fp32 else torch.bfloat16)
        st = [Guarded(self.rows, 1, torch.float32) for _ in range(2)] if stats else [None, None]
        p = lib_.LnFwdParams()
        p.x, p.ldx, p.in_row = self.x, self.ldx, None if self.in_row is None else self.in_row.data_ptr()
        p.gamma, p.beta, p.y = self.gam.data_ptr(), self.bet.data_ptr(), y.inner.data_ptr()
        p.mean, p.rstd = (None, None) if not stats else (st[0].inner.data_ptr(), st[1].inner.data_ptr())
        p.rows, p.D, p.eps, p.y_fp32 = self.rows, self.D, eps, int(y_fp32)
        _call('vt_layernorm_fwd', p, 'vt_layernorm_fwd')
        y.check('y')
        out = dict(y=y.inner.view(self.rows, self.D).cpu())
        if stats:
            for n, t in zip(('mean', 'rstd'), st):
                t.check(n)
                out[n] = t.inner.cpu()
        return out

    def bwd(self, dy, mean, rstd, out_row=None, n_out=None, dres=None, n_aux=0, untouched=SENTINEL):
        """dy fp32 or bf16 [rows, D] (CPU); mean / rstd: the forward's; dres fp32 [n_out, D] (CPU) or None.  dx has pitch
        D + 8; its rows out_row does not reach start as `untouched` and must keep its bits.  -> dict of CPU dx_rows (the dx
        row of every m, from dx or dx_aux), dx (all n_out rows), dgamma, dbeta"""
        lib_, lib = _lib()
        D, rows = self.D, self.rows
        n_out = n_out or rows
        lddx = D + 8
        t = torch.arange(rows) if out_row is None else out_row.long()
        reached = torch.zeros(n_out, dtype=torch.bool)
        reached[t[t >= 0]] = True
        dx = Guarded(n_out, lddx, torch.float32)
        dx.inner.view(n_out, lddx)[~reached.cuda(), :D] = untouched
        aux = Guarded(n_aux, D, torch.float32) if n_aux else None
        dbuf = _nan_rows(rows, D, dy.dtype)
        dbuf[:rows] = dy.cuda()
        rbuf = None
        if dres is not None:
            rbuf = torch.full((n_out, lddx), NAN, device='cuda')
            rbuf[:, :D] = dres.cuda()
        blocks = lib.vt_ln_bwd_blocks(rows)
        partials = torch.full((blocks, 2, D), NAN, device='cuda')
        p = lib_.LnBwdParams()
        p.dy, p.dy_fp32 = dbuf.data_ptr(), int(dy.dtype == torch.float32)
        p.x, p.ldx, p.in_row = self.x, self.ldx, None if self.in_row is None else self.in_row.data_ptr()
        stats = (mean.cuda(), rstd.cuda())
        p.mean, p.rstd, p.gamma = stats[0].data_ptr(), stats[1].data_ptr(), self.gam.data_ptr()
        p.dres = None if rbuf is None else rbuf.data_ptr()
        p.dx, p.lddx = dx.inner.data_ptr(), lddx
        p.dx_aux = None if aux is None else aux.inner.data_ptr()
        ort = None if out_row is None else out_row.cuda()
        p.out_row = None if ort is None else ort.data_ptr()
        p.partials, p.rows, p.D = partials.data_ptr(), rows, D
        _call('vt_layernorm_bwd', p, 'vt_layernorm_bwd')
        gb = Guarded(2, D, torch.float32)
        _reduce(partials, blocks, 2 * D, gb.inner)
        dx.check('dx', torch.arange(D))
        if aux is not None:
            aux.check('dx_aux')
        gb.check('dgamma / dbeta')
        dxc = dx.inner.view(n_out, lddx)[:, :D].cpu()
        left = dxc[~reached]
        assert torch.equal(_bits(left), _bits(torch.full_like(left, untouched))), 'dx: a row out_row does not reach was written'
        dx_rows = torch.empty(rows, D)
        pos = t >= 0
        dx_rows[pos] = dxc[t[pos]]
        if n_aux:
            dx_rows[~pos] = aux.inner.view(n_aux, D).cpu()[-t[~pos] - 1]
        g = gb.inner.view(2, D).cpu()
        return dict(dx_rows=dx_rows, dgamma=g[0], dbeta=g[1])


def _maps(kind):
    from videotransformer_pytorch_b200.ops import token_maps
    B, T, P = 8, 8, 196
    m = token_maps(B, T, P, 'cpu')
    S = 1 + P * T
    if kind == 'temporal':
        return dict(R=B * S, in_row=m['temporal'], out_row=m['temporal'], n_aux=0)
    if kind == 'spatial':
        return dict(R=B * S, in_row=m['sp_in'], out_row=m['sp_bwd'], n_aux=B * T)
    return dict(R=B * S, in_row=m['cls_rows'], out_row=m['cls_rows'], n_aux=0)      # final norm (RowsNormFn)


def run_ln_case(D, rows, maps, regime, eps, monkeypatch, seed):
    rep = R.Report()
    sm = _sm()
    cls = maps == 'cls'
    mp = _maps(maps) if maps else dict(R=rows, in_row=None, out_row=None, n_aux=0)
    in_row = mp['in_row']
    rows = rows if in_row is None else in_row.numel()
    x = R.make_rows(mp['R'], D, regime, seed)
    gam, bet = R.make_affine(D, seed + 1)
    run = LnRun(x, in_row, rows, gam, bet)
    xs = x.double() if in_row is None else x.double()[in_row.long()]
    f16, f32 = run.fwd(eps, False), run.fwd(eps, True)
    for n in ('mean', 'rstd'):
        assert torch.equal(_bits(f16[n]), _bits(f32[n])), f'{n}: differs between the bf16 and fp32 forms'
    R.check_ln_forward(xs, f32['mean'], f32['rstd'], gam, bet, eps, f32['y'], rep, names=('mean', 'rstd', 'y32'))
    assert torch.equal(_bits(f16['y']), _bits(f32['y'].bfloat16())), 'y: bf16 store is not the rounded fp32 y'
    for y32 in (False, True):
        again = run.fwd(eps, y32, stats=False)
        assert torch.equal(_bits(again['y']), _bits((f32 if y32 else f16)['y'])), 'y: stats=False gives other bits'
    g = torch.Generator().manual_seed(seed + 2)
    dy32 = torch.randn(rows, D, generator=g)
    n_out = mp['R']
    dres = None if cls else torch.randn(n_out, D, generator=g)
    gens = (1, 2) if D % 128 == 0 else (1,)
    for dt in ((torch.float32,) if cls else (torch.float32, torch.bfloat16)):
        dy = dy32.to(dt)
        for gen in gens:
            monkeypatch.setenv('VT_LN_BWD_V2', str(gen - 1))
            got = run.bwd(dy, f32['mean'], f32['rstd'], mp['out_row'], n_out, dres, mp['n_aux'], 0.0 if cls else SENTINEL)
            again = run.bwd(dy, f32['mean'], f32['rstd'], mp['out_row'], n_out, dres, mp['n_aux'], 0.0 if cls else SENTINEL)
            for n in got:
                assert torch.equal(_bits(got[n]), _bits(again[n])), f'gen{gen} {n}: two calls differ'
            res = None
            if dres is not None:
                t = torch.arange(rows) if mp['out_row'] is None else mp['out_row'].long()
                pos = t >= 0
                r = torch.zeros(rows, D, dtype=torch.float64)
                r[pos] = dres.double()[t[pos]]
                res = (r, pos.double())
            d, xhat = R.check_ln_backward(xs, f32['mean'], f32['rstd'], gam, dy, got['dx_rows'], res, rep,
                                          name=f'dx_gen{gen}')
            R.check_dgamma_dbeta(d, xhat, got['dgamma'], got['dbeta'], sm, rep)
    return rep


# rows as (multiple of 8 * cap, offset): 1, 7, 8, 9 and 8 cap - 1, 8 cap, 8 cap + 1
ROW_SPECS = [(0, 1), (0, 7), (0, 8), (0, 9), (1, -1), (1, 0), (1, 1)]
EDGE_CASES = [(D, spec, None, R.REGIMES[(i + j) % len(R.REGIMES)], (1e-5, 1e-6)[j % 2])
              for i, D in enumerate(R.LN_WIDTHS + R.LN_SMALL_WIDTHS) for j, spec in enumerate(ROW_SPECS)]
MODEL_CASES = [(768, None, 'temporal', 'randn', 1e-5), (768, None, 'spatial', 'offset', 1e-5), (768, 12552, None, 'outlier', 1e-6),
               (768, None, 'temporal', 'constant', 1e-6), (768, None, 'spatial', 'tiny', 1e-6), (768, None, 'cls', 'randn', 1e-6),
               (96, 200712, None, 'randn', 1e-6), (192, 50184, None, 'offset', 1e-6), (384, 12552, None, 'tiny', 1e-6),
               (768, 3144, None, 'constant', 1e-6)]


def _case_id(c):
    D, rows, maps, regime, eps = c
    r = f'8cap{rows[1]:+d}' if isinstance(rows, tuple) and rows[0] else (rows[1] if isinstance(rows, tuple) else rows)
    return f'D{D}-rows{r}-{maps or "id"}-{regime}-eps{eps:g}'


@pytest.mark.parametrize('case', EDGE_CASES + MODEL_CASES, ids=_case_id)
def test_layernorm_against_fp64(case, monkeypatch):
    D, rows, maps, regime, eps = case
    if isinstance(rows, tuple):
        rows = rows[0] * 8 * R.ln_cap(_sm()) + rows[1]
    rep = run_ln_case(D, rows, maps, regime, eps, monkeypatch, seed=D + (rows or 0))
    print(f'[rowwise-edges] {_case_id(case)}: {rep}')


# ---- column sums -----------------------------------------------------------------------------------------------------
def _colsum(v, counters):
    """vt_colsum_bf16 of v bf16 [M, N] (CPU) read 16 bytes into the rows of a NaN-filled [M + PAD, N + 16] buffer"""
    lib_, lib = _lib()
    M, N = v.shape
    buf = _nan_rows(M, N + 16, torch.bfloat16)
    buf[:M, 8:8 + N] = v.cuda()
    out = Guarded(1, N, torch.float32)
    ws = torch.full((lib.vt_colsum_chunks(M), N), NAN, device='cuda')
    cnt = torch.zeros(1024, dtype=torch.int32, device='cuda')
    p = lib_.ColsumParams()
    p.inp, p.ld, p.M, p.N = buf.data_ptr() + 16, N + 16, M, N
    p.out, p.workspace, p.counters = out.inner.data_ptr(), ws.data_ptr(), cnt.data_ptr() if counters else None
    _call('vt_colsum_bf16', p, 'vt_colsum_bf16')
    out.check('colsum')
    assert not bool(cnt.any()), 'colsum: arrival counters not left at zero'
    return out.inner.cpu()


@pytest.mark.parametrize('M,N', [(1, 8), (511, 768), (512, 100), (513, 3072), (63, 96), (64, 2304), (65, 100), (12544, 768),
                                 (12552, 3072)])
def test_colsum_against_fp64(M, N):
    v = torch.randn(M, N, generator=torch.Generator().manual_seed(M * 7 + N)).bfloat16()
    rep = R.Report()
    for counters in (True, False):
        a, b = _colsum(v, counters), _colsum(v, counters)
        assert torch.equal(_bits(a), _bits(b)), 'colsum: two calls differ'
        R.check_colsum('colsum', a, v, R.colsum_n(M, counters), rep)
    print(f'[rowwise-edges] colsum {M}x{N}: {rep}')


def _gcc(src, in_row, scale, rows, unscaled):
    """vt_gather_cast_colsum_bf16; src fp32 [Rs, D] (CPU) 16 bytes into the rows of a NaN-filled [Rs + PAD, D + 8] buffer,
    rows no in_row entry names NaN -> (bf16 rows, sums [1 or 2, D])"""
    lib_, lib = _lib()
    Rs, D = src.shape
    named = torch.zeros(Rs, dtype=torch.bool)
    named[in_row.long()[in_row >= 0]] = True
    buf = _nan_rows(Rs, D + 8)
    buf[:Rs, 4:4 + D] = torch.where(named[:, None], src, torch.full_like(src, NAN)).cuda()
    nsum = 2 if unscaled else 1
    dst, cs = Guarded(rows, D, torch.bfloat16), Guarded(nsum, D, torch.float32)
    nb = lib.vt_gather_cast_colsum_blocks(rows)
    ws = torch.full((nb, nsum * D), NAN, device='cuda')
    ir, sc = in_row.cuda(), scale.cuda()
    p = lib_.GatherCastColsumParams()
    p.src, p.lds, p.in_row, p.row_scale = buf.data_ptr() + 16, D + 8, ir.data_ptr(), sc.data_ptr()
    p.dst, p.rows, p.D = dst.inner.data_ptr(), rows, D
    p.colsum, p.workspace, p.workspace_rows, p.unscaled_sums = cs.inner.data_ptr(), ws.data_ptr(), nb, int(unscaled)
    _call('vt_gather_cast_colsum_bf16', p, 'vt_gather_cast_colsum_bf16')
    dst.check('dst')
    cs.check('colsum')
    return dst.inner.view(rows, D).cpu(), cs.inner.view(nsum, D).cpu()


@pytest.mark.parametrize('rows,D', [(1, 8), (7, 1000), (4225, 64), (12544, 768), (12608, 1024), (3000, 1000), (12552, 8)])
def test_gather_cast_colsum_against_fp64(rows, D):
    g = torch.Generator().manual_seed(rows + D)
    src = torch.randn(rows + 50, D, generator=g)
    in_row = torch.randint(-1, rows + 50, (rows,), generator=g, dtype=torch.int32)
    keep = 0.9
    scale = (torch.rand(rows, generator=g) < keep).float() / keep          # DropPath: 0 (dropped row) or 1 / keep
    gathered = torch.where((in_row >= 0)[:, None], src[in_row.long().clamp(min=0)], torch.zeros(1))
    ref = (scale[:, None] * gathered).bfloat16()
    _, _, n = R.gcc_plan(rows, _sm())
    rep = R.Report()
    for unscaled in (False, True):
        out, cs = _gcc(src, in_row, scale, rows, unscaled)
        out2, cs2 = _gcc(src, in_row, scale, rows, unscaled)
        assert torch.equal(_bits(out), _bits(ref)), 'dst: not bf16(row_scale * x)'
        assert torch.equal(_bits(out2), _bits(out)) and torch.equal(_bits(cs2), _bits(cs)), 'two calls differ'
        R.check_colsum('colsum', cs[0], out, n, rep)
        if unscaled:
            R.check_colsum('colsum_unscaled', cs[1], gathered.bfloat16(), n, rep)
    print(f'[rowwise-edges] gather_cast_colsum {rows}x{D}: {rep}')


@pytest.mark.parametrize('M,N', [(1, 256), (3, 8192), (777, 1536), (12552, 3072), (12544, 768)])
def test_dgelu_colsum_against_fp64(M, N):
    """dz bits of the stand-alone dGELU kernel, column sums within bound of the fp64 sums of the kernel's own dz rows"""
    lib_, lib = _lib()
    from videotransformer_pytorch_b200 import _lib as L
    g = torch.Generator().manual_seed(M + N)
    dh = torch.randn(M, N, generator=g).bfloat16()
    z = (2 * torch.randn(M, N, generator=g)).bfloat16()
    bufs = []
    for t in (dh, z):
        b = _nan_rows(M, N, torch.bfloat16)
        b[:M] = t.cuda()
        bufs.append(b)
    ref = L.K.dgelu(dh.cuda(), z.cuda()).cpu()
    _, _, n = R.gbc_plan(M, _sm())
    rep = R.Report()
    res = []
    for _ in range(2):
        out, cs = Guarded(M, N, torch.bfloat16), Guarded(1, N, torch.float32)
        nb = lib.vt_gelu_bwd_colsum_blocks(M)
        ws = torch.full((nb, N), NAN, device='cuda')
        p = lib_.GeluBwdColsumParams()
        p.z, p.dh, p.out, p.M, p.N = bufs[1].data_ptr(), bufs[0].data_ptr(), out.inner.data_ptr(), M, N
        p.colsum, p.workspace, p.workspace_rows = cs.inner.data_ptr(), ws.data_ptr(), nb
        _call('vt_gelu_bwd_colsum_bf16', p, 'vt_gelu_bwd_colsum_bf16')
        out.check('dz')
        cs.check('colsum')
        res.append((out.inner.view(M, N).cpu(), cs.inner.cpu()))
    assert torch.equal(_bits(res[0][0]), _bits(ref)), 'dz: not the stand-alone dGELU bits'
    assert torch.equal(_bits(res[0][1]), _bits(res[1][1])), 'colsum: two calls differ'
    R.check_colsum('colsum', res[0][1], res[0][0], n, rep)
    print(f'[rowwise-edges] dgelu_colsum {M}x{N}: {rep}')


@pytest.mark.parametrize('S,n,stride', [(296, 768, 768), (33, 8, 8), (592, 3072, 3072), (1000, 4, 12), (5, 256, 256), (31, 192, 384)])
def test_reduce_rows_against_fp64(S, n, stride):
    g = torch.Generator().manual_seed(S + n)
    src = torch.full((S, stride), NAN)
    src[:, :n] = torch.randn(S, n, generator=g)
    prior = torch.randn(n, generator=g)
    rep = R.Report()
    for accumulate in (0, 1):
        out = Guarded(1, n, torch.float32)
        if accumulate:
            out.inner.copy_(prior.cuda())
        _reduce(src.cuda(), S, n, out.inner, accumulate, 0.5, stride)
        out.check('reduce')
        ref, bound = R.reduce_rows_ref(src, n, 0.5, prior if accumulate else None)
        R.check('reduce', out.inner.cpu(), ref, bound, rep)
    print(f'[rowwise-edges] reduce_rows S={S} n={n}: {rep}')


@pytest.mark.parametrize('B,T,D,S', [(8, 8, 768, 1569), (3, 4, 128, 37), (1, 2, 32, 9)])
def test_cls_rows_against_fp64(B, T, D, S):
    """the copy bit for bit; cls + mean over the T replicas within gamma_T; no other row of the stream written"""
    from videotransformer_pytorch_b200 import _lib as L
    g = torch.Generator().manual_seed(B * T + D)
    x = torch.randn(B, S, D, generator=g)
    extra = torch.randn(B, T, D, generator=g)
    rep = R.Report()
    for ex in (None, extra):
        y = torch.full((B, S + 1, D), NAN, device='cuda')[:, :S]        # the row after each sample's last row is NaN too
        L.K.cls_rows(y[:, 0], x[:, 0].cuda(), extra=None if ex is None else ex.cuda(), scale=1.0 / T)
        yc = y.cpu()
        assert bool(torch.isnan(yc[:, 1:]).all()), 'cls_rows: a row other than the cls row was written'
        ref, bound = R.cls_rows_ref(x[:, 0], ex, 1.0 / T)
        if ex is None:
            assert torch.equal(_bits(yc[:, 0]), _bits(x[:, 0])), 'cls_rows: the copy is not exact'
        else:
            R.check('cls_rows', yc[:, 0], ref, bound, rep)
    print(f'[rowwise-edges] cls_rows B={B} T={T} D={D}: {rep}')


# ---- the temporal block's fused column sums against the separate kernels --------------------------------------------
def test_temporal_block_fused_column_sums_agree_with_separate_kernels(monkeypatch):
    """TemporalAttnFn.backward with DropPath on: d_fc_b and v (the column sums of the scaled rows) from the fused producer
    (gather_cast_colsum with unscaled_sums) lie within the two kernels' column-sum bounds of those of gather_cast + colsum
    run on the same arguments, over the same bf16 rows"""
    from videotransformer_pytorch_b200 import _lib as L
    from videotransformer_pytorch_b200.transformer import DividedTemporalAttentionWithPreNorm, DropPath
    torch.manual_seed(0)
    D, H, T, B, P = 768, 12, 8, 2, 196
    blk = DividedTemporalAttentionWithPreNorm(D, H, T, False, layer_drop=dict(type=DropPath, dropout_p=0.3)).cuda().train()
    with torch.no_grad():
        blk.temporal_fc.weight.normal_(std=0.02)
    x = torch.randn(B, 1 + P * T, D, device='cuda', requires_grad=True)
    y = blk(x)
    dy = torch.randn_like(y)
    Kc = type(L.K)
    seen = []
    orig = Kc.gather_cast_colsum

    def spy(self, *a, **kw):
        out = orig(self, *a, **kw)
        seen.append((a, kw, out))
        return out
    monkeypatch.setattr(Kc, 'gather_cast_colsum', spy)
    grads = torch.autograd.grad(y, [blk.temporal_fc.bias], dy)
    (a, kw, (gs, v, dfb)), = [s for s in seen if s[1].get('unscaled_sums')]
    f = dict(gs=gs, v=v, d_fc_b=dfb)
    assert torch.equal(grads[0], f['d_fc_b'])
    # the separate kernels on the fused call's arguments: the scaled rows and their sums, the unscaled rows and theirs
    gs_s = L.K.gather_cast(a[0], in_row=kw['in_row'], row_scale=kw['row_scale'], rows=kw['rows'])
    unscaled = L.K.gather_cast(a[0], in_row=kw['in_row'], rows=kw['rows'])
    s = dict(gs=gs_s, v=L.K.colsum(gs_s), d_fc_b=L.K.colsum(unscaled), unscaled=unscaled)
    assert torch.equal(_bits(f['gs']), _bits(s['gs'])), 'the fused and separate producers give other bf16 rows'
    Mt = B * P * T
    nf, ns = R.gcc_plan(Mt, _sm())[2], R.colsum_n(Mt)
    rep = R.Report()
    for name, rows in (('v', s['gs']), ('d_fc_b', s['unscaled'])):
        a = rows.double().abs().sum(0).cpu()
        R.check(name, f[name].cpu(), s[name].double().cpu(), (R.gamma(nf) + R.gamma(ns)) * a, rep)
    print(f'[rowwise-edges] temporal block fused vs separate column sums: {rep}')


# ---- refusals before any launch --------------------------------------------------------------------------------------
def _refused(fn, p, match):
    lib_, lib = _lib()
    launches = lib.vt_launch_count()
    with pytest.raises(RuntimeError, match=match):
        _call(fn, p, fn)
    assert lib.vt_launch_count() == launches, f'{fn}: launched before refusing'


def _sentinel(n, dtype=torch.float32):
    return torch.full((n,), SENTINEL, dtype=dtype, device='cuda')


def _untouched(t):
    torch.cuda.synchronize()
    assert bool((t == SENTINEL).all()), 'an output was written before the refusal'


@pytest.mark.parametrize('what', ['src', 'dst'])
def test_cast_refuses_misaligned_pointers(what):
    lib_, _ = _lib()
    src = torch.randn(1001, device='cuda')
    dst = _sentinel(1008, torch.bfloat16)
    p = lib_.CastParams()
    p.src = src.data_ptr() + (4 if what == 'src' else 0)
    p.dst = dst.data_ptr() + (2 if what == 'dst' else 0)
    p.n = 1000
    _refused('vt_cast_f32_bf16', p, '16-byte aligned')
    _untouched(dst)


def test_cast_bf16_refuses_a_misaligned_view():
    from videotransformer_pytorch_b200 import _lib as L
    with pytest.raises(RuntimeError, match='16-byte aligned'):
        L.K.cast_bf16(torch.empty(1001, device='cuda')[1:])


def _ln_bwd_params(D=256, rows=64):
    lib_, lib = _lib()
    keep = dict(dy=torch.randn(rows, D, device='cuda'), x=torch.randn(rows + 1, D + 4, device='cuda'),
                stats=torch.ones(2, rows, device='cuda'), gam=torch.ones(D, device='cuda'),
                dres=torch.randn(rows + 1, D + 4, device='cuda'), dx=_sentinel((rows + 1) * (D + 4)),
                aux=_sentinel(D + 4), partials=_sentinel(lib.vt_ln_bwd_blocks(rows) * 2 * D + 4))
    p = lib_.LnBwdParams()
    p.dy, p.dy_fp32, p.x, p.ldx = keep['dy'].data_ptr(), 1, keep['x'].data_ptr(), D + 4
    p.mean, p.rstd, p.gamma = keep['stats'][0].data_ptr(), keep['stats'][1].data_ptr(), keep['gam'].data_ptr()
    p.dres, p.dx, p.lddx = keep['dres'].data_ptr(), keep['dx'].data_ptr(), D + 4
    p.partials, p.rows, p.D = keep['partials'].data_ptr(), rows, D
    return p, keep


@pytest.mark.parametrize('what', ['ldx', 'lddx', 'x', 'dy', 'dx', 'dres', 'dx_aux', 'partials'])
def test_layernorm_backward_refuses_misaligned_operands(what):
    p, keep = _ln_bwd_params()
    if what in ('ldx', 'lddx'):
        setattr(p, what, getattr(p, what) + 2)
    elif what == 'dx_aux':
        p.dx_aux = keep['aux'].data_ptr() + 8
    else:
        setattr(p, what, getattr(p, what) + 8)
    _refused('vt_layernorm_bwd', p, 'multiples of 4' if what.startswith('ld') else 'aligned')
    for n in ('dx', 'aux', 'partials'):
        _untouched(keep[n])


def test_layernorm_backward_refuses_bf16_dy_off_8_bytes():
    p, keep = _ln_bwd_params()
    dyb = torch.zeros(64 * 256 + 8, dtype=torch.bfloat16, device='cuda')
    p.dy, p.dy_fp32 = dyb.data_ptr() + 4, 0
    _refused('vt_layernorm_bwd', p, 'aligned')
    _untouched(keep['dx'])


@pytest.mark.parametrize('what', ['x', 'y'])
def test_layernorm_forward_refuses_a_misaligned_base(what):
    lib_, _ = _lib()
    D, rows = 256, 16
    x = torch.randn(rows + 1, D, device='cuda')
    y = _sentinel(rows * D + 8)
    gb = torch.ones(2, D, device='cuda')
    p = lib_.LnFwdParams()
    p.x, p.ldx = x.data_ptr() + (4 if what == 'x' else 0), D
    p.gamma, p.beta, p.y = gb[0].data_ptr(), gb[1].data_ptr(), y.data_ptr() + (4 if what == 'y' else 0)
    p.rows, p.D, p.eps, p.y_fp32 = rows, D, 1e-5, 1
    _refused('vt_layernorm_fwd', p, 'aligned')
    _untouched(y)


@pytest.mark.parametrize('fn', ['vt_gather_cast_bf16', 'vt_gather_cast_colsum_bf16'])
@pytest.mark.parametrize('what', ['src', 'dst'])
def test_gather_cast_refuses_misaligned_pointers(fn, what):
    lib_, lib = _lib()
    rows, D = 32, 64
    src = torch.randn(rows + 1, D, device='cuda')
    dst = _sentinel(rows * D + 8, torch.bfloat16)
    cs = _sentinel(D)
    ws = _sentinel(lib.vt_gather_cast_colsum_blocks(rows) * D)
    p = lib_.GatherCastColsumParams() if 'colsum' in fn else lib_.GatherCastParams()
    p.src, p.lds = src.data_ptr() + (4 if what == 'src' else 0), D
    p.dst, p.rows, p.D = dst.data_ptr() + (8 if what == 'dst' else 0), rows, D
    if 'colsum' in fn:
        p.colsum, p.workspace, p.workspace_rows = cs.data_ptr(), ws.data_ptr(), lib.vt_gather_cast_colsum_blocks(rows)
    _refused(fn, p, '16-byte aligned')
    for t in (dst, cs, ws):
        _untouched(t)


def test_ln_bwd_refuses_non_contiguous_or_wrong_dtype_dy():
    from videotransformer_pytorch_b200 import _lib as L
    D, rows = 256, 64
    x = torch.randn(rows, D, device='cuda')
    gam, bet = torch.ones(D, device='cuda'), torch.zeros(D, device='cuda')
    _, mean, rstd = L.K.ln_fwd(x, gam, bet, 1e-5)
    dx = torch.full((rows, D), SENTINEL, device='cuda')
    for dy, match in ((torch.randn(D, rows, device='cuda').t(), 'contiguous'), (torch.randn(rows, D, device='cuda').half(), 'dtype'),
                      (torch.randn(rows, 2 * D, device='cuda')[:, ::2], 'contiguous')):
        with pytest.raises(RuntimeError, match=match):
            L.K.ln_bwd(dy, x, mean, rstd, gam, dx=dx)
    with pytest.raises(RuntimeError, match='pitch'):
        L.K.ln_bwd(torch.randn(rows, D, device='cuda'), x, mean, rstd, gam, dx=dx,
                   dres=torch.randn(rows, 2 * D, device='cuda')[:, :D])
    _untouched(dx)
