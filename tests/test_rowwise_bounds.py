"""The bounds of tests/rowwise_ref.py on the CPU: an fp32 model of each row-wise kernel, summing in the kernel's own
partition of the rows, sits inside every bound at the widths, row counts and regimes of tests/test_gpu_rowwise_edges.py,
and the checker rejects seeded defects of the kinds the kernels could have.  No GPU needed."""
import pytest
import torch

from tests import rowwise_ref as R

SM = 132                       # SM count of an H100 SXM: fixes the CTA partition the fp32 model sums by
CAP = R.ln_cap(SM)
F32 = torch.float32


def _f32(v):
    return torch.tensor(v, dtype=F32)


def _seq(t):
    """t[0] + t[1] + ... in order, fp32"""
    acc = t[0].clone()
    for i in range(1, t.shape[0]):
        acc += t[i]
    return acc


def _interleaved(v, groups, lanes):
    """per-(group, lane) sums of v [M, N] fp32 when row m = k * groups * lanes + g * lanes + l is added by lane l of
    group g at its step k (one warp or thread per row, grid-strided), in step order -> [groups, lanes, N]"""
    M, N = v.shape
    steps = R.cdiv(M, groups * lanes)
    w = torch.cat([v, v.new_zeros(steps * groups * lanes - M, N)]).view(steps, groups, lanes, N)
    return _seq(w)


def ln_fwd_model(x, gam, bet, eps, var_div=None, eps_after_sqrt=False, toward_zero=False):
    """fp32 LayerNorm of the rows of x [rows, D] -> mean, rstd, y32, y (bf16)"""
    D = x.shape[1]
    mu = x.sum(1) * _f32(1.0 / D)
    d = x - mu[:, None]
    var = (d * d).sum(1) * _f32(1.0 / (var_div or D))
    rs = 1 / (var.sqrt() + _f32(eps)) if eps_after_sqrt else torch.rsqrt(var + _f32(eps))
    y32 = d * rs[:, None] * gam + bet
    y = (y32.view(torch.int32) & -65536).view(F32).bfloat16() if toward_zero else y32.bfloat16()
    return dict(mean=mu, rstd=rs, y32=y32, y=y)


def ln_bwd_model(x, mu, rs, gam, dy, out_row=None, dres=None, n_out=None, n_aux=0, skip_res=False, res_to_aux=False,
                 drop_cta=None, double_cta=None):
    """fp32 LayerNorm backward of the rows x [rows, D] (in_row applied) -> dx [n_out, D] (rows out_row does not reach: 0),
    dx_aux [n_aux, D], dgamma, dbeta with the per-warp / per-CTA partition of the kernels"""
    rows, D = x.shape
    d = dy.float()
    xh = (x - mu[:, None]) * rs[:, None]
    gy = d * gam
    inv = _f32(1.0 / D)
    m1, m2 = gy.sum(1, keepdim=True) * inv, (gy * xh).sum(1, keepdim=True) * inv
    o = rs[:, None] * (gy - m1 - xh * m2)
    t = torch.arange(rows) if out_row is None else out_row.long()
    dx = torch.zeros(n_out or rows, D)
    aux = torch.zeros(n_aux, D)
    pos = t >= 0
    add = o[pos]
    if dres is not None and not skip_res:
        add = add + dres[t[pos]]
    dx[t[pos]] = add
    a = o[~pos]
    if dres is not None and res_to_aux:
        a = a + dres[0]
    aux[-t[~pos] - 1] = a
    blocks, _ = R.ln_plan(rows, SM)
    gb = []
    for v in (d * xh, d):
        cta = _seq(_interleaved(v, blocks, R.ROW_WARPS).transpose(0, 1))
        if drop_cta is not None:
            cta[drop_cta] = 0
        tot = _seq(cta)
        gb.append(tot + cta[double_cta] if double_cta is not None else tot)
    return dx, aux, gb[0], gb[1]


def check_ln(x, in_row, gam, bet, eps, fwd, dy, bwd, out_row=None, dres=None, n_aux=0):
    """the checks of tests/test_gpu_rowwise_edges.py on model outputs"""
    rep = R.Report()
    xs = x.double()[in_row.long()] if in_row is not None else x.double()
    R.check_ln_forward(xs, fwd['mean'], fwd['rstd'], gam, bet, eps, fwd['y32'], rep, names=('mean', 'rstd', 'y32'))
    R.check_ln_forward(xs, fwd['mean'], fwd['rstd'], gam, bet, eps, fwd['y'], rep, names=('mean', 'rstd', 'y'))
    dx, aux, dg, db = bwd
    t = torch.arange(xs.shape[0]) if out_row is None else out_row.long()
    pos = t >= 0
    rows = torch.empty_like(xs)
    rows[pos] = dx[t[pos]].double()
    rows[~pos] = aux[-t[~pos] - 1].double()
    res = None
    if dres is not None:
        r = torch.zeros_like(xs)
        r[pos] = dres[t[pos]].double()
        res = (r, pos.double())
    d, xhat = R.check_ln_backward(xs, fwd['mean'], fwd['rstd'], gam, dy, rows, res, rep)
    R.check_dgamma_dbeta(d, xhat, dg, db, SM, rep)
    return rep


def _ln_case(D, rows, regime, eps, dy_dtype, seed):
    x = R.make_rows(rows, D, regime, seed)
    gam, bet = R.make_affine(D, seed + 1)
    dy = torch.randn(rows, D, generator=torch.Generator().manual_seed(seed + 2)).to(dy_dtype)
    dres = torch.randn(rows, D, generator=torch.Generator().manual_seed(seed + 3))
    return x, gam, bet, dy, dres


ROWS = [1, 7, 8, 9, 8 * CAP - 1, 8 * CAP, 8 * CAP + 1]
LN_CASES = [(D, rows, R.REGIMES[(i + j) % len(R.REGIMES)], (1e-5, 1e-6)[j % 2], (F32, torch.bfloat16)[(i + j) % 2])
            for i, D in enumerate(R.LN_WIDTHS + R.LN_SMALL_WIDTHS) for j, rows in enumerate(ROWS)]
MODEL_CASES = [(768, 12544, 'randn', 1e-5, torch.bfloat16), (768, 12608, 'offset', 1e-5, torch.bfloat16),
               (768, 12552, 'outlier', 1e-6, F32), (96, 200712, 'randn', 1e-6, torch.bfloat16),
               (192, 50184, 'tiny', 1e-6, torch.bfloat16), (384, 12552, 'constant', 1e-6, F32), (768, 3144, 'randn', 1e-6, F32)]


def _ln_id(c):
    D, rows, regime, eps, dt = c
    return f'D{D}-rows{rows}-{regime}-eps{eps:g}-dy{"fp32" if dt == F32 else "bf16"}'


@pytest.mark.parametrize('case', LN_CASES + MODEL_CASES, ids=_ln_id)
def test_layernorm_model_sits_inside_every_bound(case):
    D, rows, regime, eps, dt = case
    x, gam, bet, dy, dres = _ln_case(D, rows, regime, eps, dt, seed=D + rows)
    fwd = ln_fwd_model(x, gam, bet, eps)
    rep = check_ln(x, None, gam, bet, eps, fwd, dy, ln_bwd_model(x, fwd['mean'], fwd['rstd'], gam, dy, dres=dres), dres=dres)
    print(f'[rowwise-bounds] {_ln_id(case)}: {rep}')


def test_layernorm_model_with_spatial_maps_and_aux_rows():
    """the spatial backward's map: cls rows to dx_aux (no residual), patch rows scattered with the residual"""
    from videotransformer_pytorch_b200.ops import token_maps
    B, T, P, D = 2, 8, 196, 256
    maps = token_maps(B, T, P, 'cpu')
    S = 1 + P * T
    x, gam, bet, _, dres = _ln_case(D, B * S, 'randn', 1e-5, F32, seed=5)
    in_row, out_row = maps['sp_in'], maps['sp_bwd']
    dy = torch.randn(in_row.numel(), D).bfloat16()
    fwd = ln_fwd_model(x[in_row.long()], gam, bet, 1e-5)
    bwd = ln_bwd_model(x[in_row.long()], fwd['mean'], fwd['rstd'], gam, dy, out_row, dres, B * S, B * T)
    rep = check_ln(x, in_row, gam, bet, 1e-5, fwd, dy, bwd, out_row, dres, B * T)
    print(f'[rowwise-bounds] spatial maps: {rep}')


# ---- column sums, reduce_rows, cls_rows ----------------------------------------------------------------------------
def colsum_model(v):
    """fp32 column sums of v [M, N] (bf16 values) in the order of colsum_kernel"""
    M, N = v.shape
    v = v.float()
    rows = R.COLSUM_ROWS
    chunks = R.cdiv(M, rows)
    w = torch.cat([v, v.new_zeros(chunks * rows - M, N)]).view(chunks, rows // R.ROW_WARPS, R.ROW_WARPS, N)
    return _seq(_seq(_seq(w.transpose(0, 1)).transpose(0, 1)))      # lanes' rows in order, then the 8 lanes, then the chunks


def gcc_model(src, in_row, scale, unscaled=False, fp32_sums=False):
    """gather_cast_colsum: bf16 rows bf16(scale * src[in_row]) (0 where in_row < 0) and their column sums (with unscaled:
    also those of bf16(src[in_row])) in the kernel's partition"""
    rows = in_row.numel()
    g = src[in_row.long().clamp(min=0)] * (in_row >= 0)[:, None]
    scaled = (scale[:, None] * g)
    out = scaled.bfloat16()
    blocks, _, _ = R.gcc_plan(rows, SM)
    sums = []
    for v in ((scaled if fp32_sums else out.float()), g.bfloat16().float()):
        sums.append(_seq(_seq(_interleaved(v, blocks, R.ROW_WARPS).transpose(0, 1))))
    return out, (torch.stack(sums) if unscaled else sums[0])


def test_colsum_models_sit_inside_their_bounds():
    g = torch.Generator().manual_seed(3)
    rep = R.Report()
    for M, N in ((1, 8), (511, 96), (512, 100), (513, 768), (63, 64), (64, 72), (65, 256), (12544, 768), (12552, 3072)):
        v = torch.randn(M, N, generator=g).bfloat16()
        for counters in (True, False):
            R.check_colsum('colsum', colsum_model(v), v, R.colsum_n(M, counters), rep)
    print(f'[rowwise-bounds] colsum: {rep}')


@pytest.mark.parametrize('rows,D', [(1, 8), (700, 1000), (12544, 768), (12608, 1024), (4225, 64)])
def test_gather_cast_colsum_model_sits_inside_its_bound(rows, D):
    src, in_row, scale = _gcc_inputs(rows, D, seed=rows + D)
    out, sums = gcc_model(src, in_row, scale, unscaled=True)
    rep = R.Report()
    _, _, n = R.gcc_plan(rows, SM)
    R.check_colsum('colsum', sums[0], out, n, rep)
    R.check_colsum('colsum_unscaled', sums[1], _gathered(src, in_row).bfloat16(), n, rep)
    print(f'[rowwise-bounds] gather_cast_colsum {rows}x{D}: {rep}')


def _gcc_inputs(rows, D, seed, keep=0.9):
    g = torch.Generator().manual_seed(seed)
    src = torch.randn(rows + 50, D, generator=g)
    in_row = torch.randint(-1, rows + 50, (rows,), generator=g, dtype=torch.int32)
    scale = (torch.rand(rows, generator=g) < keep).float() / keep      # DropPath: 0 or 1 / keep
    return src, in_row, scale


def _gathered(src, in_row):
    return src[in_row.long().clamp(min=0)] * (in_row >= 0)[:, None]


def test_reduce_rows_and_cls_rows_inside_their_bounds():
    g = torch.Generator().manual_seed(4)
    rep = R.Report()
    for S, n in ((296, 768), (33, 8), (5, 256), (1000, 4)):
        inp = torch.randn(S, n, generator=g)
        prior = torch.randn(n, generator=g)
        ref, bound = R.reduce_rows_ref(inp, n, 0.5, prior)
        R.check('reduce', prior + _f32(0.5) * _seq(inp), ref, bound, rep)
    src, extra = torch.randn(8, 768, generator=g), torch.randn(8, 8, 768, generator=g)
    ref, bound = R.cls_rows_ref(src, extra, 1 / 8)
    R.check('cls_rows', torch.addcmul(src, _seq(extra.transpose(0, 1)), _f32(1 / 8)), ref, bound, rep)
    print(f'[rowwise-bounds] reduce_rows / cls_rows: {rep}')


# ---- seeded defects ------------------------------------------------------------------------------------------------
D0, ROWS0 = 768, 8 * CAP + 1          # past the CTA cap: warps walk two rows and accumulate dgamma / dbeta across them


def _ln_setup(regime='randn', scale=1.0):
    x, gam, bet, dy, dres = _ln_case(D0, ROWS0, regime, 1e-5, F32, seed=9)
    x = x * scale
    return x, gam, bet, dy, dres, ln_fwd_model(x, gam, bet, 1e-5)


def _rejects(name, *args, **kw):
    with pytest.raises(AssertionError, match=f'^{name}: '):
        check_ln(*args, **kw)


def test_clean_layernorm_passes():
    x, gam, bet, dy, dres, fwd = _ln_setup()
    check_ln(x, None, gam, bet, 1e-5, fwd, dy, ln_bwd_model(x, fwd['mean'], fwd['rstd'], gam, dy, dres=dres), dres=dres)


@pytest.mark.parametrize('defect', ['drop', 'double'])
def test_rejects_dgamma_cta_partial_missing_or_doubled(defect):
    x, gam, bet, dy, dres, fwd = _ln_setup()
    kw = {'drop_cta': CAP - 1} if defect == 'drop' else {'double_cta': 17}
    bwd = ln_bwd_model(x, fwd['mean'], fwd['rstd'], gam, dy, dres=dres, **kw)
    _rejects('dgamma', x, None, gam, bet, 1e-5, fwd, dy, bwd, dres=dres)


@pytest.mark.parametrize('defect', ['var_over_D_minus_1', 'eps_after_sqrt'])
def test_rejects_wrong_variance(defect):
    x, gam, bet, dy, dres, _ = _ln_setup(scale=3e-3)         # variance ~1e-5: eps matters
    fwd = ln_fwd_model(x, gam, bet, 1e-5, **({'var_div': D0 - 1} if defect == 'var_over_D_minus_1' else {'eps_after_sqrt': True}))
    _rejects('rstd', x, None, gam, bet, 1e-5, fwd, dy, ln_bwd_model(x, fwd['mean'], fwd['rstd'], gam, dy, dres=dres), dres=dres)


def test_rejects_y_rounded_toward_zero():
    x, gam, bet, dy, dres, fwd = _ln_setup()
    fwd['y'] = ln_fwd_model(x, gam, bet, 1e-5, toward_zero=True)['y']
    with pytest.raises(AssertionError, match='^y: '):
        rep = R.Report()
        R.check_ln_forward(x.double(), fwd['mean'], fwd['rstd'], gam, bet, 1e-5, fwd['y'], rep, names=('mean', 'rstd', 'y'))


@pytest.mark.parametrize('defect', ['skip_res', 'res_to_aux'])
def test_rejects_residual_missing_or_added_to_aux_rows(defect):
    from videotransformer_pytorch_b200.ops import token_maps
    B, T, P, D = 1, 4, 9, 128
    maps = token_maps(B, T, P, 'cpu')
    S = 1 + P * T
    x, gam, bet, _, dres = _ln_case(D, B * S, 'randn', 1e-5, F32, seed=6)
    in_row, out_row = maps['sp_in'], maps['sp_bwd']
    xs = x[in_row.long()]
    dy = torch.randn(in_row.numel(), D)
    fwd = ln_fwd_model(xs, gam, bet, 1e-5)
    bwd = ln_bwd_model(xs, fwd['mean'], fwd['rstd'], gam, dy, out_row, dres, B * S, B * T, **{defect: True})
    _rejects('dx', x, in_row, gam, bet, 1e-5, fwd, dy, bwd, out_row, dres, B * T)


def test_rejects_column_sums_of_the_fp32_values():
    src, in_row, scale = _gcc_inputs(12544, 768, seed=1)
    out, _ = gcc_model(src, in_row, scale)
    _, sums = gcc_model(src, in_row, scale, fp32_sums=True)
    with pytest.raises(AssertionError, match='^colsum: '):
        R.check_colsum('colsum', sums, out, R.gcc_plan(12544, SM)[2], R.Report())


def test_rejects_dual_sum_rows_swapped():
    src, in_row, scale = _gcc_inputs(4096, 256, seed=2, keep=0.5)
    out, sums = gcc_model(src, in_row, scale, unscaled=True)
    with pytest.raises(AssertionError, match='^colsum: '):
        R.check_colsum('colsum', sums[1], out, R.gcc_plan(4096, SM)[2], R.Report())


def test_rejects_cls_rows_mean_over_T_minus_1():
    g = torch.Generator().manual_seed(8)
    src, extra, T = torch.randn(4, 128, generator=g), torch.randn(4, 8, 128, generator=g), 8
    ref, bound = R.cls_rows_ref(src, extra, 1 / T)
    with pytest.raises(AssertionError, match='^cls_rows: '):
        R.check('cls_rows', src + extra.sum(1) / (T - 1), ref, bound, R.Report())
