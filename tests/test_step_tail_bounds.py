"""The bounds of tests/step_tail_ref.py on the CPU: an fp32 model of each kernel at the end of the step, summing in the
kernel's own order, sits inside every bound at the shapes and regimes of tests/test_gpu_step_tail_edges.py, and the
checkers reject planted defects of the kinds these kernels could have.  No GPU needed."""
import pytest
import torch

from tests import step_tail_ref as S

F32 = torch.float32


def fma(a, b, c):
    """fp32 fma: the product is exact in fp64, the sum rounds once to fp64 and once to fp32 (within the same bound)"""
    return (a.double() * b.double() + c.double()).float()


def _tree(v):
    """lane 0's value after the 5-level xor shuffle tree over the last dimension (32 lanes)"""
    while v.shape[-1] > 1:
        h = v.shape[-1] // 2
        v = v[..., :h] + v[..., h:]
    return v[..., 0]


def _seq(v, dim):
    """v summed in index order along dim, fp32, starting from 0"""
    acc = torch.zeros_like(v.select(dim, 0))
    for i in range(v.shape[dim]):
        acc = acc + v.select(dim, i)
    return acc


# ---- fp32 models of the kernels -----------------------------------------------------------------------------------------
def ls_fwd_model(x, w, b, drop_tail=False, bias_twice=False):
    M, K = x.shape
    N, G = w.shape[0], K // 4
    xg, wg = x.view(M, G, 4), w.view(N, G, 4)
    acc = torch.zeros(M, N, 32)
    for s in range(S.cdiv(G, 32)):
        g = torch.arange(s * 32, s * 32 + 32)
        ok = g < (G - 1 if drop_tail else G)
        gi = g.clamp_max(G - 1)
        xs = torch.where(ok[None, :, None], xg[:, gi], 0.0)
        ws = torch.where(ok[None, :, None], wg[:, gi], 0.0)
        for c in (3, 2, 1, 0):
            acc = fma(xs[:, None, :, c], ws[None, :, :, c], acc)
    y = _tree(acc)
    if b is not None:
        y = y + b
        if bias_twice:
            y = y + b
    return y


def ls_wgrad_model(dy, x, swap_cols=False):
    M, K = x.shape
    acc = torch.zeros(dy.shape[1], K)
    db = torch.zeros(dy.shape[1])
    for m in range(M):
        acc = fma(dy[m][:, None], x[m][None, :], acc)
        db = db + dy[m]
    if swap_cols and K > 1:
        acc[:, [0, K - 1]] = acc[:, [K - 1, 0]]
    return acc, db


def ls_dgrad_model(dy, w, drop_row=False):
    M, N = dy.shape
    K = w.shape[1]
    acc = torch.zeros(M, 8, K)
    for j in range(S.cdiv(N, 8)):
        n = torch.arange(j * 8, j * 8 + 8)
        ok = n < N
        ni = n.clamp_max(N - 1)
        acc = fma(torch.where(ok[None, :], dy[:, ni], 0.0)[:, :, None], torch.where(ok[:, None], w[ni], 0.0)[None], acc)
    dx = _seq(acc, 1)
    if drop_row:
        dx[-1] = 0
    return dx


def _block_sum(v):
    """the kernel's row sum of v [M, N]: thread c sums columns c, c + 256, ... in order, a shuffle tree per warp, then the
    8 warp partials in order"""
    M, N = v.shape
    steps = S.cdiv(N, 256)
    p = torch.cat([v, v.new_zeros(M, steps * 256 - N)], 1).view(M, steps, 256)
    per_thread = _seq(p, 1).view(M, 8, 32)
    return _seq(_tree(per_thread), 1)


def ce_model(z, t, old_form=False, swap_cols=False, drop_row=False):
    """fp32 softmax_ce -> (loss, dz, row); old_form: the parent's row loss (mx + log se) ts - sum t z, without skipping t = 0"""
    M, N = z.shape
    mx = z.max(1, keepdim=True).values
    d = z - mx
    e = torch.exp(d)
    se = _block_sum(e)
    ts = _block_sum(t)
    if old_form:
        tz = _block_sum_fma(t, z, skip_zero=False)
    else:
        tz = _block_sum_fma(t, d, skip_zero=True)
    inv_m = torch.tensor(1.0, dtype=F32) / torch.tensor(float(M), dtype=F32)
    dz = (e * (1 / se)[:, None] * ts[:, None] - t) * inv_m
    row = (mx[:, 0] + torch.log(se)) * ts - tz if old_form else torch.log(se) * ts - tz
    if swap_cols and N > 1:
        dz[:, [0, N - 1]] = dz[:, [N - 1, 0]]
    if drop_row:
        row[-1] = 0
    total = torch.zeros((), dtype=F32)
    for m in range(M):
        total = total + row[m]
    return total * inv_m, dz, row


def _block_sum_fma(t, v, skip_zero):
    M, N = t.shape
    steps = S.cdiv(N, 256)
    pad = lambda a: torch.cat([a, a.new_zeros(M, steps * 256 - N)], 1).view(M, steps, 256)
    tp, vp = pad(t), pad(v)
    acc = torch.zeros(M, 256)
    for s in range(steps):
        nxt = fma(tp[:, s], vp[:, s], acc)
        acc = torch.where(tp[:, s] != 0, nxt, acc) if skip_zero else nxt
    return _seq(_tree(acc.view(M, 8, 32)), 1)


def norm2_model(g, aligned, drop_last_chunk=False):
    parts = []
    for off in range(0, g.numel(), S.CHUNK):
        c = g[off:off + S.CHUNK]
        L = c.numel()
        if aligned:
            n4 = L >> 2
            steps = max(1, S.cdiv(n4, 256))
            q = torch.cat([c[:n4 * 4], c.new_zeros(steps * 1024 - n4 * 4)]).view(steps, 256, 4)
            per = _seq((q[..., 0] * q[..., 0] + q[..., 1] * q[..., 1]) + (q[..., 2] * q[..., 2] + q[..., 3] * q[..., 3]), 0)
            tail = c[n4 * 4:]
            per[:tail.numel()] = per[:tail.numel()] + tail * tail
        else:
            steps = S.cdiv(L, 256)
            q = torch.cat([c, c.new_zeros(steps * 256 - L)]).view(steps, 256)
            per = _seq(q * q, 0)
        parts.append(_seq(_tree(per.view(8, 32)).view(8, 1), 0)[0])
    if drop_last_chunk and len(parts) > 1:
        parts = parts[:-1]
    return _seq(torch.stack(parts).view(-1, 1), 0)[0]


def coef32(n2, clip):
    if clip <= 0:
        return torch.tensor(1.0)
    c = torch.tensor(clip, dtype=F32) / (torch.sqrt(n2) + torch.tensor(S.CLIP_EPS, dtype=F32))
    return torch.clamp(c, max=1.0)


def sgd_model(w, g, buf, coef, lr, wd, mom, nesterov, first, momentum_on_first=False):
    lr, wd, mom = (torch.tensor(v, dtype=F32) for v in (lr, wd, mom))
    d = fma(wd.expand_as(w), w, g * coef)
    b = d if first and not momentum_on_first else fma(mom.expand_as(buf), buf, d)
    dn = fma(mom.expand_as(b), b, d) if nesterov else b
    return fma((-lr).expand_as(dn), dn, w), b


def adamw_model(w, g, m, v, coef, lr, wd, b1, b2, eps, bc1, bc2):
    lr, wd, b1, b2, eps, bc1, bc2 = (torch.tensor(x, dtype=F32) for x in (lr, wd, b1, b2, eps, bc1, bc2))
    gi = g * coef
    w1 = w * (1 - lr * wd)
    mi = fma(b1.expand_as(m), m, (1 - b1) * gi)
    vi = fma(b2.expand_as(v), v, (1 - b2) * gi * gi)
    p = w1 - (lr / bc1) * mi / (torch.sqrt(vi) * torch.rsqrt(bc2) + eps)
    return p, mi, vi


# ---- linear_small ---------------------------------------------------------------------------------------------------------
def _check_ls(M, N, K, exact, seed, fwd=None, wgrad=None, dgrad=None, report=None):
    x, w, b, dy = S.ls_inputs(M, N, K, exact, seed)
    report = S.Report() if report is None else report
    for bias in (b, None):
        ref, bd = S.linear_fwd_ref(x, w, bias)
        S.check('fwd', (fwd or ls_fwd_model)(x, w, bias), ref, 0 * bd if exact else bd, report)
    dw_ref, dwb, db_ref, dbb = S.linear_wgrad_ref(dy, x)
    dw, db = (wgrad or ls_wgrad_model)(dy, x)
    S.check('dw', dw, dw_ref, 0 * dwb if exact else dwb, report)
    S.check('db', db, db_ref, 0 * dbb if exact else dbb, report)
    dx_ref, dxb = S.linear_dgrad_ref(dy, w)
    S.check('dx', (dgrad or ls_dgrad_model)(dy, w), dx_ref, 0 * dxb if exact else dxb, report)
    return report


@pytest.mark.parametrize('exact', [True, False])
@pytest.mark.parametrize('M,N,K', S.LS_TRIPLES)
def test_linear_small_model_within_bounds(M, N, K, exact):
    _check_ls(M, N, K, exact, seed=M * 7 + N * 3 + K)


@pytest.mark.parametrize('defect', ['k_tail', 'bias_twice', 'swap_dw_cols', 'drop_dx_row'])
def test_linear_small_checker_rejects(defect):
    M, N, K = 9, 8, 132
    kw = dict(k_tail=dict(fwd=lambda x, w, b: ls_fwd_model(x, w, b, drop_tail=True)),
              bias_twice=dict(fwd=lambda x, w, b: ls_fwd_model(x, w, b, bias_twice=True)),
              swap_dw_cols=dict(wgrad=lambda dy, x: ls_wgrad_model(dy, x, swap_cols=True)),
              drop_dx_row=dict(dgrad=lambda dy, w: ls_dgrad_model(dy, w, drop_row=True)))[defect]
    for exact in (True, False):
        with pytest.raises(AssertionError):
            _check_ls(M, N, K, exact, seed=1, **kw)


# ---- softmax_ce ---------------------------------------------------------------------------------------------------------
def _check_ce(M, N, regime, soft, model=ce_model):
    z, _, t = S.ce_inputs(M, N, regime, soft, seed=M + N)
    r = S.softmax_ce_ref(z, t)
    loss, dz, row = model(z, t)
    rep = S.Report()
    S.check('dlogits', dz, r['dz'], r['dz_bound'], rep)
    S.check('row_loss', row, r['row'], r['row_bound'], rep)
    S.check('loss', loss, r['loss'], r['loss_bound'], rep)
    return rep


def _ce_cases():
    for M in S.CE_M:
        for N in S.CE_N:
            for regime in S.CE_REGIMES:
                for soft in (False, True):
                    if (regime == 'neg_inf' and soft) or (regime == 'unnormalised' and not soft):
                        continue
                    yield M, N, regime, soft


@pytest.mark.parametrize('M', S.CE_M)
def test_softmax_ce_model_within_bounds(M):
    for _, N, regime, soft in (c for c in _ce_cases() if c[0] == M):
        _check_ce(M, N, regime, soft)


@pytest.mark.parametrize('defect,regime', [('old_loss_form', 'offset_up'), ('old_loss_form', 'neg_inf'),
                                           ('swap_cols', 'randn'), ('drop_row', 'randn')])
def test_softmax_ce_checker_rejects(defect, regime):
    model = dict(old_loss_form=lambda z, t: ce_model(z, t, old_form=True),
                 swap_cols=lambda z, t: ce_model(z, t, swap_cols=True),
                 drop_row=lambda z, t: ce_model(z, t, drop_row=True))[defect]
    with pytest.raises(AssertionError):
        _check_ce(8, 400, regime, False, model=model)


def test_softmax_ce_reference_is_torch_cross_entropy():
    """the fp64 reference is F.cross_entropy for hard labels, a -inf logit off the label included"""
    import torch.nn.functional as F
    for regime in ('randn', 'neg_inf', 'dominant'):
        z, labels, t = S.ce_inputs(8, 257, regime, False, seed=3)
        r = S.softmax_ce_ref(z, t)
        want = F.cross_entropy(z.double(), labels, reduction='none')
        assert torch.allclose(r['row'], want, rtol=1e-12, atol=1e-12)
        zg = z.double().requires_grad_(True)
        F.cross_entropy(zg, labels).backward()
        assert torch.allclose(r['dz'], zg.grad, rtol=1e-12, atol=1e-15)


# ---- top-k ---------------------------------------------------------------------------------------------------------------
def test_topk_twin_rejects_a_tie_ranked_the_wrong_way():
    """with the label tied with other classes, ranking ties ahead of the label changes the count"""
    C, V = 400, 3
    z = torch.randn(2 * V, C, generator=torch.Generator().manual_seed(0))
    labels = torch.tensor([5, 9])
    a, b = z[:V], z[V:]                # the view rows of clip 0 and clip 1
    a[:, 5] += 100
    a[:, 17] = a[:, 5]                 # clip 0: the label tied with one other class
    a[:, 6] = a[:, 5] + 50             # ... and one class above: rank 1
    b[:, 9] += 100                     # clip 1: the label on top, tied with five others: rank 0
    b[:, 30:35] = b[:, 9:10]
    ks = (1, 2, 5)
    good, _ = S.topk_twin(z, labels, V, ks)
    bad, _ = S.topk_twin(z, labels, V, ks, strict=False)
    assert good == [1, 2, 2] and bad != good


# ---- fused optimizer -----------------------------------------------------------------------------------------------------
def _opt_case(seed=0):
    shapes = S.opt_shapes()
    grads = S.opt_grads(shapes, seed)
    gen = torch.Generator().manual_seed(seed + 1)
    params = [torch.randn(g.numel(), generator=gen) for g in grads]
    state = [0.1 * torch.randn(g.numel(), generator=gen) for g in grads]
    state2 = [0.01 * torch.rand(g.numel(), generator=gen) for g in grads]
    return shapes, grads, params, state, state2


def _norm2_check(grads, model=norm2_model, report=None):
    report = S.Report() if report is None else report
    out = []
    for i, g in enumerate(grads):
        n2 = model(g, S.opt_misalign(i) == 0)
        ref, bd = S.norm2_ref(g)
        S.check(f'norm2[{i}]', n2.view(1), ref.view(1), bd.view(1), report)
        out.append(n2)
    return out


def test_norm2_model_within_bounds():
    _, grads, _, _, _ = _opt_case()
    _norm2_check(grads)


def test_norm2_checker_rejects_a_dropped_last_chunk():
    _, grads, _, _, _ = _opt_case()
    big = [g for g in grads if g.numel() > 3 * S.CHUNK]
    with pytest.raises(AssertionError):
        _norm2_check(big, model=lambda g, a: norm2_model(g, a, drop_last_chunk=True))


def _sgd_check(nesterov, first, lr_shift=0, wd_shift=0, momentum_on_first=False, clip=S.OPT_CLIP):
    shapes, grads, params, state, _ = _opt_case()
    n2 = _norm2_check(grads)
    lrs, wds = S.opt_hyper(len(grads))
    rep = S.Report()
    for i, (w, g, buf) in enumerate(zip(params, grads, state)):
        j, k = (i + lr_shift) % len(grads), (i + wd_shift) % len(grads)
        p, b = sgd_model(w, g, buf, coef32(n2[i], clip), lrs[j], wds[k], S.f32(0.9), nesterov, first, momentum_on_first)
        pr, pb, br, bb = S.sgd_step_ref(w, g, buf, S.clip_coef_ref(n2[i], clip), lrs[i], wds[i], S.f32(0.9), nesterov, first)
        S.check('param', p, pr, pb, rep)
        S.check('momentum', b, br, bb, rep)
    return rep


@pytest.mark.parametrize('first', [True, False])
@pytest.mark.parametrize('nesterov', [True, False])
def test_sgd_model_within_bounds(nesterov, first):
    _sgd_check(nesterov, first)
    _sgd_check(nesterov, first, clip=0.0)


@pytest.mark.parametrize('defect', ['lr_wrong_tensor', 'wd_wrong_tensor', 'momentum_on_first_step'])
def test_sgd_checker_rejects(defect):
    kw = dict(lr_wrong_tensor=dict(lr_shift=1), wd_wrong_tensor=dict(wd_shift=1),
              momentum_on_first_step=dict(momentum_on_first=True))[defect]
    with pytest.raises(AssertionError):
        _sgd_check(True, True, **kw)


@pytest.mark.parametrize('step', [1, 1000])
def test_adamw_model_within_bounds(step):
    shapes, grads, params, m, v = _opt_case(seed=2)
    if step == 1:
        m, v = [torch.zeros_like(t) for t in m], [torch.zeros_like(t) for t in v]
    n2 = _norm2_check(grads)
    lrs, wds = S.opt_hyper(len(grads), lr=1e-3)
    b1, b2, eps = S.f32(0.9), S.f32(0.999), S.f32(1e-8)
    bc1, bc2 = S.f32(1 - 0.9 ** step), S.f32(1 - 0.999 ** step)
    rep = S.Report()
    for i in range(len(grads)):
        p, mi, vi = adamw_model(params[i], grads[i], m[i], v[i], coef32(n2[i], S.OPT_CLIP), lrs[i], wds[i], b1, b2, eps, bc1, bc2)
        pr, pb, mr, mb, vr, vb = S.adamw_step_ref(params[i], grads[i], m[i], v[i], S.clip_coef_ref(n2[i], S.OPT_CLIP),
                                                 lrs[i], wds[i], b1, b2, eps, bc1, bc2)
        S.check('param', p, pr, pb, rep)
        S.check('exp_avg', mi, mr, mb, rep)
        S.check('exp_avg_sq', vi, vr, vb, rep)


def test_adamw_checker_rejects_lr_on_the_wrong_tensor():
    shapes, grads, params, m, v = _opt_case(seed=2)
    lrs, wds = S.opt_hyper(len(grads), lr=1e-3)
    args = (S.f32(0.9), S.f32(0.999), S.f32(1e-8), S.f32(0.1), S.f32(0.001))
    with pytest.raises(AssertionError):
        for i in range(len(grads)):
            p, _, _ = adamw_model(params[i], grads[i], m[i], v[i], 1.0, lrs[(i + 1) % len(grads)], wds[i], *args)
            pr, pb, *_ = S.adamw_step_ref(params[i], grads[i], m[i], v[i], (1.0, 0.0), lrs[i], wds[i], *args)
            S.check('param', p, pr, pb, S.Report())
