"""The kernels at the end of every step element by element against fp64: the classification head's linear_small fwd /
wgrad / db / dgrad, softmax cross-entropy, the top-k counters and the fused clip + optimizer step.  -m gpu

Every output is checked per element against the bounds of tests/step_tail_ref.py (shown to hold for an fp32 model and to
reject planted defects in tests/test_step_tail_bounds.py); the top-k counts must equal the fp32 twin exactly.  The kernels
are driven through ctypes: inputs sit in buffers whose elements past the end are NaN, outputs start as NaN between NaN
guard rows (the guards must keep their bits), and the optimizer's tensors are views into flat buffers with NaN gaps
between them, some gradients 1, 2 or 3 floats off 16-byte alignment.  The worst error / bound ratios are printed
(STEP-TAIL-REPORT lines).
"""
import ctypes as C

import pytest
import torch
import torch.nn.functional as F

from tests import step_tail_ref as S
from tests.test_gpu_attention_edges import Guarded, _call, _lib

pytestmark = pytest.mark.gpu

PAD = 64                     # NaN elements past the end of every input
GAP = 13                     # NaN floats between two optimizer tensors
NAN = float('nan')
REPORT = S.Report()


def _report(rep, tag):
    for k, v in rep.items():
        REPORT.add(f'{tag} {k}', v)
    print('STEP-TAIL-REPORT ' + ', '.join(f'{k} {v:.3f}' for k, v in sorted(REPORT.items()) if k.startswith(tag)))


def _padded(t, shift=0):
    """t (CPU) copied to the device, `shift` floats into a NaN buffer with PAD NaN elements after it -> (buffer, address)"""
    flat = t.reshape(-1)
    buf = torch.full((flat.numel() + shift + PAD,), NAN, dtype=t.dtype, device='cuda')
    buf[shift:shift + flat.numel()] = flat.cuda()
    return buf, buf.data_ptr() + shift * t.element_size()


# ---- linear_small -------------------------------------------------------------------------------------------------------
def run_linear(x, w, b, dy, want_dw=True, want_db=True, want_dx=True, shift=None):
    """fwd and bwd through the C ABI -> dict of CPU outputs; shift = {'x' | 'w' | 'dw' | 'dx': floats} misaligns one operand"""
    shift = shift or {}
    M, K = x.shape
    N = w.shape[0]
    keep = []
    xb, xp = _padded(x, shift.get('x', 0))
    wb, wp = _padded(w, shift.get('w', 0))
    keep += [xb, wb]
    bp = None
    if b is not None:
        bb, bp = _padded(b)
        keep.append(bb)
    y = Guarded(M, N, torch.float32)
    p = _lib()[0].LinearSmallParams()
    p.x, p.w, p.b, p.y, p.M, p.N, p.K = xp, wp, bp, y.inner.data_ptr(), M, N, K
    _call('vt_linear_small_fwd', p, 'vt_linear_small_fwd')
    y.check('y')
    out = dict(y=y.inner.view(M, N).cpu())
    dyb, dyp = _padded(dy)
    dw = Guarded(N, K + shift.get('dw', 0), torch.float32) if want_dw else None
    db = Guarded(1, N, torch.float32) if want_db else None
    dx = Guarded(M, K + shift.get('dx', 0), torch.float32) if want_dx else None
    q = _lib()[0].LinearSmallBwdParams()
    q.dy, q.x, q.w = dyp, xp, wp
    q.dw = None if dw is None else dw.inner.data_ptr() + 4 * shift.get('dw', 0)
    q.db = None if db is None else db.inner.data_ptr()
    q.dx = None if dx is None else dx.inner.data_ptr() + 4 * shift.get('dx', 0)
    q.M, q.N, q.K = M, N, K
    _call('vt_linear_small_bwd', q, 'vt_linear_small_bwd')
    for name, g, rows, cols in (('dw', dw, N, K), ('db', db, 1, N), ('dx', dx, M, K)):
        if g is None:
            continue
        g.check(name)
        out[name] = g.inner.view(rows, cols).cpu() if name != 'db' else g.inner.cpu()
    return out


@pytest.mark.parametrize('exact', [True, False])
@pytest.mark.parametrize('M,N,K', S.LS_TRIPLES)
def test_linear_small_per_element(M, N, K, exact):
    x, w, b, dy = S.ls_inputs(M, N, K, exact, seed=M * 7 + N * 3 + K)
    rep = S.Report()
    exactly = (lambda bd: 0 * bd) if exact else (lambda bd: bd)
    for bias, skip in ((b, None), (None, 'dw'), (b, 'dx')):
        out = run_linear(x, w, bias, dy, want_dw=skip != 'dw', want_db=bias is not None and skip != 'dw',
                         want_dx=skip != 'dx')
        ref, bd = S.linear_fwd_ref(x, w, bias)
        S.check('fwd', out['y'], ref, exactly(bd), rep)
        dw_ref, dwb, db_ref, dbb = S.linear_wgrad_ref(dy, x)
        if 'dw' in out:
            S.check('dw', out['dw'], dw_ref, exactly(dwb), rep)
        if 'db' in out:
            S.check('db', out['db'], db_ref, exactly(dbb), rep)
        if 'dx' in out:
            dx_ref, dxb = S.linear_dgrad_ref(dy, w)
            S.check('dx', out['dx'], dx_ref, exactly(dxb), rep)
    _report(rep, 'linear_small exact' if exact else 'linear_small randn')


def test_linear_small_refusals():
    x, w, b, dy = S.ls_inputs(4097, 8, 128, True, seed=0)
    with pytest.raises(RuntimeError, match='not skinny'):
        run_linear(x, w, b, dy)
    x, w, b, dy = S.ls_inputs(8, 8, 130, True, seed=0)
    with pytest.raises(RuntimeError, match='bad shape'):
        run_linear(x, w, b, dy)
    x, w, b, dy = S.ls_inputs(8, 9, 128, True, seed=0)
    for name in ('x', 'w'):
        for s in (1, 2, 3):
            with pytest.raises(RuntimeError, match='vt_linear_small_fwd: x and w must be 16-byte aligned'):
                run_linear(x, w, b, dy, shift={name: s})
    for name in ('dw', 'dx'):
        with pytest.raises(RuntimeError, match='vt_linear_small_bwd: x, w, dw and dx must be 16-byte aligned'):
            run_linear(x, w, b, dy, shift={name: 1})


# ---- softmax_ce ---------------------------------------------------------------------------------------------------------
def run_ce(z, labels=None, t=None):
    M, N = z.shape
    zb, zp = _padded(z)
    keep = [zb]
    p = _lib()[0].SoftmaxCeParams()
    p.logits = zp
    if labels is not None:
        lb = labels.cuda()
        keep.append(lb)
        p.labels = lb.data_ptr()
    if t is not None:
        tb, tp = _padded(t)
        keep.append(tb)
        p.soft_targets = tp
    loss, row, dz = Guarded(1, 1, torch.float32), Guarded(M, 1, torch.float32), Guarded(M, N, torch.float32)
    p.loss, p.row_loss, p.dlogits, p.M, p.N = loss.inner.data_ptr(), row.inner.data_ptr(), dz.inner.data_ptr(), M, N
    _call('vt_softmax_ce', p, 'vt_softmax_ce')
    for g, n in ((loss, 'loss'), (row, 'row_loss'), (dz, 'dlogits')):
        g.check(n)
    return loss.inner.cpu()[0], dz.inner.view(M, N).cpu(), row.inner.cpu()


def _ce_cases():
    for M in S.CE_M:
        for N in S.CE_N:
            for regime in S.CE_REGIMES:
                for soft in (False, True):
                    if (regime == 'neg_inf' and soft) or (regime == 'unnormalised' and not soft):
                        continue
                    yield M, N, regime, soft


@pytest.mark.parametrize('M,N,regime,soft', list(_ce_cases()))
def test_softmax_ce_per_element(M, N, regime, soft):
    z, labels, t = S.ce_inputs(M, N, regime, soft, seed=M + N)
    loss, dz, row = run_ce(z, labels=None if soft else labels, t=t if soft else None)
    r = S.softmax_ce_ref(z, t)
    rep = S.Report()
    S.check('dlogits', dz, r['dz'], r['dz_bound'], rep)
    S.check('row_loss', row, r['row'], r['row_bound'], rep)
    # the loss against the mean of the fp64 row losses, and within summation error of the mean of the kernel's own rows
    S.check('loss', loss.view(1), r['loss'].view(1), r['loss_bound'].view(1), rep)
    own = row.double()
    S.check('loss vs rows', loss.view(1), own.mean().view(1), (S.gamma(M + 2) * own.abs().mean()).view(1), rep)
    _report(rep, 'softmax_ce')


def test_softmax_ce_neg_inf_logit_matches_torch():
    """hard labels with -inf logits off the label: F.cross_entropy's finite loss and gradient (0 * -inf once made NaN)"""
    z, labels, t = S.ce_inputs(8, 400, 'neg_inf', False, seed=5)
    loss, dz, row = run_ce(z, labels=labels)
    want = F.cross_entropy(z.double(), labels, reduction='none')
    zg = z.double().requires_grad_(True)
    F.cross_entropy(zg, labels).backward()
    r = S.softmax_ce_ref(z, t)
    rep = S.Report()
    S.check('row_loss', row, want, r['row_bound'], rep)
    S.check('loss', loss.view(1), want.mean().view(1), r['loss_bound'].view(1), rep)
    S.check('dlogits', dz, zg.grad, r['dz_bound'], rep)
    assert bool((dz[torch.isinf(z)] == 0).all())


def test_softmax_ce_refusals():
    z, labels, t = S.ce_inputs(4097, 7, 'randn', True, seed=0)
    with pytest.raises(RuntimeError, match='bad shape M=4097'):
        run_ce(z, labels=labels)
    z, labels, t = S.ce_inputs(8, 7, 'randn', True, seed=0)
    for kw in (dict(labels=labels, t=t), dict()):
        with pytest.raises(RuntimeError, match='exactly one'):
            run_ce(z, **kw)


# ---- topk_hits ----------------------------------------------------------------------------------------------------------
def run_topk(logits, labels, V, ks, counters=None, probs=True):
    """-> (hits list, samples, probs CPU | None, counters buffer); counters: the int64 buffer of an earlier call to add to"""
    BV, C_ = logits.shape
    B = labels.numel()
    lb, lp = _padded(logits)
    lab = labels.cuda()
    if counters is None:
        counters = torch.full((16,), -7, dtype=torch.int64, device='cuda')    # guards around hits [4, 8) and samples [8]
        counters[4:9] = 0
    pr = Guarded(B, C_, torch.float32) if probs else None
    p = _lib()[0].TopkHitsParams()
    p.logits, p.labels, p.probs = lp, lab.data_ptr(), None if pr is None else pr.inner.data_ptr()
    p.hits, p.samples = counters.data_ptr() + 4 * 8, counters.data_ptr() + 8 * 8
    p.B, p.V, p.C, p.n_k = B, V, C_, len(ks)
    for i, k in enumerate(ks):
        p.k[i] = k
    _call('vt_topk_hits', p, 'vt_topk_hits')
    torch.cuda.synchronize()
    c = counters.cpu()
    assert bool((c[:4] == -7).all() and (c[9:] == -7).all()), 'topk_hits: store outside the counters'
    assert bool((c[4 + len(ks):8] == 0).all()), 'topk_hits: a counter past n_k was written'
    if pr is not None:
        pr.check('probs')
    return c[4:4 + len(ks)].tolist(), int(c[8]), None if pr is None else pr.inner.view(B, C_).cpu(), counters


def topk_inputs(B, V, C_, ties, seed):
    """logits [B*V, C]; clip b's label is tied (same logits in every view) with `ties` other classes"""
    g = torch.Generator().manual_seed(seed)
    z = torch.randn(B * V, C_, generator=g).view(B, V, C_)
    labels = torch.randint(0, C_, (B,), generator=g)
    for b in range(B):
        lab = int(labels[b])
        others = [c for c in torch.randperm(C_, generator=g).tolist() if c != lab][:ties]
        z[b, :, lab] += 1.5 * b / B                    # labels at different ranks
        for c in others:
            z[b, :, c] = z[b, :, lab]
    return z.reshape(B * V, C_).contiguous(), labels


KS = (1, 2, 5, 10)


@pytest.mark.parametrize('C_', [1, 400, 12000])
@pytest.mark.parametrize('V', [1, 2, 3, 5, 10])
def test_topk_hits_counts_equal_the_fp32_twin(V, C_):
    B = 24
    rep = S.Report()
    for ties in (0, 1, 5):
        if ties >= C_:
            continue
        z, labels = topk_inputs(B, V, C_, ties, seed=V * 100 + C_ + ties)
        hits, samples, probs, _ = run_topk(z, labels, V, KS)
        assert (hits, samples) == S.topk_twin(z, labels, V, KS), (ties, hits)
        ref, bd = S.probs_ref(S.view_mean32(z, V))
        S.check('probs', probs, ref, bd, rep)
        z[:V, labels[0]] = NAN                                # clip 0: a NaN label score (a miss)
        labels[1], labels[2], labels[3] = -1, C_, C_ + 5      # labels out of range (misses)
        for n_k in (0, 1, 4):
            ks = KS[:n_k]
            hits, samples, _, _ = run_topk(z, labels, V, ks, probs=False)
            want, nb = S.topk_twin(z, labels, V, ks)
            assert (hits, samples) == (want, nb), (ties, n_k, hits, want)
    _report(rep, 'topk_hits')


def test_topk_hits_counters_accumulate_across_calls():
    z1, l1 = topk_inputs(16, 2, 400, 1, seed=1)
    z2, l2 = topk_inputs(9, 2, 400, 5, seed=2)
    h1, s1, _, cnt = run_topk(z1, l1, 2, KS, probs=False)
    h2, s2, _, _ = run_topk(z2, l2, 2, KS, counters=cnt, probs=False)
    w1, _ = S.topk_twin(z1, l1, 2, KS)
    w2, _ = S.topk_twin(z2, l2, 2, KS)
    assert h1 == w1 and s1 == 16
    assert h2 == [a + b for a, b in zip(w1, w2)] and s2 == 25


def test_topk_hits_refuses_too_many_classes():
    z, labels = topk_inputs(2, 1, 12001, 0, seed=0)
    with pytest.raises(RuntimeError, match='C=12001 classes unsupported'):
        run_topk(z, labels, 1, KS)


# ---- fused optimizer -----------------------------------------------------------------------------------------------------
class OptLayout:
    """parameters, gradients and state as views into flat NaN-filled device buffers, GAP NaN floats between tensors;
    gradient i starts S.opt_misalign(i) floats past 16-byte alignment"""

    def __init__(self, sizes, grads, params, s1, s2, lrs, wds):
        self.sizes = sizes
        self.off, self.goff = [], []
        o = go = 0
        for i, n in enumerate(sizes):
            o = S.cdiv(o + GAP, 4) * 4
            go = S.cdiv(go + GAP, 4) * 4 + S.opt_misalign(i)
            self.off.append(o)
            self.goff.append(go)
            o, go = o + n, go + n
        self.total, self.gtotal = o + GAP, go + GAP
        self.p = torch.full((self.total,), NAN, device='cuda')
        self.s1 = torch.full((self.total,), NAN, device='cuda')
        self.s2 = torch.full((self.total,), NAN, device='cuda')
        self.g = torch.full((self.gtotal,), NAN, device='cuda')
        self.set(self.p, params)
        self.set(self.s1, s1)
        self.set(self.s2, s2)
        self.set(self.g, grads, grad=True)
        rows = []
        for i, n in enumerate(sizes):
            for c in range(0, n, S.CHUNK):
                rows.append(((min(S.CHUNK, n - c) << 32) | i, c))
        self.chunks = torch.tensor(rows, dtype=torch.int64, device='cuda')
        addr = lambda buf, offs: torch.tensor([buf.data_ptr() + 4 * o for o in offs], dtype=torch.int64, device='cuda')
        self.pptr, self.gptr = addr(self.p, self.off), addr(self.g, self.goff)
        self.s1ptr, self.s2ptr = addr(self.s1, self.off), addr(self.s2, self.off)
        self.norm2 = torch.full((len(sizes) + 2 * GAP,), NAN, device='cuda')
        self.partials = torch.full((len(rows),), NAN, device='cuda')
        self.lr = torch.tensor(lrs, dtype=torch.float32, device='cuda')
        self.wd = torch.tensor(wds, dtype=torch.float32, device='cuda')

    def set(self, buf, ts, grad=False):
        for t, o in zip(ts, self.goff if grad else self.off):
            buf[o:o + t.numel()] = t.reshape(-1).cuda()

    def get(self, buf, grad=False):
        torch.cuda.synchronize()
        c = buf.cpu()
        return [c[o:o + n] for o, n in zip(self.goff if grad else self.off, self.sizes)]

    def gaps_intact(self):
        torch.cuda.synchronize()
        for buf, offs in ((self.p, self.off), (self.s1, self.off), (self.s2, self.off), (self.g, self.goff)):
            keep = torch.ones(buf.numel(), dtype=torch.bool)
            for o, n in zip(offs, self.sizes):
                keep[o:o + n] = False
            assert bool(torch.isnan(buf.cpu()[keep]).all()), 'optimizer: store outside a tensor'
        n2 = self.norm2.cpu()
        assert bool(torch.isnan(n2[len(self.sizes):]).all()), 'norm2: store past the tensors'

    def params(self, clip=0.0, **hp):
        p = _lib()[0].OptParams()
        p.chunks, p.n_chunks, p.n_tensors = self.chunks.data_ptr(), self.chunks.shape[0], len(self.sizes)
        p.pptr, p.gptr, p.s1ptr, p.s2ptr = self.pptr.data_ptr(), self.gptr.data_ptr(), self.s1ptr.data_ptr(), self.s2ptr.data_ptr()
        p.norm2, p.lr, p.wd, p.partials = self.norm2.data_ptr(), self.lr.data_ptr(), self.wd.data_ptr(), self.partials.data_ptr()
        p.clip = clip
        for k, v in hp.items():
            setattr(p, k, v)
        return p

    def norm2_call(self):
        _call('vt_opt_norm2', self.params(), 'vt_opt_norm2')
        torch.cuda.synchronize()
        return self.norm2.cpu()[:len(self.sizes)]


def _opt_setup(seed, adam=False, first=False):
    shapes = S.opt_shapes()
    sizes = [int(torch.tensor(s).prod()) for s in shapes]
    grads = S.opt_grads(shapes, seed)
    gen = torch.Generator().manual_seed(seed + 1)
    params = [torch.randn(n, generator=gen) for n in sizes]
    s1 = [0.1 * torch.randn(n, generator=gen) for n in sizes]        # on a first SGD step: junk the kernel must not read
    s2 = [0.01 * torch.rand(n, generator=gen) for n in sizes]
    if adam and first:
        s1, s2 = [torch.zeros(n) for n in sizes], [torch.zeros(n) for n in sizes]
    lrs, wds = S.opt_hyper(len(sizes), lr=1e-3 if adam else 0.05)
    return OptLayout(sizes, grads, params, s1, s2, lrs, wds), grads, lrs, wds


def _check_norm2(lay, grads, rep):
    n2 = lay.norm2_call()
    for i, g in enumerate(grads):
        ref, bd = S.norm2_ref(g)
        S.check(f'norm2 size {g.numel()}', n2[i].view(1), ref.view(1), bd.view(1), rep)
    return n2


def test_opt_norm2_per_tensor():
    lay, grads, _, _ = _opt_setup(0)
    rep = S.Report()
    _check_norm2(lay, grads, rep)
    lay.gaps_intact()
    _report(rep, 'opt_norm2')


def _new_grads(lay, seed):
    grads = S.opt_grads(S.opt_shapes(), seed)
    lay.set(lay.g, grads, grad=True)
    return grads


@pytest.mark.parametrize('clip', [S.OPT_CLIP, 0.0])
@pytest.mark.parametrize('nesterov', [True, False])
def test_opt_sgd_one_step_at_a_time(nesterov, clip):
    lay, grads, lrs, wds = _opt_setup(1)
    mom = S.f32(0.9)
    rep = S.Report()
    for step in range(3):
        if step:
            grads = _new_grads(lay, 10 + step)
        n2 = _check_norm2(lay, grads, rep)
        w0, b0 = lay.get(lay.p), lay.get(lay.s1)
        _call('vt_opt_sgd', lay.params(clip, momentum=mom, nesterov=int(nesterov), first_step=int(step == 0)), 'vt_opt_sgd')
        w1, b1 = lay.get(lay.p), lay.get(lay.s1)
        lay.gaps_intact()
        for i, g in enumerate(grads):
            pr, pb, br, bb = S.sgd_step_ref(w0[i], g, b0[i], S.clip_coef_ref(n2[i], clip), lrs[i], wds[i], mom, nesterov, step == 0)
            S.check('sgd param', w1[i], pr, pb, rep)
            S.check('sgd momentum', b1[i], br, bb, rep)
    _report(rep, 'opt_sgd')


@pytest.mark.parametrize('step', [1, 1000])
def test_opt_adamw_one_step_at_a_time(step):
    lay, grads, lrs, wds = _opt_setup(2, adam=True, first=step == 1)
    b1, b2, eps = S.f32(0.9), S.f32(0.999), S.f32(1e-8)
    rep = S.Report()
    for t in (step, step + 1):
        if t != step:
            grads = _new_grads(lay, 20 + t)
        bc1, bc2 = S.f32(1 - 0.9 ** t), S.f32(1 - 0.999 ** t)
        n2 = _check_norm2(lay, grads, rep)
        w0, m0, v0 = lay.get(lay.p), lay.get(lay.s1), lay.get(lay.s2)
        _call('vt_opt_adamw', lay.params(S.OPT_CLIP, beta1=b1, beta2=b2, eps=eps, bc1=bc1, bc2=bc2), 'vt_opt_adamw')
        w1, m1, v1 = lay.get(lay.p), lay.get(lay.s1), lay.get(lay.s2)
        lay.gaps_intact()
        for i, g in enumerate(grads):
            pr, pb, mr, mb, vr, vb = S.adamw_step_ref(w0[i], g, m0[i], v0[i], S.clip_coef_ref(n2[i], S.OPT_CLIP),
                                                     lrs[i], wds[i], b1, b2, eps, bc1, bc2)
            S.check('adamw param', w1[i], pr, pb, rep)
            S.check('adamw exp_avg', m1[i], mr, mb, rep)
            S.check('adamw exp_avg_sq', v1[i], vr, vb, rep)
    _report(rep, 'opt_adamw')


def test_opt_norm2_and_step_are_bitwise_reproducible():
    """the 36-chunk fc1 weight's norm2, and the clipped SGD step that follows, give the same bits on ten calls"""
    shapes = [(3072, 768), (5,), (65537,)]
    sizes = [int(torch.tensor(s).prod()) for s in shapes]
    gen = torch.Generator().manual_seed(7)
    grads = [torch.randn(n, generator=gen) * 1e-3 for n in sizes]
    params = [torch.randn(n, generator=gen) for n in sizes]
    mom = [torch.randn(n, generator=gen) for n in sizes]
    lay = OptLayout(sizes, grads, params, mom, mom, [0.05] * 3, [1e-4] * 3)
    assert S.chunks_of(sizes[0]) == 36
    first = None
    for _ in range(10):
        lay.set(lay.p, params)
        lay.set(lay.s1, mom)
        n2 = lay.norm2_call()
        _call('vt_opt_sgd', lay.params(0.5, momentum=0.9, nesterov=1, first_step=0), 'vt_opt_sgd')
        got = (n2.view(torch.int32).clone(), lay.p.cpu().view(torch.int32), lay.s1.cpu().view(torch.int32))
        if first is None:
            first = got
        else:
            for a, b in zip(first, got):
                assert torch.equal(a, b), 'the optimizer step is not reproducible'
