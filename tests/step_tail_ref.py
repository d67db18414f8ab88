"""fp64 references and per-element bounds for the kernels at the end of every training and evaluation step: the
classification head (linear_small fwd / wgrad / db / dgrad), softmax cross-entropy, the top-k counters (csrc/vt_head.cu)
and the fused clip + optimizer step (csrc/vt_optim.cu).  CPU only.

With u = 2^-24 and gamma_n = n u / (1 - n u), a value formed by a tree of additions (or fmas) whose longest chain has n
roundings is within gamma_n sum|terms| of the exact sum, whatever the shape of the tree.  Each n below is that chain in
the kernel's own order of operations:

  linear_small_fwd   lane l walks the float4 groups l, l + 32, ... of K in order, 4 fmas per group: 4 ceil(K / 128)
                     roundings; then the 5-level shuffle tree and the bias: n = 4 ceil(K / 128) + 6 over sum|x w| + |b|
  wgrad / db         one chain over the M rows: n = M over sum_m |dy x| (sum_m |dy| for db)
  dgrad              warp q walks n = q, q + 8, ... (ceil(N / 8) fmas), then the 8 warp partials in order: n = ceil(N / 8) + 7
  softmax_ce         every row sum (sum e^(z - mx), sum t, sum t (z - mx)) is ceil(N / 256) terms per thread, a 5-level
                     shuffle tree and the 8 warp partials in order: n = ceil(N / 256) + 12; expf is within 2 ulp (4u
                     relative), logf within 1 ulp (2u), z - mx rounds once (u |z - mx|, so e^(z - mx) gains u |z - mx|);
                     a subnormal e^(z - mx) carries an absolute error of a few 2^-149, covered by ETA
  topk probs         the same softmax over the fp32 view mean, ceil(C / 256) + 12 terms
  opt_norm2          a thread's ceil(len / 256) squares of one chunk (plus the float4 pair sums and one tail element),
                     the shuffle tree, the 8 warp partials, then the tensor's chunk partials in chunk order:
                     n = ceil(min(len, CHUNK) / 256) + 3 + 5 + 8 + chunks over sum g^2
  opt_sgd / adamw    one step from the kernel's own fp32 state: every rounding of the update, in the kernel's order, bounded
                     relative to the fp64 value it rounds (see sgd_step_ref / adamw_step_ref); the clip coefficient
                     clip / (sqrtf(norm2) + 1e-6f) is 3 roundings (gamma_3), and min(1, .) does not increase an error

Every bound is multiplied by SECOND_ORDER, which covers the products of two or more u terms the first-order sums leave out.
The top-k counts have no bound: they must equal topk_twin, an fp32 replay of the contract in include/vt_b200.h.
"""
import torch

from tests.mvit_pool_ref import U, gamma, check, Report  # noqa: F401  (re-exported for the tests)

SECOND_ORDER = 1 + 2.0 ** -10
EXP_REL = 4 * U                  # expf: 2 ulp
LOG_REL = 2 * U                  # logf: 1 ulp
RSQRT_REL = 4 * U                # rsqrtf: 2 ulp
ETA = 2.0 ** -140                # absolute slack for subnormal softmax terms (a few ulps of 2^-149, after scaling)
CHUNK = 1 << 16                  # optim.CHUNK: elements per optimizer chunk
CLIP_EPS = float(torch.tensor(1e-6, dtype=torch.float32))
F32 = torch.float32


def cdiv(a, b):
    return -(-a // b)


def f32(v):
    """v rounded to fp32, as a Python float (how a hyperparameter reaches the kernels)"""
    return float(torch.tensor(v, dtype=F32))


# ---- linear_small -------------------------------------------------------------------------------------------------------
def ls_fwd_n(K):
    return 4 * cdiv(K, 128) + 6


def ls_dgrad_n(N):
    return cdiv(N, 8) + 7


def linear_fwd_ref(x, w, b):
    """(ref, bound) of y = x w^T + b"""
    xd, wd = x.double(), w.double()
    ref, mag = xd @ wd.T, xd.abs() @ wd.abs().T
    if b is not None:
        ref, mag = ref + b.double(), mag + b.double().abs()
    return ref, SECOND_ORDER * gamma(ls_fwd_n(x.shape[1])) * mag


def linear_wgrad_ref(dy, x):
    """(dw, bound, db, bound) of dw = dy^T x, db = colsum(dy)"""
    M = x.shape[0]
    d, xd = dy.double(), x.double()
    g = SECOND_ORDER * gamma(M)
    return d.T @ xd, g * (d.abs().T @ xd.abs()), d.sum(0), g * d.abs().sum(0)


def linear_dgrad_ref(dy, w):
    """(ref, bound) of dx = dy w"""
    d, wd = dy.double(), w.double()
    return d @ wd, SECOND_ORDER * gamma(ls_dgrad_n(w.shape[0])) * (d.abs() @ wd.abs())


# ---- softmax cross-entropy ----------------------------------------------------------------------------------------------
def ce_n(N):
    return cdiv(N, 256) + 12


def _exp_rel(d):
    """relative error bound of expf(fl(d)) against e^d per element (d <= 0; -inf gives an exact 0)"""
    r = (1 + EXP_REL) * torch.exp(U * d.abs()) - 1
    return torch.where(torch.isfinite(d), r, torch.zeros_like(r))


def softmax_ce_ref(z, t):
    """z fp32 [M, N] logits, t [M, N] targets (one-hot rows for hard labels) -> dict of fp64 references and bounds:
    dz / dz_bound [M, N], row / row_bound [M], loss / loss_bound (the loss against the mean of `row`).  Terms with t = 0 are
    left out of sum t (z - mx), as the kernel and torch's log_softmax form do."""
    M, N = z.shape
    zd, td = z.double(), t.double()
    n = ce_n(N)
    g = float(gamma(n))
    mx = zd.max(1, keepdim=True).values
    d = zd - mx
    e = torch.exp(d)
    se = e.sum(1, keepdim=True)
    ts = td.sum(1, keepdim=True)
    e_ts = g * td.abs().sum(1, keepdim=True)                   # |error| of the kernel's sum t
    de = _exp_rel(d)
    th = (e * de).sum(1, keepdim=True) / se + g * (1 + de.max(1, keepdim=True).values)   # relative error of sum e
    p = e / se
    P = p * ts
    dz = (P - td) / M
    dzb = SECOND_ORDER * ((P * (de + th + 3 * U) + p * e_ts) * (1 + U) + 3 * U * (P - td).abs()) / M + ETA
    ls = torch.log(se)
    tdm = torch.where(td != 0, td * d, torch.zeros_like(d))
    tzm = tdm.sum(1, keepdim=True)
    L1 = ts * ls
    row = L1 - tzm
    err_l1 = ts.abs() * (th / (1 - th) + LOG_REL * ls.abs()) + ls.abs() * e_ts + U * L1.abs()
    err_tz = (U + g * (1 + U)) * tdm.abs().sum(1, keepdim=True)
    rowb = SECOND_ORDER * (err_l1 + err_tz + U * (L1.abs() + tzm.abs()))
    row, rowb = row[:, 0], rowb[:, 0]
    loss = row.mean()
    lossb = SECOND_ORDER * (rowb.sum() / M + gamma(M + 2) * (row.abs() + rowb).sum() / M)
    return dict(dz=dz, dz_bound=dzb, row=row, row_bound=rowb, loss=loss, loss_bound=lossb)


def one_hot(labels, N):
    """fp32 [M, N] targets of hard labels (a label outside [0, N) gives a zero row)"""
    t = torch.zeros(labels.numel(), N)
    ok = (labels >= 0) & (labels < N)
    t[torch.arange(labels.numel())[ok], labels[ok]] = 1
    return t


# ---- top-k counters -----------------------------------------------------------------------------------------------------
def view_mean32(logits, V):
    """the fp32 mean of vt_topk_hits: views summed in order, then times the fp32 1 / V"""
    BV, C = logits.shape
    z = logits.view(BV // V, V, C)
    m = z[:, 0].clone()
    for v in range(1, V):
        m = m + z[:, v]
    return m * (torch.tensor(1.0, dtype=F32) / torch.tensor(float(V), dtype=F32))


def topk_twin(logits, labels, V, ks, strict=True):
    """(hits per k, samples) of one vt_topk_hits call, exactly: rank = #classes whose fp32 mean is strictly greater than the
    label's; a label outside [0, C) or a NaN label score is a miss for every k.  strict=False ranks ties against the label
    (a planted defect)."""
    mean = view_mean32(logits, V)
    B, C = mean.shape
    hits = [0] * len(ks)
    for b in range(B):
        lab = int(labels[b])
        if 0 <= lab < C and not bool(torch.isnan(mean[b, lab])):
            ml = mean[b, lab]
            rank = int((mean[b] > ml).sum()) if strict else int((mean[b] >= ml).sum()) - 1
        else:
            rank = C
        for i, k in enumerate(ks):
            hits[i] += int(rank < k)
    return hits, B


def probs_ref(mean):
    """(ref, bound) of softmax over the fp32 view mean [B, C] as the kernel forms it"""
    md = mean.double()
    d = md - md.max(1, keepdim=True).values
    e = torch.exp(d)
    se = e.sum(1, keepdim=True)
    de = _exp_rel(d)
    th = (e * de).sum(1, keepdim=True) / se + float(gamma(ce_n(mean.shape[1]))) * (1 + de.max(1, keepdim=True).values)
    p = e / se
    return p, SECOND_ORDER * p * (de + th + 2 * U) + ETA


# ---- fused optimizer ----------------------------------------------------------------------------------------------------
def chunks_of(n):
    return cdiv(n, CHUNK)


def norm2_n(n):
    return cdiv(min(n, CHUNK), 256) + 3 + 5 + 8 + chunks_of(n)


def norm2_ref(g):
    """(ref, bound) of sum(g^2) of one gradient tensor"""
    s = (g.double() ** 2).sum()
    return s, SECOND_ORDER * gamma(norm2_n(g.numel())) * s


def clip_coef_ref(norm2, clip):
    """(coef, |error| bound) of min(1, clip / (sqrtf(norm2) + 1e-6f)) from the kernel's own fp32 norm2; clip <= 0: 1"""
    if clip <= 0:
        return 1.0, 0.0
    c = clip / (float(norm2) ** 0.5 + CLIP_EPS)
    err = SECOND_ORDER * float(gamma(3)) * c if c < 1 + 8 * U else 0.0
    return min(c, 1.0), err


def sgd_step_ref(w, g, buf, coef, lr, wd, mom, nesterov, first):
    """fp64 (p, buf) after one SGD step from the fp32 state (w, g, buf) and their bounds; coef = (value, error)"""
    c, ec = coef
    w, g, buf = w.double(), g.double(), buf.double()
    gc = g * c
    e_gc = g.abs() * ec + U * gc.abs()
    d = gc + wd * w
    e_d = e_gc + U * d.abs()
    b = d if first else mom * buf + d
    e_b = e_d + U * b.abs()
    dn = d + mom * b if nesterov else b
    e_dn = (mom * e_b + e_d + U * dn.abs()) if nesterov else e_b
    p = w - lr * dn
    e_p = lr * e_dn + U * p.abs()
    return p, SECOND_ORDER * e_p, b, SECOND_ORDER * e_b


def adamw_step_ref(w, g, m, v, coef, lr, wd, b1, b2, eps, bc1, bc2):
    """fp64 (p, m, v) after one AdamW step from the fp32 state and their bounds; hyperparameters as the kernel's fp32"""
    c, ec = coef
    w, g, m, v = w.double(), g.double(), m.double(), v.double()
    gi = g * c
    e_g = g.abs() * ec + U * gi.abs()
    f = 1 - lr * wd
    e_f = U * lr * wd + U * abs(f)
    w1 = w * f
    e_w1 = w.abs() * e_f + U * w1.abs()
    mi = b1 * m + (1 - b1) * gi
    e_m = (1 - b1) * (e_g + U * gi.abs()) + U * mi.abs()
    vi = b2 * v + (1 - b2) * gi * gi
    e_v = (1 - b2) * (2 * gi.abs() * e_g + 2 * U * gi * gi) + U * vi.abs()
    ss, isb = lr / bc1, bc2 ** -0.5
    sq = vi.sqrt()
    e_sq = torch.minimum(e_v.sqrt(), torch.where(sq > 0, e_v / sq.clamp_min(1e-300), torch.full_like(sq, float('inf'))))
    den = sq * isb + eps
    e_den = isb * e_sq + sq * isb * (2 * U + RSQRT_REL) + U * den
    upd = ss * mi / den
    e_upd = ss * e_m / den + upd.abs() * (e_den / den + 3 * U)
    p = w1 - upd
    e_p = e_w1 + e_upd + U * p.abs()
    so = SECOND_ORDER
    return p, so * e_p, mi, so * e_m, vi, so * e_v


def timesformer_b_shapes():
    """parameter shapes of TimeSformer-B's embeddings, cls token, one divided space-time block and the 400-class head"""
    D, F = 768, 3072
    s = [(D, 3, 1, 16, 16), (D,), (1, 1, D), (1, 197, D), (1, 8, D)]
    for _ in range(2):                                   # temporal then spatial attention
        s += [(D,), (D,), (3 * D, D), (3 * D,), (D, D), (D,)]
    s += [(D, D), (D,)]                                  # temporal_fc
    s += [(D,), (D,), (F, D), (F,), (D, F), (D,)]        # FFN norm, fc1, fc2
    s += [(D,), (D,), (400, D), (400,)]                  # final norm, head
    return s


# ---- the cases of tests/test_gpu_step_tail_edges.py (also replayed by the fp32 models of tests/test_step_tail_bounds.py) --
# (M, N, K): every M, N and K of the head's edges at least once; 4095 / 4096 rows, K below 128, K % 128 != 0, N % 8 != 0
LS_TRIPLES = [(1, 400, 768), (7, 1, 4), (8, 7, 96), (9, 8, 100), (72, 9, 124), (4095, 174, 128), (4096, 9, 132),
              (8, 1000, 1024), (9, 700, 132), (1, 174, 100), (72, 400, 768), (4096, 1, 1024), (7, 1000, 4), (4095, 8, 96)]
CE_M = (1, 8, 4096)
CE_N = (1, 7, 255, 256, 257, 400, 700, 1000)
CE_REGIMES = ('randn', 'equal', 'dominant', 'offset_up', 'offset_down', 'label_min', 'unnormalised', 'neg_inf')


def ls_inputs(M, N, K, exact, seed):
    """x [M, K], w [N, K], b [N], dy [M, N]: integers in [-8, 8] (every sum exact in fp32 in any order) or randn"""
    g = torch.Generator().manual_seed(seed)
    if exact:
        mk = lambda *s: torch.randint(-8, 9, s, generator=g).float()
    else:
        mk = lambda *s: torch.randn(*s, generator=g)
    return mk(M, K), mk(N, K), mk(N), mk(M, N)


def ce_inputs(M, N, regime, soft, seed):
    """-> (z fp32 [M, N], labels int64 [M], targets fp32 [M, N]).  Soft targets are Mixup of the label with another class
    plus label smoothing 0.1; 'unnormalised' scales each soft row by a factor in [0.5, 1.5] so it does not sum to 1.
    'neg_inf' (hard labels) sets every third logit that is not the label to -inf."""
    g = torch.Generator().manual_seed(seed)
    z = 3 * torch.randn(M, N, generator=g)
    labels = torch.randint(0, N, (M,), generator=g)
    if regime == 'equal':
        z = torch.full((M, N), 1.75)
    elif regime == 'dominant':
        z[torch.arange(M), labels] = z.max(1).values + 100
    elif regime == 'offset_up':
        z = z + 1e4
    elif regime == 'offset_down':
        z = z - 1e4
    elif regime == 'label_min':
        labels = z.argmin(1)
    if not soft:
        if regime == 'neg_inf':
            mask = (torch.arange(N)[None, :] % 3 == 1) & (torch.arange(N)[None, :] != labels[:, None])
            z = torch.where(mask, torch.full_like(z, float('-inf')), z)
        return z.contiguous(), labels, one_hot(labels, N)
    other = torch.randint(0, N, (M,), generator=g)
    lam = torch.rand(M, 1, generator=g)
    t = lam * one_hot(labels, N) + (1 - lam) * one_hot(other, N)
    t = t * 0.9 + 0.1 / N
    if regime == 'unnormalised':
        t = t * (0.5 + torch.rand(M, 1, generator=g))
    return z.contiguous(), labels, t.float().contiguous()


OPT_SIZES = [1, 3, 4, 5, 65535, 65536, 65537, 3 * 65536 + 5]
OPT_CLIP = 1.0


def opt_shapes():
    return [(n,) for n in OPT_SIZES] + timesformer_b_shapes()


def opt_misalign(i):
    """floats by which tensor i's gradient view starts past 16-byte alignment: 0, 1, 2, 3, 0, ..."""
    return i % 4


def opt_grads(shapes, seed):
    """gradients whose norms fall on both sides of OPT_CLIP, every 7th element 0; tensor 2 (4 elements of +-0.5) has a norm of
    exactly OPT_CLIP, tensor 0 (one element, 1.0) too, tensor 3 (5 elements) is all zero"""
    g = torch.Generator().manual_seed(seed)
    out = []
    for i, s in enumerate(shapes):
        n = 1
        for d in s:
            n *= d
        t = torch.randn(n, generator=g) * ((0.25, 4.0, 0.9, 1.6)[i % 4] / max(n, 1) ** 0.5)
        t[::7] = 0
        if i == 0:
            t = torch.ones(1)
        elif i == 2:
            t = torch.tensor([0.5, -0.5, 0.5, -0.5])
        elif i == 3:
            t = torch.zeros(5)
        assert t.numel() == n, (i, s)
        out.append(t.float())
    return out


def opt_hyper(n_tensors, lr=0.05, wd=0.05):
    """per-tensor fp32 lr (base lr times a per-group lr_scale) and weight decay (0 for a no-decay group)"""
    lrs = [f32(lr * (1.0, 0.5, 0.25)[i % 3]) for i in range(n_tensors)]
    wds = [f32(0.0 if i % 5 == 1 else wd * (1 + i % 2)) for i in range(n_tensors)]
    return lrs, wds
