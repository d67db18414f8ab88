"""CPU model of the tensor-core flash attention (videotransformer_pytorch_b200/csrc/vt_attention_mma.cu), a closed-form fp64
reference of the same operation, and the per-row error metric the attention tests gate on.

The model walks the kernels' 64-row tiles:
  forward : key tiles of 64, running max m, corr = exp2(m_old - m_new), l summed from the unrounded P, P rounded to bf16
            before P V; scores in the log2 domain (s * scale * log2 e); lse stored as (m + log2 l) * ln 2.
  dQ      : key tiles of 64, P = exp2(s * scale * log2 e - lse * log2 e), dS = P (dP - delta) rounded to bf16 before dS K.
  dK / dV : every query tile in turn; P and dS rounded to bf16 before the dV and dK MMAs.
Rows past Nq and Nk are staged as zeros (stage_rows), keys past Nk are masked to -inf (forward) or P = 0 (dQ), query rows
past Nq get lse = +inf (P = 0) in the dK / dV walk, and delta = rowsum(dO * O) is recomputed from the O and dO it is given
(the bf16 tensors, on the GPU).  Rows are independent, so all query rows of the forward and dQ walks (all key rows of the
dK / dV walk) are processed together; only the tile loop that accumulates is sequential.

Modes:
  'exact'    fp64, no rounding: must agree with `reference` to ~1e-12.
  'bf16'     rounds where the tensor-core kernels do: P before P V, O and dQ on output, P and dS before the dV / dK MMAs, and
             dK / dV on output for the packed-qkv path (`dkv_bf16=True`; the strided path stores fp32).  Arithmetic stays
             fp64, so this is the bf16 noise a correct kernel shows, without the (much smaller) fp32-order and ex2.approx
             noise.
  'bf16_out' rounds only the stored bf16 outputs: the noise model of the CUDA-core kernels (fp32 probabilities).
Operands are [P, rows, hd] (P independent problems).  Arrays may hold rows past Nq / Nk (what lies in memory after the
last row); the model never reads them, like the kernels.
"""
from collections import namedtuple

import torch

MT = 64
LOG2E = 1.4426950408889634
LN2 = 0.6931471805599453
F64 = torch.float64


def bf16(x):
    """round to bf16 (round-to-nearest-even from fp32, as __floats2bfloat162_rn) and back"""
    return x.to(torch.float32).to(torch.bfloat16).to(F64)


def _same(x):
    return x


def _tiles(x, limit):
    """rows [0, limit) of x [P, R, hd] zero-padded to a multiple of MT rows"""
    n = -(-limit // MT) * MT
    t = x.new_zeros((x.shape[0], n, x.shape[2]), dtype=F64)
    t[:, :limit] = x[:, :limit]
    return t


def _stage(x, r0, limit):
    """stage_rows: rows [r0, r0 + MT) of x; rows >= limit are zero"""
    t = x.new_zeros((x.shape[0], MT, x.shape[2]), dtype=F64)
    n = min(MT, limit - r0)
    t[:, :n] = x[:, r0:r0 + n]
    return t


def _rounding(mode):
    if mode not in ('exact', 'bf16', 'bf16_out'):
        raise ValueError(f'unknown mode {mode!r}')
    return (bf16 if mode == 'bf16' else _same), (_same if mode == 'exact' else bf16)


def fwd(q, k, v, scale, mode='exact', Nq=None, Nk=None):
    """-> o [P, Nq, hd], lse [P, Nq] (natural log)"""
    Nq = q.shape[1] if Nq is None else Nq
    Nk = k.shape[1] if Nk is None else Nk
    rnd_p, rnd_out = _rounding(mode)
    Q = _tiles(q, Nq)
    c = scale * LOG2E
    m = torch.full(Q.shape[:2], -torch.inf, dtype=F64)
    l = torch.zeros(Q.shape[:2], dtype=F64)
    o = torch.zeros(Q.shape, dtype=F64)
    for k0 in range(0, Nk, MT):
        Ks, Vs = _stage(k, k0, Nk), _stage(v, k0, Nk)
        s = (Q @ Ks.transpose(1, 2)) * c
        s[:, :, Nk - k0:] = -torch.inf
        mn = torch.maximum(m, s.amax(-1))                   # finite: every tile holds at least one key
        corr = torch.exp2(m - mn)
        p = torch.exp2(s - mn[..., None])
        l = l * corr + p.sum(-1)
        o = o * corr[..., None] + rnd_p(p) @ Vs
        m = mn
    return rnd_out(o / l[..., None])[:, :Nq], ((m + torch.log2(l)) * LN2)[:, :Nq]


def bwd(q, k, v, o, do, lse, scale, mode='exact', dkv_bf16=False, Nq=None, Nk=None):
    """-> dq [P, Nq, hd], dk, dv [P, Nk, hd]; dkv_bf16: dK / dV stored as bf16 (packed qkv) instead of fp32 (strided)"""
    Nq = q.shape[1] if Nq is None else Nq
    Nk = k.shape[1] if Nk is None else Nk
    rnd_p, rnd_out = _rounding(mode)
    rnd_dkv = rnd_out if dkv_bf16 else _same
    c = scale * LOG2E
    Q, dO, O = _tiles(q, Nq), _tiles(do, Nq), _tiles(o, Nq)
    L = torch.full(Q.shape[:2], torch.inf, dtype=F64)        # rows past Nq: +inf => P = 0
    L[:, :Nq] = lse[:, :Nq].to(F64) * LOG2E
    delta = (dO * O).sum(-1)
    # dQ: CTA = 64 query rows, key tiles streamed
    dq = torch.zeros(Q.shape, dtype=F64)
    for k0 in range(0, Nk, MT):
        Ks, Vs = _stage(k, k0, Nk), _stage(v, k0, Nk)
        p = torch.exp2((Q @ Ks.transpose(1, 2)) * c - L[..., None])
        p[:, :, Nk - k0:] = 0.0
        ds = p * (dO @ Vs.transpose(1, 2) - delta[..., None])
        dq = dq + rnd_p(ds) @ Ks
    # dK / dV: CTA = 64 key rows, every query tile in turn
    Kr, Vr = _tiles(k, Nk), _tiles(v, Nk)
    dk = torch.zeros(Kr.shape, dtype=F64)
    dv = torch.zeros(Kr.shape, dtype=F64)
    for q0 in range(0, Nq, MT):
        Qs, dOs = _stage(q, q0, Nq), _stage(do, q0, Nq)
        Ls, Ds = L[:, q0:q0 + MT], delta[:, q0:q0 + MT]
        p = torch.exp2((Kr @ Qs.transpose(1, 2)) * c - Ls[:, None, :])
        ds = p * (Vr @ dOs.transpose(1, 2) - Ds[:, None, :])
        dv = dv + rnd_p(p) @ dOs
        dk = dk + rnd_p(ds) @ Qs
    return rnd_out(dq * scale)[:, :Nq], rnd_dkv(dk * scale)[:, :Nk], rnd_dkv(dv)[:, :Nk]


def reference(q, k, v, do, scale):
    """closed-form fp64 attention and its gradients: (o, lse, dq, dk, dv); q [P, Nq, hd], k / v [P, Nk, hd]"""
    q, k, v, do = (t.to(F64) for t in (q, k, v, do))
    s = (q @ k.transpose(1, 2)) * scale
    lse = torch.logsumexp(s, -1)
    p = torch.exp(s - lse[..., None])
    o = p @ v
    ds = p * (do @ v.transpose(1, 2) - (do * o).sum(-1, keepdim=True))
    return o, lse, scale * (ds @ k), scale * (ds.transpose(1, 2) @ q), p.transpose(1, 2) @ do


# ---- per-row error metric ---------------------------------------------------------------------------------------------
RowErr = namedtuple('RowErr', 'worst where glob')
ROW_FLOOR = 0.1     # rows shorter than this fraction of the rms row norm are measured against that floor


def row_errors(got, ref, floor=ROW_FLOOR):
    """Compare one output with its fp64 reference row by row.  got / ref: [B, H, R, hd] (or [P, R, hd] = [P, 1, R, hd]); a row
    is one (b, h, query) of o / dq or one (b, h, key) of dk / dv.  Row error = |got - ref| / max(|ref row|, floor * rms row
    norm).  A reference that is zero everywhere is compared absolutely.
    -> RowErr(worst row error, (b, h, row) where it occurs, global relative L2)"""
    got, ref = got.detach().cpu().to(F64), ref.detach().cpu().to(F64)
    if ref.dim() == 3:
        got, ref = got[:, None], ref[:, None]
    assert got.shape == ref.shape, (got.shape, ref.shape)
    err = (got - ref).norm(dim=-1)
    norm = ref.norm(dim=-1)
    rms = float(norm.square().mean().sqrt())
    den = norm.clamp(min=floor * rms) if rms > 0 else torch.ones_like(norm)
    e = err / den
    e = torch.where(torch.isnan(e), torch.full_like(e, torch.inf), e)
    i = int(e.argmax())
    B, H, R = e.shape
    glob = float(err.square().sum().sqrt()) / (float(norm.square().sum().sqrt()) if rms > 0 else 1.0)
    return RowErr(float(e.reshape(-1)[i]), (i // (H * R), (i // R) % H, i % R), glob)


# Gates.  Against fp64: a kernel output passes when its worst row is within C_ROW times the worst row of the model of the
# same kernel on the same inputs, and its global error within C_GLOB times the model's, each plus ABS_FLOOR (fp32
# accumulation noise where the model rounds nothing, e.g. fp32 dK / dV).  Against the model itself (same rounding points):
# the global distance must stay within D_GLOB times the model's own global error against fp64.
# The factors were fixed once on the CPU.  The GPU differs from the model by fp32 summation order and ex2.approx (relative
# ~1e-7 .. 1e-6), which matter only where they flip a bf16 rounding of P, dS or an output.  The same flips arise when the
# 'bf16' model runs in fp32 instead of fp64 arithmetic; over the shapes, scales and logit regimes of
# tests/test_gpu_attention_edges.py (4 problems each) that fp32 run against the fp64 one gave worst-row ratios of at most
# 1.03, global ratios of at most 1.01, and a global distance of at most 0.24 times the model's error.  A per-row distance to
# the model is not gated: one flipped output element can move a well-conditioned row by up to 1.6x the model's worst row.
C_ROW, C_GLOB, D_GLOB, ABS_FLOOR = 1.5, 1.2, 0.5, 2e-4
LSE_TOL = 2e-5      # |lse - ref| / (1 + |ref|): fp32 scores, ex2.approx and log2f, no bf16 rounding on the way


def within_budget(got, ref, model):
    """-> (ok, RowErr of got, RowErr of the model): the fp64 gate above"""
    g, m = row_errors(got, ref), row_errors(model, ref)
    return g.worst <= C_ROW * m.worst + ABS_FLOOR and g.glob <= C_GLOB * m.glob + ABS_FLOOR, g, m


# ---- inputs -----------------------------------------------------------------------------------------------------------
REGIMES = ('benign', 'max_last', 'max_first', 'uniform', 'zero_row')


def make_inputs(P, Nq, Nk, hd, scale, regime='benign', seed=0):
    """bf16-valued fp64 q, do [P, Nq, hd] and k, v [P, Nk, hd] whose scaled logits follow `regime`:
      benign    logits ~ N(0, 1.5^2) whatever the scale;
      max_last  keys of the last 64-key tile at about +28 .. +31, the others ~ N(0, 1.5^2): the running max moves late;
      max_first keys after the first tile about 100 below the first tile's: their exp2 underflows;
      uniform   every logit of a row equal (P = 1 / Nk, l = Nk); k differs between keys only where q is zero, so dq != 0;
      zero_row  benign with query rows 0, Nq / 2 and Nq - 1 all zero."""
    g = torch.Generator().manual_seed(seed)
    rn = lambda n: torch.randn(P, n, hd, generator=g, dtype=F64)
    a = (1.5 / (scale * hd ** 0.5)) ** 0.5
    q, k, v, do = rn(Nq) * a, rn(Nk) * a, rn(Nk), rn(Nq)
    if regime in ('max_last', 'max_first'):
        q[:, :, 0] = 1.0
        last = (Nk - 1) // MT * MT
        if regime == 'max_last':
            k[:, :, 0] = 0.0
            k[:, last:, 0] = 28.0 / scale
        else:
            k[:, :MT, 0] = 0.0
            k[:, MT:, 0] = -100.0 / scale
    elif regime == 'uniform':
        q[:, :, hd // 2:] = 0.0
        k[:, :, :hd // 2] = k[:, :1, :hd // 2]
    elif regime == 'zero_row':
        q[:, [0, Nq // 2, Nq - 1]] = 0.0
    elif regime != 'benign':
        raise ValueError(regime)
    return tuple(bf16(t) for t in (q, k, v, do))


def lse_error(got, ref):
    """worst |got - ref| / (1 + |ref|) of a log-sum-exp [..., R] and the flat index where it occurs"""
    got, ref = got.detach().cpu().to(F64).reshape(-1), ref.detach().cpu().to(F64).reshape(-1)
    e = (got - ref).abs() / (1 + ref.abs())
    e = torch.where(torch.isnan(e), torch.full_like(e, torch.inf), e)
    i = int(e.argmax())
    return float(e[i]), i
