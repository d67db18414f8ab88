"""Reference arithmetic of the element-wise GEMM checks (test_gpu_gemm_exact.py), kept apart so that the host tests can
check it without a GPU.

Exact regime.  Operands are integers in [-3, 3] stored as bf16, so every product is an integer of magnitude <= 9 and
every partial sum of K products an integer of magnitude <= 9 K.  While 9 K < 2^24 each fp32 addition is exact in any
order: split-K partials, any tile order and the CUDA-core remainder rows all give the same integer.  bias, bias2 and aux
are multiples of 1/4 and row_scale is +-2^j with j in [-2, 2], so the epilogue's intermediates are multiples of 1/16; the
premise check below bounds each intermediate's magnitude over its resolution by 2^24, so that every step of the epilogue
(either order of the additions, with or without an FMA) is exact in fp32.  The expected output is then the float64 result
rounded once: to fp32 it is the value itself, to bf16 its round-to-nearest-even.

GELU.  The kernels compute erf with Abramowitz-Stegun 7.1.26 (erf_fast_pos in vt_common.cuh):
    erf(x) ~ 1 - P(t) t e,   t = 1 / (1 + p x),   e = exp(-x^2),   |error| <= 1.5e-7 (A-S, for x >= 0)
with P of degree 4 evaluated by Horner's rule in fp32, t by a correctly rounded reciprocal and e by __expf.  With
u = 2^-24, x = |z| / sqrt(2), S(t) = sum_i |a_i| t^i (i = 1..5, the polynomial's absolute weights):
  - Horner with one rounding per FMA step errs by at most 4 u S(t) (Higham, Thm 5.1, FMA form); t carries two roundings
    (the FMA and the reciprocal), which a degree-5 polynomial in t amplifies at most 5-fold: 10 u S(t); the two products
    P t and (P t) e add 2 u S(t).  Together 16 u S(t) e.
  - __expf(y) errs by at most (2 + floor(1.173 |y|)) ulp (CUDA C Programming Guide, intrinsic functions), i.e. that many
    2^-23 relative, and the fp32 argument x^2 = (|z| fl(1/sqrt 2))^2 carries 5 roundings relative, which exp turns into
    5 u x^2 relative; results below 2^-126 lose relative precision: at most 2^-126 absolute.  Weighted by P t <= S(t).
  - 1 - P t e rounds once (u), and the argument rounding moves erf by at most (2/sqrt pi) e x 2u.
This is E_erf(z).  The fp32 GELU 0.5 z (1 + erf) then carries 0.5 |z| E_erf plus two roundings (the sum and the product,
0.5 z being exact), and its derivative 0.5 (1 + erf) + z c e (c = 1/sqrt(2 pi)) carries 0.5 E_erf, |z| c e (eps_e + 3u)
and two roundings of at most 1 + |d|.  The stored result is the bf16 rounding of that fp32 value: half a bf16 ulp of the
reference moved by the fp32 error, which covers the case where the two fall in different binades.  None of the terms is
fitted: the A-S constant is the published one and the rest follow from the operation count.

Random operands.  Gaussian operands accumulate in fp32 with an error of at most K 2^-23 (|A||B|)_mn, the bound of a
truncating adder (unit roundoff 2^-23) summing K products; split-K adds S - 1 more additions of the partials.  The
epilogue adds at most four roundings of the sum of its terms' magnitudes T = |s| (|A||B| + |bias|) + |aux| + |bias2|:
three for s (acc + bias) + (aux + bias2) in either order (fmaf(s, acc + bias, aux + bias2) or ((s (acc + bias)) + aux) +
bias2), and one for the second-order terms.
"""

import math

import numpy as np
import torch

U24 = 2.0 ** -24                 # fp32 unit roundoff (round to nearest)
U23 = 2.0 ** -23                 # a truncating fp32 adder's unit roundoff
AS_ERR = 1.5e-7                  # Abramowitz-Stegun 7.1.26: |erf error| <= 1.5e-7
AS_P = 0.3275911
AS_A = (0.254829592, -0.284496736, 1.421413741, -1.453152027, 1.061405429)
TINY = 2.0 ** -126               # smallest normal fp32
C_PDF = 1.0 / math.sqrt(2.0 * math.pi)

INT_MAX = 3                      # operands are integers in [-INT_MAX, INT_MAX]
QUARTER_LIMIT = 2.0 ** 12        # bias, bias2, aux: multiples of 1/4 below this in magnitude
SCALE_EXP = (-2, 2)              # row_scale = +-2^j, j in this closed range


# ---- exact-regime operand generators ------------------------------------------------------------------------------
def _gen(seed):
    return torch.Generator(device='cpu').manual_seed(seed)


def int_operand(shape, seed):
    """integers in [-3, 3] (float32 on the CPU; exact in bf16)"""
    return torch.randint(-INT_MAX, INT_MAX + 1, shape, generator=_gen(seed)).float()


def quarter_values(shape, seed, limit=256.0):
    """multiples of 1/4 with magnitude below `limit` (<= QUARTER_LIMIT)"""
    assert limit <= QUARTER_LIMIT
    q = int(limit * 4) - 1
    return torch.randint(-q, q + 1, shape, generator=_gen(seed)).float() / 4


def pow2_scale(n, seed):
    """+-2^j, j uniform in SCALE_EXP"""
    g = _gen(seed)
    j = torch.randint(SCALE_EXP[0], SCALE_EXP[1] + 1, (n,), generator=g)
    sign = torch.randint(0, 2, (n,), generator=g) * 2 - 1
    return sign.float() * torch.pow(2.0, j.float())


def _on_grid(t, res):
    t = t.double().cpu()
    return bool(torch.equal(torch.round(t / res) * res, t))


def exact_premise(K, bias=None, bias2=None, aux=None, row_scale=None, amax=INT_MAX, bmax=INT_MAX):
    """Assert that every intermediate of the epilogue is exact in fp32 for these epilogue operands: each tensor is on its
    grid and bounded, and every intermediate's magnitude over its resolution stays below 2^24.  Returns the largest
    magnitude / resolution ratio (log2) for the record."""
    def mx(t):
        return 0.0 if t is None else float(t.double().abs().max()) if t.numel() else 0.0
    for t in (bias, bias2, aux):
        if t is not None:
            assert _on_grid(t, 0.25), 'not a multiple of 1/4'
            assert mx(t) < QUARTER_LIMIT, mx(t)
    smin, smax = 1.0, 1.0
    if row_scale is not None:
        r = row_scale.double().cpu().abs()
        assert bool(torch.equal(torch.exp2(torch.round(torch.log2(r))), r)), 'row_scale not a power of two'
        lo, hi = float(r.min()), float(r.max())
        assert 2.0 ** SCALE_EXP[0] <= lo and hi <= 2.0 ** SCALE_EXP[1], (lo, hi)
        smin, smax = lo, hi
    acc = amax * bmax * K                                      # integer, resolution 1
    res_v = 0.25 if bias is not None else 1.0
    v = acc + mx(bias)                                          # acc + bias
    sv = smax * v                                               # s (acc + bias), resolution res_v * smin
    add = mx(aux) + mx(bias2)                                   # aux + bias2, resolution 1/4
    out = sv + add
    res_out = min(res_v * smin, 0.25 if (aux is not None or bias2 is not None) else 1.0)
    ratios = [acc / 1.0, v / res_v, sv / (res_v * smin), add / 0.25, (sv + mx(aux)) / res_out, out / res_out]
    worst = max(ratios)
    assert worst < 2.0 ** 24, f'exactness premise fails: magnitude / resolution = 2^{math.log2(worst):.2f}'
    return math.log2(max(worst, 1.0))


# ---- rounding -----------------------------------------------------------------------------------------------------
def bf16_rne_bits(x):
    """float32 tensor -> int16 bit patterns of its bf16 round-to-nearest-even (NaN -> quiet NaN of the same sign)"""
    assert x.dtype == torch.float32
    u = x.view(torch.int32).long() & 0xFFFFFFFF
    r = (u + 0x7FFF + ((u >> 16) & 1)) >> 16
    nan = torch.isnan(x)
    r = torch.where(nan, (u >> 16) | 0x0040, r) & 0xFFFF
    return ((r ^ 0x8000) - 0x8000).to(torch.int16)


def round_once(x64, dtype):
    """the float64 value of an exact-regime output rounded once to `dtype` (float32 or bfloat16); asserts it is exact in
    fp32 first, so that the bf16 rounding from fp32 is the rounding of the exact value"""
    f = x64.float()
    assert bool(torch.equal(f.double(), x64)), 'exact-regime value not representable in fp32'
    if dtype == torch.float32:
        return f
    return bf16_rne_bits(f).view(torch.bfloat16)


def bf16_half_ulp(x):
    """half the bf16 spacing at |x| (float64 tensor or array): 2^(e - 8) for |x| in [2^e, 2^(e+1)), 2^-134 below 2^-126"""
    if isinstance(x, torch.Tensor):
        e = torch.floor(torch.log2(x.double().abs().clamp(min=TINY)))
        return torch.exp2(e - 8)
    a = np.abs(np.asarray(x, dtype=np.float64))
    e = np.floor(np.log2(np.maximum(a, TINY)))
    return np.ldexp(1.0, (e - 8).astype(np.int64))


# ---- GELU reference and bounds ------------------------------------------------------------------------------------
def gelu64(z):
    from scipy.special import erf
    z = np.asarray(z, dtype=np.float64)
    return 0.5 * z * (1.0 + erf(z / math.sqrt(2.0)))


def dgelu64(z):
    from scipy.special import erf
    z = np.asarray(z, dtype=np.float64)
    return 0.5 * (1.0 + erf(z / math.sqrt(2.0))) + z * C_PDF * np.exp(-0.5 * z * z)


def erf_fast_error(z, as_err=AS_ERR):
    """E_erf(z): bound on |computed erf_fast_pos(|z| / sqrt 2) - erf(|z| / sqrt 2)| (module docstring)"""
    x = np.abs(np.asarray(z, dtype=np.float64)) / math.sqrt(2.0)
    with np.errstate(over='ignore', invalid='ignore'):
        y = x * x
        t = 1.0 / (1.0 + AS_P * x)
        S = sum(abs(a) * t ** (i + 1) for i, a in enumerate(AS_A))
        e = np.exp(-y)
        eps_e = (2.0 + np.floor(1.173 * y)) * U23 + 5.0 * U24 * y
        e_eps = np.where(e > 0, e * eps_e, 0.0)                 # e eps_e -> 0 where y is huge
        xe = np.where(e > 0, x * e, 0.0)
    return as_err + U24 + 16.0 * U24 * S * e + S * (e_eps + TINY) + (2.0 / math.sqrt(math.pi)) * xe * 2.0 * U24


def gelu_bound(z, ref=None, as_err=AS_ERR):
    """per-element bound on |bf16 gelu_fast(z) - gelu(z)| for finite z"""
    z = np.asarray(z, dtype=np.float64)
    ref = gelu64(z) if ref is None else ref
    err32 = 0.5 * np.abs(z) * erf_fast_error(z, as_err) + 2.0 * U24 * np.abs(ref)
    return err32 + bf16_half_ulp(np.abs(ref) + err32)


def dgelu_bound(z, ref=None, as_err=AS_ERR):
    """per-element bound on |bf16 dgelu_fast(z) - gelu'(z)| for finite z (dh = 1)"""
    z = np.asarray(z, dtype=np.float64)
    ref = dgelu64(z) if ref is None else ref
    x = np.abs(z) / math.sqrt(2.0)
    with np.errstate(over='ignore', invalid='ignore'):
        y = x * x
        e = np.exp(-y)
        eps_e = (2.0 + np.floor(1.173 * y)) * U23 + 5.0 * U24 * y
        pdf = np.where(e > 0, np.abs(z) * C_PDF * e * (eps_e + 3.0 * U24), 0.0)
    err32 = 0.5 * erf_fast_error(z, as_err) + pdf + np.abs(z) * C_PDF * TINY + 2.0 * U24 * (1.0 + np.abs(ref))
    return err32 + bf16_half_ulp(np.abs(ref) + err32)


# ---- random-operand bound -----------------------------------------------------------------------------------------
def accumulation_bound(K, absprod, scale=None, epi_terms=None, splits=1, bf16_ref=None):
    """Per-element bound on |got - ref| of a GEMM with Gaussian operands (module docstring).
    absprod: (|A||B|)_mn in float64; scale: |s| per row [M, 1] or None; epi_terms: T = |s| (|A||B| + |bias|) + |aux| +
    |bias2| (float64, broadcastable), None for a bare fp32 accumulator; bf16_ref: |reference| when the output is bf16."""
    s = 1.0 if scale is None else scale
    acc = (K + splits - 1) * U23 * absprod * s
    b = acc * (1.0 + 4.0 * U24)
    if epi_terms is not None:
        b = b + 4.0 * U24 * epi_terms
    if bf16_ref is not None:
        b = b + bf16_half_ulp(bf16_ref + b)
    return b
