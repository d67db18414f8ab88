"""fp64 references and per-element bounds for the row-wise kernels between the GEMMs: LayerNorm forward / backward
(csrc/vt_elementwise.cu for D % 128 == 0, the narrow ln_small_* kernels of csrc/vt_mvit.cu for D = 32 ... 224), the dY
producers that also emit column sums (gather_cast_colsum, dgelu_colsum), colsum, reduce_rows and cls_rows.  CPU only.

The LayerNorm bounds are those of tests/mvit_pool_ref.py at any width (check_ln_forward, ln_backward, ln_backward_bound,
check_dgamma_dbeta with the row plan ln_plan).  This module adds, with u = 2^-24 and gamma_n = n u / (1 - n u):

  dx        the LayerNorm backward row plus the residual dres (one more rounding); rows sent to dx_aux get no residual
  colsums   gamma_n sum|v| per column over the kernel's own bf16 rows v, n = the longest chain of additions in the kernel's
            partition of the rows (colsum_n, gcc_plan, gbc_plan).  A bound with n = M rows (7e-4 relative at 12.5k rows)
            could not tell sums of the bf16 rows from sums of the fp32 values they were rounded from; these n are ~100.
  reduce    out (+)= scale * sum_s in[s]: gamma_{depth + 2} over |scale| sum|in| (+ |out| when accumulating)
  cls_rows  src + scale * sum_t extra[t]: gamma_T; the plain copy (no extra) is exact
"""
import torch

from tests import mvit_pool_ref as P

U, gamma, check, Report = P.U, P.gamma, P.check, P.Report
check_ln_forward, ln_backward, ln_backward_bound, check_dgamma_dbeta, ln_plan = (
    P.check_ln_forward, P.ln_backward, P.ln_backward_bound, P.check_dgamma_dbeta, P.ln_plan)

ROW_WARPS = P.ROW_WARPS              # rows per CTA step of every warp-per-row kernel
LN_CTAS_PER_SM = 4                   # ln_blocks / row_blocks(rows, 4) / vt_ln_bwd_blocks
COLSUM_ROWS = 512                    # colsum_kernel: rows per chunk, walked by 8 row lanes
GCC_CTAS_PER_SM = 2                  # vt_gather_cast_colsum_blocks
GBC_CTAS_PER_SM, GBC_UNROLL = 4, 2   # vt_gelu_bwd_colsum_blocks: 2 rows per CTA step
RT_TALL_MIN, RT_LANES = 32, 64       # reduce_rows: tall kernel from 32 partial rows, 64 row lanes, then 16 + 4 lanes

LN_WIDTHS = [128 * v for v in range(1, 9)]          # ln_fwd_kernel / ln_bwd_kernel / ln_bwd2_kernel, V = 1 .. 8
LN_SMALL_WIDTHS = [32, 64, 96, 160, 192, 224]       # ln_small_*: D % 128 != 0
REGIMES = ('randn', 'offset', 'constant', 'outlier', 'tiny')


def cdiv(a, b):
    return -(-a // b)


def ln_cap(sm_count):
    """the CTA cap of the LayerNorm kernels: beyond 8 * cap rows a warp walks more than one row"""
    return LN_CTAS_PER_SM * sm_count


def reduce_depth(S):
    """additions on the longest path of reduce_rows over S partial rows: in order (flat kernel), or one row lane's
    ceil(S / 64) rows, 4 lanes, then 16 (tall kernel)"""
    return S if S < RT_TALL_MIN else cdiv(S, RT_LANES) + 3 + 15


def colsum_n(M, counters=True):
    """n of the colsum bound over M rows: rows per row lane + 8 lanes + the chunk partials (summed in order by the last CTA,
    or by reduce_rows in the two-launch form)"""
    chunks = cdiv(M, COLSUM_ROWS)
    return cdiv(min(M, COLSUM_ROWS), ROW_WARPS) + ROW_WARPS + (chunks if counters else reduce_depth(chunks))


def gcc_plan(rows, sm_count):
    """(CTAs, rows per warp, n) of gather_cast_colsum_kernel: 8 warps, one row per warp and step, then reduce_rows"""
    blocks = max(1, min(cdiv(rows, ROW_WARPS), GCC_CTAS_PER_SM * sm_count))
    per_warp = cdiv(rows, ROW_WARPS * blocks)
    return blocks, per_warp, per_warp + ROW_WARPS + reduce_depth(blocks)


def gbc_plan(M, sm_count):
    """(CTAs, rows per thread, n) of gelu_bwd_colsum_kernel: a thread adds 2 rows per step of its CTA, then reduce_rows"""
    blocks = max(1, min(cdiv(M, GBC_UNROLL), GBC_CTAS_PER_SM * sm_count))
    per_thread = GBC_UNROLL * cdiv(M, GBC_UNROLL * blocks)
    return blocks, per_thread, per_thread + reduce_depth(blocks)


def check_colsum(name, got, rows, n, report):
    """got fp32 [N] against the fp64 column sums of rows ([M, N], the kernel's own bf16 output), within gamma_n sum|v|"""
    v = rows.double()
    check(name, got, v.sum(0), gamma(n) * v.abs().sum(0), report)


def check_ln_backward(xs, mu, rs, gam, dy, dx_rows, res_rows, report, name='dx'):
    """xs fp64 [rows, D]: the x rows the backward read (in_row applied); mu / rs the kernel's statistics; dy as given (fp32
    or bf16); dx_rows [rows, D]: the kernel's dx row of every m (from dx or dx_aux); res_rows: the residual added to row m
    (fp64, zeros where none) and a mask of the rows that got one, or None.  Returns (d, xhat) for check_dgamma_dbeta."""
    d = dy.double()
    ref, xhat, gy, m1, m2 = ln_backward(xs, mu.double(), rs.double(), gam, d)
    bound = ln_backward_bound(rs.double(), xhat, gy, m1, m2)
    if res_rows is not None:
        res, has = res_rows
        ref = ref + res
        bound = bound + has[:, None] * U * (ref.abs() + bound)
    check(name, dx_rows, ref, bound, report)
    return d, xhat


def reduce_rows_ref(inp, n, scale, prior=None):
    """inp fp32 [S, stride] -> (ref, bound) of vt_reduce_rows over the first n columns; prior: the output's value before an
    accumulating call"""
    v = inp[:, :n].double()
    s = float(torch.tensor(scale, dtype=torch.float32))
    ref = s * v.sum(0)
    mag = abs(s) * v.abs().sum(0)
    if prior is not None:
        ref = ref + prior.double()
        mag = mag + prior.double().abs()
    return ref, gamma(reduce_depth(inp.shape[0]) + 2) * mag


def cls_rows_ref(src, extra, scale):
    """(ref, bound) of vt_cls_rows: src [B, D] + scale * extra [B, T, D].sum(1) (scale as the kernel's fp32); no extra:
    the copy, bound 0 (bit for bit)"""
    ref = src.double()
    if extra is None:
        return ref, torch.zeros_like(ref)
    s = float(torch.tensor(scale, dtype=torch.float32))
    e = extra.double()
    ref = ref + s * e.sum(1)
    return ref, gamma(e.shape[1]) * (abs(s) * e.abs().sum(1) + src.double().abs())


def make_rows(n, D, regime, seed):
    """fp32 [n, D] LayerNorm inputs.  offset: mean 500 times the spread (the rstd bound's mean-error term matters);
    constant: every row one value (variance 0: rstd = eps^-1/2, xhat within bound of 0); outlier: one element per row 1000
    times the rest; tiny: spread 1e-6 around a value of order 1 (variance far below eps)"""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(n, D, generator=g)
    c = 3 * torch.randn(n, 1, generator=g)
    if regime == 'offset':
        x = 500 + x
    elif regime == 'constant':
        x = c.expand(n, D).clone()
    elif regime == 'outlier':
        j = torch.randint(0, D, (n,), generator=g)
        x[torch.arange(n), j] = 1000 * torch.sign(c[:, 0] + 1e-3)
    elif regime == 'tiny':
        x = c + 1e-6 * x
    return x.contiguous()


def make_affine(D, seed):
    """gamma with exact zeros and negative entries, beta of order 0.1"""
    g = torch.Generator().manual_seed(seed)
    gam = 1 + 0.5 * torch.randn(D, generator=g)
    gam[::7] = 0
    gam[3::11] = -gam[3::11].abs()
    return gam, 0.1 * torch.randn(D, generator=g)
