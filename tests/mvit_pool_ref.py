"""fp64 reference and per-element error bounds for the q/k/v pooling kernels of csrc/vt_mvit.cu.  CPU only.

The pooling is a depthwise 3x3x3 Conv3d (padding 1, strided) over the (T, H, W) token grid of each head plus
LayerNorm(96); the cls row bypasses the convolution.  Every stage is compared with fp64 computed from the kernel's own
fp32 outputs of the stage before it (pooled, mean, rstd, and the dpooled scratch), so errors do not compound and each
bound covers only the arithmetic of one stage.  With u = 2^-24 and gamma_n = n u / (1 - n u), a sum of n fp32 roundings
is within gamma_n of the sum of the absolute values of its terms, in any order of summation:

  pooled   gamma_n sum|w x| over the n <= 27 taps in range; the cls row is an exact copy
  mean     gamma_97 mean|pooled|: 95 additions, the rounded 1/96 and the product (gamma_{D+1} at width D)
  rstd     gamma_101 (gamma_{D+5}) on mean((x - mean_k)^2) + eps (squares, sum, scale, eps), the kernel's own mean error delta entering as
           (1 + delta^2 / (var + eps)), and the 2 ulp of rsqrtf
  out      gamma_4 |xhat gamma| + u |beta|, then half a bf16 ulp
  dpooled  first-order LayerNorm backward with absolute sums (see ln_backward_bound)
  din      gamma_27 sum|dp w| over the covering taps, then half a bf16 ulp; exactly +0 where no window covers the token
  dw       gamma_n sum|dp x|, n = rows one thread accumulates + slot sums + per-CTA partials (dw_plan)
  dgamma   gamma_n sum|d xhat|, n = rows per warp + 8 warps + per-CTA partials (+2 for xhat's own roundings); dbeta alike

The first-order bounds drop products of two gammas, each below 1e-5 at these sizes; SECOND_ORDER covers them.
"""
import math

import torch
import torch.nn.functional as F
from torch.nn.grad import conv3d_input, conv3d_weight

HD = 96
U = 2.0 ** -24                      # fp32 unit roundoff
RSQRT_REL = 2.0 ** -22              # rsqrtf: at most 2 ulp, an ulp being at most 2^-23 of the result
SECOND_ORDER = 1 + 2.0 ** -10
EPS = 1e-5                          # pool_norm_eps of maskfeat_config
EPS32 = float(torch.tensor(EPS, dtype=torch.float32))
INV_HD32 = torch.tensor(1.0 / HD, dtype=torch.float32)   # the kernels' 1.0f / 96
ROW_WARPS = 8                       # rows per CTA step of ln_small_bwd_kernel
DW_MIN_ROWS_GEN1 = 64               # pool_dw_kernel: rows per CTA at least
DW_MIN_ROWS_GEN2 = 8                # pool_dw_v2_kernel
DW_SLOTS = 4                        # pool_dw_v2_kernel: rows in flight per CTA, summed at the end


def gamma(n):
    n = torch.as_tensor(n, dtype=torch.float64)
    return n * U / (1 - n * U)


def half_ulp_bf16(a):
    """half a bf16 ulp at magnitude a >= 0: the rounding error bound of bf16(v) for |v| <= a"""
    a = a.double()
    _, e = torch.frexp(a)                                       # a in [2^(e-1), 2^e): bf16 ulp 2^(e-8)
    return torch.where(a > 0, torch.pow(2.0, (e - 9).double()), torch.zeros_like(a))


def out_thw(thw, stride):
    return tuple((n - 1) // s + 1 for n, s in zip(thw, stride))


def config_shapes(img_size=224, num_frames=16):
    """(thw, stride, heads) of every q / k / v pooling of the MViT-B blocks that maskfeat_config builds, without repeats"""
    from oracle.mvit_oracle import maskfeat_config
    cfg = maskfeat_config(img_size=img_size, num_frames=num_frames)
    thw, shapes = tuple(cfg['thw']), []
    for blk in cfg['blocks']:
        assert blk['dim'] // blk['heads'] == HD and blk['kernel_kv'] == [3, 3, 3]
        for s in (blk['stride_q'], blk['stride_kv']):
            if s and (thw, tuple(s), blk['heads']) not in shapes:
                shapes.append((thw, tuple(s), blk['heads']))
        if blk['stride_q']:
            thw = out_thw(thw, blk['stride_q'])
    return shapes


LAYOUTS = (0, 1, 2, 'contig')       # slot of a fused [B*N, 3, H*96] q/k/v projection, or a contiguous [B*N, H*96] tensor

# (thw, stride, heads, batch, layout, regime)
CONFIG_CASES = [(thw, s, h, 1, LAYOUTS[i % 4], 'randn') for i, (thw, s, h) in enumerate(config_shapes())]
EDGE_CASES = [
    # Hin, Win mod s in {0, 1, s - 1} for s = 2, 4, 8
    ((2, 8, 9), (1, 2, 2), 2, 3, 0, 'randn'),
    ((3, 9, 8), (1, 2, 2), 1, 1, 1, 'offset'),
    ((2, 16, 17), (1, 4, 4), 8, 1, 2, 'randn'),
    ((2, 19, 16), (1, 4, 4), 1, 3, 'contig', 'randn'),
    ((2, 17, 19), (2, 4, 4), 2, 1, 0, 'randn'),
    ((2, 16, 23), (1, 8, 8), 1, 3, 1, 'randn'),
    ((1, 17, 24), (1, 8, 8), 2, 1, 2, 'offset'),
    ((2, 23, 17), (1, 8, 8), 8, 1, 'contig', 'randn'),
    # T = 1; T = 2 and 3 with st = 2
    ((1, 6, 7), (1, 2, 2), 2, 3, 0, 'randn'),
    ((2, 5, 5), (2, 2, 2), 1, 3, 1, 'randn'),
    ((3, 4, 6), (2, 1, 1), 2, 1, 'contig', 'randn'),
    # 1x1 spatial grids
    ((4, 1, 1), (1, 1, 1), 8, 3, 2, 'randn'),
    ((3, 1, 1), (2, 2, 2), 1, 1, 0, 'randn'),
    # 64 per axis, the largest grid the backward takes
    ((2, 64, 64), (1, 8, 8), 1, 1, 1, 'randn'),
    ((64, 2, 3), (2, 1, 2), 2, 1, 'contig', 'randn'),
    ((1, 64, 5), (1, 2, 1), 1, 3, 2, 'offset'),
]
CASES = CONFIG_CASES + EDGE_CASES


def case_id(c):
    thw, s, h, b, layout, regime = c
    return f'{"x".join(map(str, thw))}-s{"".join(map(str, s))}-H{h}-B{b}-{layout}-{regime}'


def make_inputs(B, H, thw, stride, regime='randn', seed=0):
    """-> x bf16 [B, 1+T*Hin*Win, H*96], w fp32 [96, 27], gamma, beta fp32 [96], dout fp32 [B, H, 1+Lo, 96].
    regime 'offset': inputs near 1 and filters near 0.1, so pooled rows have a mean about 100 times their spread"""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, 1 + math.prod(thw), H * HD, generator=g)
    w = torch.randn(HD, 27, generator=g)
    if regime == 'offset':
        x, w = 1 + 0.05 * x, 0.1 + 0.002 * w
    else:
        w = 0.3 * w
    gam, bet = 1 + 0.1 * torch.randn(HD, generator=g), 0.1 * torch.randn(HD, generator=g)
    dout = torch.randn(B, H, 1 + math.prod(out_thw(thw, stride)), HD, generator=g)
    return x.bfloat16(), w, gam, bet, dout


def heads(x, H):
    """[B, N, H*96] -> [B, H, N, 96] fp64"""
    B, N, _ = x.shape
    return x.double().reshape(B, N, H, HD).permute(0, 2, 1, 3)


def _vol(body, thw):
    """[B, H, L, 96] -> [B*H, 96, T, Hin, Win]"""
    B, H, _, _ = body.shape
    return body.reshape(B * H, *thw, HD).permute(0, 4, 1, 2, 3)


def _rows(vol, B, H):
    """[B*H, 96, To, Ho, Wo] -> [B, H, Lo, 96]"""
    return vol.reshape(B, H, HD, -1).transpose(2, 3)


def _w5(w):
    return w.double().reshape(HD, 1, 3, 3, 3)


def conv(body, w, thw, stride):
    B, H = body.shape[:2]
    return _rows(F.conv3d(_vol(body, thw), _w5(w), stride=tuple(stride), padding=1, groups=HD), B, H)


def conv_adjoint(dbody, w, thw, stride):
    """gradient of conv() w.r.t. its input: [B, H, Lo, 96] -> [B, H, L, 96]"""
    B, H = dbody.shape[:2]
    g = conv3d_input((B * H, HD, *thw), _w5(w), _vol(dbody, out_thw(thw, stride)), stride=tuple(stride), padding=1, groups=HD)
    return _rows(g, B, H)


def conv_wgrad(body, dbody, thw, stride):
    """gradient of conv() w.r.t. its filter: -> [96, 27]"""
    g = conv3d_weight(_vol(body, thw), (HD, 1, 3, 3, 3), _vol(dbody, out_thw(thw, stride)), stride=tuple(stride), padding=1,
                      groups=HD)
    return g.reshape(HD, 27)


def taps_in_range(thw, stride):
    """[Lo] number of the 27 taps of each output window that fall inside the grid"""
    one = torch.ones(1, 1, *thw, dtype=torch.float64)
    return F.conv3d(one, torch.ones(1, 1, 3, 3, 3, dtype=torch.float64), stride=tuple(stride), padding=1).reshape(-1)


def covered(thw, stride):
    """[L] bool: the input token lies in at least one output window"""
    n = conv3d_input((1, 1, *thw), torch.ones(1, 1, 3, 3, 3, dtype=torch.float64),
                     torch.ones(1, 1, *out_thw(thw, stride), dtype=torch.float64), stride=tuple(stride), padding=1)
    return n.reshape(-1) > 0


def pool_forward(xh, w, thw, stride, gam=None, bet=None):
    """fp64 pooling of xh [B, H, 1+L, 96] (cls row copied); with gam / bet also the LayerNorm -> (pooled, out or None)"""
    pooled = torch.cat([xh[:, :, :1], conv(xh[:, :, 1:], w, thw, stride)], 2)
    out = None if gam is None else F.layer_norm(pooled, (HD,), gam.double(), bet.double(), EPS)
    return pooled, out


def ln_plan(rows, sm_count):
    """(CTAs, rows per warp) of every LayerNorm kernel over `rows` rows: 8 warps per CTA, one row per warp and step, at
    most 4 CTAs per SM (vt_ln_bwd_blocks; ln_blocks of the D % 128 == 0 kernels, row_blocks(rows, 4) of the narrow
    forward)"""
    blocks = max(1, min((rows + ROW_WARPS - 1) // ROW_WARPS, 4 * sm_count))
    return blocks, -(-rows // (ROW_WARPS * blocks))


def dw_plan(rows_conv, gen, sm_count):
    """(CTAs, rows per CTA) of the filter-gradient kernel of generation `gen` over rows_conv pooled rows (vt_pool_bwd)"""
    blocks = max(1, min(-(-rows_conv // DW_MIN_ROWS_GEN2), 2 * sm_count))
    if gen == 1:
        blocks = min(blocks, -(-rows_conv // DW_MIN_ROWS_GEN1))
    rpc = -(-rows_conv // blocks)
    return -(-rows_conv // rpc), rpc


class Report(dict):
    """worst error / bound ratio per output"""

    def add(self, name, ratio):
        self[name] = max(self.get(name, 0.0), ratio)

    def __str__(self):
        return ', '.join(f'{k} {v:.3f}' for k, v in self.items())


def check(name, got, ref, bound, report):
    """|got - ref| <= bound element by element (a zero bound demands equality); NaN or inf fails"""
    got = got.double()
    assert got.shape == ref.shape, (name, tuple(got.shape), tuple(ref.shape))
    bad = ~torch.isfinite(got)
    assert not bool(bad.any()), f'{name}: {int(bad.sum())} elements not finite, first at {bad.nonzero()[0].tolist()}'
    bound = bound.expand_as(ref)
    err = (got - ref).abs()
    ratio = torch.where(err == 0, torch.zeros_like(err), err / bound)
    i = int(ratio.argmax())
    worst = float(ratio.reshape(-1)[i])
    if worst > 1:
        at = list(torch.unravel_index(torch.tensor(i), ref.shape))
        raise AssertionError(f'{name}: error {float(err.reshape(-1)[i]):.4e} against bound {float(bound.reshape(-1)[i]):.4e} '
                             f'at {[int(a) for a in at]} (got {float(got.reshape(-1)[i]):.8e}, fp64 {float(ref.reshape(-1)[i]):.8e}); '
                             f'{int((ratio > 1).sum())} elements out of bound')
    report.add(name, worst)


def check_forward(xh, w, gam, bet, thw, stride, got, report):
    """xh [B, H, 1+L, 96] fp64 inputs; got: the kernel's pooled (fp32), mean, rstd ([B, H, 1+Lo]) and out (bf16)"""
    pooled_ref, _ = pool_forward(xh, w, thw, stride)
    absum = torch.cat([torch.zeros_like(xh[:, :, :1]), conv(xh[:, :, 1:].abs(), w.abs(), thw, stride)], 2)
    taps = torch.cat([torch.zeros(1, dtype=torch.float64), taps_in_range(thw, stride)])
    check('pooled', got['pooled'], pooled_ref, gamma(taps)[:, None] * absum, report)
    check_ln_forward(got['pooled'].double(), got['mean'], got['rstd'], gam, bet, EPS, got['out'], report)


def check_ln_forward(p, mu, rs, gam, bet, eps, out, report, names=('mean', 'rstd', 'out')):
    """LayerNorm forward over the last dim (any width D) of the fp32 rows p (fp64 tensor [..., D]): the kernel's mean and
    rstd against fp64, and its output (bf16, or fp32) against fp64 computed from the kernel's own mean and rstd.  The
    kernels sum D terms, scale by the rounded 1/D (mean: gamma_{D+1}), and for rstd square D rounded differences, sum, scale
    and add eps (gamma_{D+5}); out is (x - mean) * rstd * gamma + beta (gamma_4, u |beta|)."""
    D = p.shape[-1]
    mu, rs = mu.double(), rs.double()
    mean = p.mean(-1)
    check(names[0], mu, mean, gamma(D + 1) * p.abs().mean(-1), report)
    var = (p - mean[..., None]).square().mean(-1)
    a = var + float(torch.tensor(eps, dtype=torch.float32))
    q = 1 + (mu - mean).square() / a
    g = gamma(D + 5)
    rstd = a.rsqrt()
    rel = torch.maximum((q * (1 - g)).rsqrt() * (1 + RSQRT_REL) - 1, 1 - (q * (1 + g)).rsqrt() * (1 - RSQRT_REL))
    check(names[1], rs, rstd, rstd * rel, report)
    xg = (p - mu[..., None]) * rs[..., None] * gam.double()
    ref = xg + bet.double()
    e32 = gamma(4) * xg.abs() + U * bet.double().abs()
    if out.dtype == torch.bfloat16:
        e32 = e32 + half_ulp_bf16(ref.abs() + e32)
    check(names[2], out, ref, e32, report)


def ln_backward(p, mu, rs, gam, dout):
    """closed-form LayerNorm backward with the kernel's mean / rstd -> (dpooled, xhat, gy, m1, m2)"""
    xhat = (p - mu[..., None]) * rs[..., None]
    gy = dout.double() * gam.double()
    m1 = gy.mean(-1, keepdim=True)
    m2 = (gy * xhat).mean(-1, keepdim=True)
    return rs[..., None] * (gy - m1 - xhat * m2), xhat, gy, m1, m2


def ln_backward_bound(rs, xhat, gy, m1, m2):
    """first order, rows of width D: gy rounded (u), m1 from D rounded terms (gamma_{D+2}), m2 from terms with xhat's two
    roundings (gamma_{D+5}), xhat itself (gamma_2), the product and two subtractions and the final scaling (gamma_4)"""
    D = gy.shape[-1]
    return rs[..., None] * (U * gy.abs() + gamma(D + 2) * gy.abs().mean(-1, keepdim=True)
                            + gamma(D + 5) * xhat.abs() * (gy * xhat).abs().mean(-1, keepdim=True)
                            + gamma(2) * m2.abs() * xhat.abs()
                            + gamma(4) * (gy.abs() + m1.abs() + (xhat * m2).abs())) * SECOND_ORDER


def check_backward(xh, w, gam, thw, stride, fwd, dout, got, gen, sm_count, report, parts=('dpooled', 'din', 'dw', 'dgb')):
    """fwd: the kernel's pooled / mean / rstd; got: its dpooled scratch [B, H, 1+Lo, 96], din (bf16 [B, H, 1+L, 96]), dw
    [96, 27], dgamma, dbeta; gen: the generation whose dw is checked"""
    B, H = xh.shape[:2]
    p, mu, rs = fwd['pooled'].double(), fwd['mean'].double(), fwd['rstd'].double()
    d = dout.double()
    dp_ref, xhat, gy, m1, m2 = ln_backward(p, mu, rs, gam, d)
    if 'dpooled' in parts:
        check('dpooled', got['dpooled'], dp_ref, ln_backward_bound(rs, xhat, gy, m1, m2), report)
    dp = got['dpooled'].double()
    if 'din' in parts:
        din_ref = torch.cat([dp[:, :, :1], conv_adjoint(dp[:, :, 1:], w, thw, stride)], 2)
        absum = torch.cat([torch.zeros_like(dp[:, :, :1]), conv_adjoint(dp[:, :, 1:].abs(), w.abs(), thw, stride)], 2)
        e32 = gamma(27) * absum
        check('din', got['din'], din_ref, e32 + half_ulp_bf16(din_ref.abs() + e32), report)
        bits = got['din'][:, :, 1:][:, :, ~covered(thw, stride)].contiguous().view(torch.int16)
        assert not bool(bits.any()), f'din: {int((bits != 0).sum())} elements of tokens no window covers are not +0'
    if 'dw' in parts:
        rows_conv = B * H * (p.shape[2] - 1)
        blocks, rpc = dw_plan(rows_conv, gen, sm_count)
        n = rpc + DW_SLOTS + blocks
        check('dw', got['dw'], conv_wgrad(xh[:, :, 1:], dp[:, :, 1:], thw, stride),
              gamma(n) * conv_wgrad(xh[:, :, 1:].abs(), dp[:, :, 1:].abs(), thw, stride), report)
    if 'dgb' in parts:
        check_dgamma_dbeta(d, xhat, got['dgamma'], got['dbeta'], sm_count, report)


def check_dgamma_dbeta(d, xhat, dgamma, dbeta, sm_count, report):
    """d, xhat fp64 [..., D] over every row the backward walked; a warp adds its rows' d * xhat and d per column, the 8
    warps of a CTA are summed, then the CTAs' partial rows: n = rows per warp + 8 warps + CTAs (ln_plan), +2 for xhat's
    own roundings"""
    d, xhat = d.reshape(-1, d.shape[-1]), xhat.reshape(-1, d.shape[-1])
    blocks, per_warp = ln_plan(d.shape[0], sm_count)
    n = per_warp + ROW_WARPS + blocks
    check('dgamma', dgamma, (d * xhat).sum(0), gamma(n + 2) * (d * xhat).abs().sum(0), report)
    check('dbeta', dbeta, d.sum(0), gamma(n) * d.abs().sum(0), report)
