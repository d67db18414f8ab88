"""CPU walk-through of the index arithmetic and tiling of the MViT CUDA kernels (csrc/vt_mvit.cu) and of the tensor-core flash
attention (csrc/vt_attention_mma.cu, modelled in tests/attn_mma_emu.py).

There is no GPU in the build container, so the kernels' *algorithms* — row decoding, gather conditions of the adjoint
kernels, tile masking, log2-domain softmax bookkeeping — are transcribed loop-for-loop into numpy here and compared
with the contract emulation (tests/emu_kernels.py, itself checked against the reference goldens).  This does not
execute device code; the -m gpu tests do.  It exists to catch index/formula mistakes before spending GPU time.
"""
import numpy as np
import pytest
import torch

from tests import attn_mma_emu as AE
from tests.emu_kernels import EmuKernels

HD = 96
LOG2E = 1.4426950408889634
LN2 = 0.6931471805599453


def rel(a, b):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    return float(np.linalg.norm(a - b) / (np.linalg.norm(b) + 1e-30))


def out_dims(thw, stride):
    return tuple((n + 2 - 3) // s + 1 for n, s in zip(thw, stride))


# ---- pool_ln_fwd_kernel / pool_din_kernel / pool_dw_kernel ------------------------------------------
def sim_pool_fwd(inp, in_bs, in_rs, w, B, H, thw, stride):
    T, Hin, Win = thw
    st, sh, sw = stride
    To, Ho, Wo = out_dims(thw, stride)
    Lo1 = 1 + To * Ho * Wo
    pooled = np.zeros((B * H * Lo1, HD))
    for r in range(B * H * Lo1):
        bh = r // Lo1
        l = r - bh * Lo1
        b = bh // H
        h = bh - b * H
        base = b * in_bs + h * HD
        if l == 0:
            pooled[r] = inp[base:base + HD]
            continue
        o = l - 1
        o2 = o // Wo
        ow, ot = o - o2 * Wo, o2 // Ho
        oh = o2 - ot * Ho
        hrow, wcol, hok, wok = [0] * 3, [0] * 3, [False] * 3, [False] * 3
        for k in range(3):
            hi, wi = oh * sh - 1 + k, ow * sw - 1 + k
            hok[k], wok[k] = 0 <= hi < Hin, 0 <= wi < Win
            hrow[k], wcol[k] = min(max(hi, 0), Hin - 1), min(max(wi, 0), Win - 1)
        acc = np.zeros(HD)
        for dt in range(3):
            ti = ot * st - 1 + dt
            if ti < 0 or ti >= T:
                continue
            for dh in range(3):
                for dw in range(3):
                    n = 1 + (ti * Hin + hrow[dh]) * Win + wcol[dw]          # clamped address, masked value
                    x = inp[base + n * in_rs: base + n * in_rs + HD]
                    acc += (x if (hok[dh] and wok[dw]) else 0.0) * w[:, (dt * 3 + dh) * 3 + dw]
        pooled[r] = acc
    return pooled.reshape(B, H, Lo1, HD)


def sim_pool_din(dpooled, w, B, H, thw, stride):
    """token-per-warp kernel with per-axis (tap, coordinate) -> output-coordinate tables"""
    T, Hin, Win = thw
    To, Ho, Wo = out_dims(thw, stride)
    L1, Lo1 = 1 + T * Hin * Win, 1 + To * Ho * Wo
    tab = np.full((3, 3, 64), -1, dtype=np.int64)
    for axis, (n_in, s_, n_out) in enumerate(((T, stride[0], To), (Hin, stride[1], Ho), (Win, stride[2], Wo))):
        for k in range(3):
            for c in range(64):
                if c < n_in:
                    nn = c + 1 - k
                    if nn >= 0 and nn % s_ == 0 and nn // s_ < n_out:
                        tab[axis, k, c] = nn // s_
    din = np.zeros((B, L1, H, HD))
    dp_all = dpooled.reshape(B * H, Lo1, HD)
    for tok in range(B * L1):
        b = tok // L1
        n = tok - b * L1
        if n > 0:
            idx = n - 1
            t2 = idx // Win
            wi, ti = idx - t2 * Win, t2 // Hin
            hi = t2 - ti * Hin
            ot3, oh3, ow3 = tab[0, :, ti], tab[1, :, hi], tab[2, :, wi]
        for h in range(H):
            dp = dp_all[b * H + h]
            if n == 0:
                din[b, n, h] = dp[0]
                continue
            acc = np.zeros(HD)
            for dt in range(3):
                if ot3[dt] < 0:
                    continue
                for dh in range(3):
                    if oh3[dh] < 0:
                        continue
                    for dw in range(3):
                        if ow3[dw] < 0:
                            continue
                        acc += dp[1 + (ot3[dt] * Ho + oh3[dh]) * Wo + ow3[dw]] * w[:, (dt * 3 + dh) * 3 + dw]
            din[b, n, h] = acc
    return din.reshape(B, L1, H * HD)


def sim_pool_dw(dpooled, inp, in_bs, in_rs, B, H, thw, stride, rows_per_cta=5, unroll=4):
    """tap-per-warp kernel: CTAs own row ranges, rows are walked `unroll` at a time with clamped duplicates masked."""
    T, Hin, Win = thw
    st, sh, sw = stride
    To, Ho, Wo = out_dims(thw, stride)
    Lo = To * Ho * Wo
    rows = B * H * Lo
    nblocks = (rows + rows_per_cta - 1) // rows_per_cta
    partials = np.zeros((nblocks, HD * 27))
    dp = dpooled.reshape(B * H, Lo + 1, HD)
    for blk in range(nblocks):
        r0, r1 = blk * rows_per_cta, min(rows, (blk + 1) * rows_per_cta)
        for tap in range(27):
            dt, dh, dw = tap // 9, (tap // 3) % 3, tap % 3
            acc = np.zeros(HD)
            rs = min(r0, rows - 1)
            o = rs % Lo
            bh = rs // Lo
            h, b = bh % H, bh // H
            ow, oh, ot = o % Wo, (o // Wo) % Ho, o // (Wo * Ho)
            for rb in range(r0, r1, unroll):
                for u in range(unroll):
                    live = rb + u < r1
                    ti, hi, wi = ot * st - 1 + dt, oh * sh - 1 + dh, ow * sw - 1 + dw
                    ok = live and 0 <= ti < T and 0 <= hi < Hin and 0 <= wi < Win
                    tc, hc, wc = min(max(ti, 0), T - 1), min(max(hi, 0), Hin - 1), min(max(wi, 0), Win - 1)
                    o = (ot * Ho + oh) * Wo + ow
                    g = dp[b * H + h, 1 + o]
                    off = b * in_bs + h * HD + (1 + (tc * Hin + hc) * Win + wc) * in_rs
                    acc += (g if ok else 0.0) * inp[off:off + HD]
                    if rb + u + 1 < r1:                      # odometer advance
                        ow += 1
                        if ow == Wo:
                            ow = 0
                            oh += 1
                            if oh == Ho:
                                oh = 0
                                ot += 1
                                if ot == To:
                                    ot = 0
                                    h += 1
                                    if h == H:
                                        h = 0
                                        b += 1
            partials[blk, np.arange(HD) * 27 + tap] = acc
    return partials.sum(0).reshape(HD, 27)


def sim_pool_din_v2(dpooled, w, B, H, thw, stride):
    """second generation: CTA = one (b, ti) plane x one head (+ one extra plane index for the cls tokens), warp = token;
    (dh, dw) -> output row offsets tabulated per token, the nine taps of a valid time plane gathered together."""
    T, Hin, Win = thw
    To, Ho, Wo = out_dims(thw, stride)
    L1, Lo1 = 1 + T * Hin * Win, 1 + To * Ho * Wo
    tab = np.full((3, 3, 64), -1, dtype=np.int64)
    for axis, (n_in, s_, n_out) in enumerate(((T, stride[0], To), (Hin, stride[1], Ho), (Win, stride[2], Wo))):
        for k in range(3):
            for c in range(n_in):
                nn = c + 1 - k
                if nn >= 0 and nn % s_ == 0 and nn // s_ < n_out:
                    tab[axis, k, c] = nn // s_
    din = np.zeros((B, L1, H, HD))
    dp_all = dpooled.reshape(B * H, Lo1, HD)
    planes = B * T
    for h in range(H):                                   # blockIdx.z
        for plane in range(planes + 1):                  # blockIdx.y
            if plane == planes:
                for b in range(B):
                    din[b, 0, h] = dp_all[b * H + h, 0]
                continue
            b, ti = plane // T, plane % T
            ot3 = tab[0, :, ti]
            t_any = (ot3 >= 0).any()
            dp = dp_all[b * H + h, 1:]                   # rows after the cls row
            for idx in range(Hin * Win):                 # warps of the CTA(s) stride over the plane's tokens
                hi, wi = idx // Win, idx % Win
                rowoff = np.full(9, -1, dtype=np.int64)
                for dh in range(3):
                    for dw in range(3):
                        oh, ow = tab[1, dh, hi], tab[2, dw, wi]
                        if oh >= 0 and ow >= 0:
                            rowoff[dh * 3 + dw] = oh * Wo + ow
                acc = np.zeros(HD)
                if (rowoff >= 0).any() and t_any:
                    for dt in range(3):
                        if ot3[dt] < 0:
                            continue
                        plane_rows = dp[ot3[dt] * Ho * Wo:]
                        for k in range(9):
                            if rowoff[k] >= 0:
                                acc += plane_rows[rowoff[k]] * w[:, dt * 9 + k]
                din[b, 1 + ti * Hin * Win + idx, h] = acc
    return din.reshape(B, L1, H * HD)


def sim_pool_dw_v2(dpooled, inp, in_bs, in_rs, B, H, thw, stride, rows_per_cta=5, slots=4):
    """second generation: warp = (pooled row, time tap): 12 warps per CTA = `slots` row slots x 3 time taps; each lane keeps
    9 taps x 4 channels; the slots are summed in slot order, one partial row per CTA."""
    T, Hin, Win = thw
    st, sh, sw = stride
    To, Ho, Wo = out_dims(thw, stride)
    Lo = To * Ho * Wo
    rows = B * H * Lo
    nblocks = (rows + rows_per_cta - 1) // rows_per_cta
    partials = np.zeros((nblocks, HD * 27))
    dp = dpooled.reshape(B * H, Lo + 1, HD)
    for blk in range(nblocks):
        r0, r1 = blk * rows_per_cta, min(rows, (blk + 1) * rows_per_cta)
        red = np.zeros((slots, HD * 27))
        for slot in range(slots):
            for dt in range(3):
                acc = np.zeros((9, HD))
                for r in range(r0 + slot, r1, slots):
                    bh, o = r // Lo, r % Lo
                    b, h = bh // H, bh % H
                    o2 = o // Wo
                    ow, ot, oh = o - o2 * Wo, o2 // Ho, o2 % Ho
                    ti = ot * st - 1 + dt
                    if ti < 0 or ti >= T:
                        continue
                    g = dp[bh, 1 + o]
                    for dh in range(3):
                        for dw in range(3):
                            hi, wi = oh * sh - 1 + dh, ow * sw - 1 + dw
                            ok = 0 <= hi < Hin and 0 <= wi < Win
                            hc, wc = min(max(hi, 0), Hin - 1), min(max(wi, 0), Win - 1)
                            off = b * in_bs + h * HD + (1 + (ti * Hin + hc) * Win + wc) * in_rs
                            acc[dh * 3 + dw] += (g if ok else 0.0) * inp[off:off + HD]
                for k in range(9):
                    red[slot, np.arange(HD) * 27 + dt * 9 + k] = acc[k]
        partials[blk] = red[0] + red[1] + red[2] + red[3] if slots == 4 else red.sum(0)
    return partials.sum(0).reshape(HD, 27)


@pytest.mark.parametrize('thw,stride,H', [((2, 4, 4), (1, 2, 2), 2), ((3, 5, 6), (1, 4, 4), 1), ((2, 3, 3), (1, 1, 1), 2),
                                          ((2, 8, 8), (1, 8, 8), 1)])
def test_pool_kernels_index_math(thw, stride, H):
    g = torch.Generator().manual_seed(0)
    B = 2
    N1 = 1 + thw[0] * thw[1] * thw[2]
    d = H * HD
    emu = EmuKernels(exact=True, dtype=torch.float64)
    qkv = torch.randn(B * N1, 3 * d, generator=g, dtype=torch.float64)
    src = qkv.view(B, N1, 3 * d)[:, :, d:2 * d]                   # the k slot
    w = torch.randn(HD, 27, generator=g, dtype=torch.float64)
    gamma, beta = torch.randn(HD, generator=g, dtype=torch.float64), torch.randn(HD, generator=g, dtype=torch.float64)
    out, pooled, mean, rstd, othw = emu.pool_fwd(src, H, HD, thw, stride, w, gamma, beta, 1e-5)
    assert tuple(othw) == out_dims(thw, stride)
    flat = qkv.numpy().reshape(-1)
    off = d                                                      # pointer offset of the slot inside the fused buffer
    sim = sim_pool_fwd(flat[off:], N1 * 3 * d, 3 * d, w.numpy(), B, H, thw, stride)
    assert rel(sim, pooled.numpy()) < 1e-12
    dout = torch.randn(pooled.shape, generator=g, dtype=torch.float64)
    dqkv = torch.zeros_like(qkv)
    din = dqkv.view(B, N1, 3 * d)[:, :, d:2 * d]
    dw, dgamma, dbeta = emu.pool_bwd(dout, pooled, mean, rstd, gamma, src, w, din, H, HD, thw, stride)
    # LayerNorm backward in closed form (what ln_small_bwd_kernel computes) feeding the two adjoint kernels
    shp = pooled.shape[:-1] + (1,)
    xh = (pooled - mean.reshape(shp)) * rstd.reshape(shp)
    gy = dout * gamma
    dpooled = rstd.reshape(shp) * (gy - gy.mean(-1, keepdim=True) - xh * (gy * xh).mean(-1, keepdim=True))
    sim_din = sim_pool_din(dpooled.numpy(), w.numpy(), B, H, thw, stride)
    assert rel(sim_din, din.numpy()) < 1e-12
    sim_dw = sim_pool_dw(dpooled.numpy(), flat[off:], N1 * 3 * d, 3 * d, B, H, thw, stride)
    assert rel(sim_dw, dw.numpy()) < 1e-12
    # second generation of the two adjoint kernels (csrc/vt_mvit.cu: pool_din_v2_kernel, pool_dw_v2_kernel)
    assert rel(sim_pool_din_v2(dpooled.numpy(), w.numpy(), B, H, thw, stride), din.numpy()) < 1e-12
    assert rel(sim_pool_dw_v2(dpooled.numpy(), flat[off:], N1 * 3 * d, 3 * d, B, H, thw, stride), dw.numpy()) < 1e-12


# ---- maxpool_fwd_kernel / maxpool_bwd_kernel ---------------------------------------------------------
def sim_maxpool(x, B, D, thw, kernel, stride):
    T, H, W = thw
    kt, kh, kw = kernel
    st, sh, sw = stride
    pt, ph, pw = kt // 2, kh // 2, kw // 2
    To, Ho, Wo = [(n + 2 * (k // 2) - k) // s + 1 for n, k, s in zip(thw, kernel, stride)]
    Lo1, L1 = 1 + To * Ho * Wo, 1 + T * H * W
    y = np.zeros((B, Lo1, D))
    idx = np.zeros((B, Lo1, D), dtype=np.int64)
    for b in range(B):
        for l in range(Lo1):
            if l == 0:
                y[b, 0] = x[b, 0]
                continue
            o = l - 1
            ow, oh, ot = o % Wo, (o // Wo) % Ho, o // (Wo * Ho)
            best = np.full(D, -np.inf)
            arg = np.full(D, 255)
            for dt in range(kt):
                ti = ot * st - pt + dt
                if ti < 0 or ti >= T:
                    continue
                for dh in range(kh):
                    hi = oh * sh - ph + dh
                    if hi < 0 or hi >= H:
                        continue
                    for dw in range(kw):
                        wi = ow * sw - pw + dw
                        if wi < 0 or wi >= W:
                            continue
                        val = x[b, 1 + (ti * H + hi) * W + wi]
                        take = (val > best) | (arg == 255)
                        best = np.where(take, val, best)
                        arg = np.where(take, (dt * kh + dh) * kw + dw, arg)
            y[b, l], idx[b, l] = best, arg
    return y, idx, (To, Ho, Wo)


def sim_maxpool_bwd(dy, idx, B, D, thw, kernel, stride, othw):
    T, H, W = thw
    kt, kh, kw = kernel
    st, sh, sw = stride
    pt, ph, pw = kt // 2, kh // 2, kw // 2
    To, Ho, Wo = othw
    L1 = 1 + T * H * W
    dx = np.zeros((B, L1, D))
    for b in range(B):
        for l in range(L1):
            if l == 0:
                dx[b, 0] = dy[b, 0]
                continue
            i = l - 1
            wi, hi, ti = i % W, (i // W) % H, i // (W * H)
            acc = np.zeros(D)
            for dt in range(kt):
                nt = ti + pt - dt
                if nt < 0 or nt % st != 0:
                    continue
                ot = nt // st
                if ot >= To:
                    continue
                for dh in range(kh):
                    nh = hi + ph - dh
                    if nh < 0 or nh % sh != 0:
                        continue
                    oh = nh // sh
                    if oh >= Ho:
                        continue
                    for dw in range(kw):
                        nw = wi + pw - dw
                        if nw < 0 or nw % sw != 0:
                            continue
                        ow = nw // sw
                        if ow >= Wo:
                            continue
                        at = 1 + (ot * Ho + oh) * Wo + ow
                        acc += np.where(idx[b, at] == (dt * kh + dh) * kw + dw, dy[b, at], 0.0)
            dx[b, l] = acc
    return dx


@pytest.mark.parametrize('thw,stride', [((2, 4, 4), (1, 2, 2)), ((3, 5, 7), (1, 2, 2)), ((4, 6, 6), (2, 2, 2))])
def test_maxpool_kernels_index_math(thw, stride):
    g = torch.Generator().manual_seed(1)
    B, D = 2, 5
    kernel = tuple(s + 1 if s > 1 else s for s in stride)
    x = torch.randn(B, 1 + thw[0] * thw[1] * thw[2], D, generator=g, dtype=torch.float64)
    emu = EmuKernels(exact=True, dtype=torch.float64)
    y, idx_emu, othw = emu.maxpool_fwd(x, thw, kernel, stride)
    ys, idx, othw_s = sim_maxpool(x.numpy(), B, D, thw, kernel, stride)
    assert tuple(othw) == tuple(othw_s)
    assert rel(ys, y.numpy()) == 0.0
    dy = torch.randn(y.shape, generator=g, dtype=torch.float64)
    dx = emu.maxpool_bwd(dy, idx_emu, thw, kernel, stride)
    dxs = sim_maxpool_bwd(dy.numpy(), idx, B, D, thw, kernel, stride, othw_s)
    assert rel(dxs, dx.numpy()) < 1e-14


# ---- im2col3d_kernel -----------------------------------------------------------------------------------
def test_im2col3d_index_math():
    g = torch.Generator().manual_seed(2)
    B, T, C, H, W = 2, 4, 3, 12, 12
    kernel, stride, padding, kpad = (3, 7, 7), (2, 4, 4), (1, 3, 3), 448
    x = torch.randn(B, T, C, H, W, generator=g, dtype=torch.float64)
    emu = EmuKernels(exact=True, dtype=torch.float64)
    cols, (To, Ho, Wo) = emu.im2col3d(x, kernel, stride, padding, kpad)
    kt, kh, kw = kernel
    xs = x.numpy().reshape(-1)
    sim = np.full((B * To * Ho * Wo, kpad), np.nan)
    kreal = C * kt * kh * kw
    groups = (kpad + kw - 1) // kw
    for row in range(sim.shape[0]):
        ow, oh, ot = row % Wo, (row // Wo) % Ho, (row // (Wo * Ho)) % To
        b = row // (Wo * Ho * To)
        for grp in range(groups):
            col0 = grp * kw
            ncol = min(kw, kpad - col0)
            if col0 >= kreal:
                sim[row, col0:col0 + ncol] = 0.0
                continue
            dh, dt, c = grp % kh, (grp // kh) % kt, grp // (kh * kt)
            ti, hi, w0 = ot * stride[0] - padding[0] + dt, oh * stride[1] - padding[1] + dh, ow * stride[2] - padding[2]
            line_ok = 0 <= ti < T and 0 <= hi < H
            base = (((b * T + (ti if line_ok else 0)) * C + c) * H + (hi if line_ok else 0)) * W
            for j in range(ncol):
                wi = w0 + j
                sim[row, col0 + j] = xs[base + wi] if (line_ok and 0 <= wi < W) else 0.0
    assert rel(sim, cols.numpy()) == 0.0
    # and the GEMM against the flattened filter reproduces conv3d on the reference's transposed input
    w = torch.randn(8, C, kt, kh, kw, generator=g, dtype=torch.float64)
    ref = torch.nn.functional.conv3d(x.transpose(1, 2), w, None, stride=stride, padding=padding).flatten(2).transpose(1, 2)
    mine = (cols[:, :kreal] @ w.reshape(8, -1).t()).reshape(B, To * Ho * Wo, 8)
    assert rel(mine.numpy(), ref.numpy()) < 1e-13


# ---- mse kernels ---------------------------------------------------------------------------------------
def test_mse_index_math():
    g = torch.Generator().manual_seed(3)
    dims = (B, t, dt, h, w, dc) = (2, 3, 2, 2, 3, 5)
    hw, F, L1, PD = h * w, t * dt, 1 + t * h * w, dt * dc
    pred = torch.randn(B * L1, PD, generator=g, dtype=torch.float64)
    target = torch.randn(B, F, h, w, dc, generator=g, dtype=torch.float64)
    mask = (torch.rand(B, F, h, w, generator=g) < 0.5).double()
    emu = EmuKernels(exact=True, dtype=torch.float64)
    num = emu.mse_fwd(pred, target, mask, dims)[0].item()
    p, tg, m = pred.numpy().reshape(-1), target.numpy().reshape(-1), mask.numpy().reshape(-1)
    acc = 0.0
    for cell in range(B * F * hw):
        if m[cell] == 0:
            continue
        pp, f, b = cell % hw, (cell // hw) % F, cell // (hw * F)
        pr = ((b * L1 + 1 + (f // dt) * hw + pp) * PD) + (f % dt) * dc
        e = p[pr:pr + dc] - tg[cell * dc:(cell + 1) * dc]
        acc += m[cell] * float((e * e).sum()) / dc
    assert abs(acc - num) < 1e-12 * max(1.0, abs(num))
    coef = torch.tensor([0.37], dtype=torch.float64)
    dp = emu.mse_bwd(pred, target, mask, coef, dims).numpy().reshape(-1)
    sim = np.zeros(B * L1 * PD)
    for e in range(sim.size):
        j, l1, b = e % PD, (e // PD) % L1, e // (PD * L1)
        if l1 == 0:
            continue
        l = l1 - 1
        tt, pp = l // hw, l % hw
        f, c = tt * dt + j // dc, j % dc
        cell = (b * F + f) * hw + pp
        if m[cell] != 0:
            sim[e] = 0.37 * m[cell] * (p[e] - tg[cell * dc + c])
    assert rel(sim, dp) < 1e-14


# ---- xattn kernels: tile loop, log2-domain online softmax, masking, scale bookkeeping -------------------
def sim_xattn_fwd(q, k, v, scale, KT=16):
    Nq, Nk = q.shape[0], k.shape[0]
    qr = q * (scale * LOG2E)
    m = np.full(Nq, -np.inf)
    l = np.zeros(Nq)
    acc = np.zeros_like(q)
    for k0 in range(0, Nk, KT):
        nk = min(KT, Nk - k0)
        Ks = np.zeros((KT, HD)); Vs = np.zeros((KT, HD))
        Ks[:nk], Vs[:nk] = k[k0:k0 + nk], v[k0:k0 + nk]
        sc = qr @ Ks.T
        sc[:, nk:] = -np.inf
        mn = np.maximum(m, sc.max(1))
        corr = np.exp2(m - mn)
        l *= corr
        acc *= corr[:, None]
        p = np.exp2(sc - mn[:, None])
        l += p.sum(1)
        acc += p @ Vs
        m = mn
    return acc / l[:, None], (m + np.log2(l)) * LN2


def sim_xattn_bwd(q, k, v, o, do, lse, scale, KT=16, QT=16, QCHUNK=32):
    Nq, Nk = q.shape[0], k.shape[0]
    # dQ kernel
    qr = q * (scale * LOG2E)
    dl = (do * o).sum(1)
    lse2 = lse * LOG2E
    dq = np.zeros_like(q)
    for k0 in range(0, Nk, KT):
        nk = min(KT, Nk - k0)
        Ks = np.zeros((KT, HD)); Vs = np.zeros((KT, HD))
        Ks[:nk], Vs[:nk] = k[k0:k0 + nk], v[k0:k0 + nk]
        p1, p2 = qr @ Ks.T, do @ Vs.T
        pj = np.exp2(p1 - lse2[:, None])
        pj[:, nk:] = 0.0
        ds = pj * (p2 - dl[:, None])
        dq += ds @ Ks
    dq *= scale
    # dK/dV kernel (query range split in chunks, tiles of QT, atomics across chunks)
    kr = k * (scale * LOG2E)
    dk, dv = np.zeros_like(k), np.zeros_like(v)
    for q_begin in range(0, Nq, QCHUNK):
        q_end = min(Nq, q_begin + QCHUNK)
        dkr, dvr = np.zeros_like(k), np.zeros_like(v)
        for q0 in range(q_begin, q_end, QT):
            n = max(0, min(QT, q_end - q0))
            Qs = np.zeros((QT, HD)); Ds = np.zeros((QT, HD))
            Qs[:n], Ds[:n] = q[q0:q0 + n], do[q0:q0 + n]
            Ls = np.full(QT, np.inf); Dl = np.zeros(QT)
            Ls[:n], Dl[:n] = lse2[q0:q0 + n], dl[q0:q0 + n]
            p1, p2 = kr @ Qs.T, v @ Ds.T                     # [Nk, QT]
            pj = np.exp2(p1 - Ls[None, :])
            ds = pj * (p2 - Dl[None, :])
            dvr += pj @ Ds
            dkr += ds @ Qs
        dk += dkr * scale
        dv += dvr
    return dq, dk, dv


@pytest.mark.parametrize('Nq,Nk', [(70, 37), (16, 16), (5, 1), (33, 50)])
def test_xattn_tile_algorithm(Nq, Nk):
    rng = np.random.default_rng(4)
    q, k, v = rng.standard_normal((Nq, HD)), rng.standard_normal((Nk, HD)), rng.standard_normal((Nk, HD))
    scale = HD ** -0.5
    s = (q @ k.T) * scale
    mx = s.max(1, keepdims=True)
    lse = (mx + np.log(np.exp(s - mx).sum(1, keepdims=True)))[:, 0]
    p = np.exp(s - lse[:, None])
    o = p @ v
    so, slse = sim_xattn_fwd(q, k, v, scale)
    assert rel(so, o) < 1e-13 and rel(slse, lse) < 1e-13
    do = rng.standard_normal((Nq, HD))
    dv = p.T @ do
    dp = do @ v.T
    ds = p * (dp - (do * o).sum(1, keepdims=True)) * scale
    dq, dk = ds @ k, ds.T @ q
    sdq, sdk, sdv = sim_xattn_bwd(q, k, v, o, do, lse, scale)
    for mine, ref in ((sdq, dq), (sdk, dk), (sdv, dv)):      # one key => dq, dk are exactly 0: compare absolutely
        assert np.abs(mine - ref).max() < 1e-12 * max(1.0, np.abs(ref).max())


# ---- tensor-core flash attention (vt_attention_mma.cu): the tile walk of tests/attn_mma_emu.py ------------------------

@pytest.mark.parametrize('hd', [64, 96])
@pytest.mark.parametrize('Nq,Nk', [(1, 1), (5, 1), (63, 65), (64, 64), (65, 129), (129, 63), (197, 197), (300, 393)])
def test_attn_mma_model_exact(Nq, Nk, hd):
    """The model in 'exact' mode (64-row tiles, online softmax in the log2 domain, masking, lse = +inf past Nq in the
    backward) reproduces closed-form fp64 attention; finite junk in the rows past Nq / Nk (the next problem's rows in memory)
    must not reach the result."""
    rng = torch.Generator().manual_seed(9)
    P, scale = 2, hd ** -0.5
    pad = lambda x, n: torch.cat([x, torch.randn(P, 64 + 7, hd, generator=rng, dtype=torch.float64) * 7.0], 1)
    q, k, v, do = (torch.randn(P, n, hd, generator=rng, dtype=torch.float64) for n in (Nq, Nk, Nk, Nq))
    o, lse, dq, dk, dv = AE.reference(q, k, v, do, scale)
    so, slse = AE.fwd(pad(q, Nq), pad(k, Nk), pad(v, Nk), scale, 'exact', Nq=Nq, Nk=Nk)
    assert rel(so, o) < 1e-12 and rel(slse, lse) < 1e-12
    sdq, sdk, sdv = AE.bwd(pad(q, Nq), pad(k, Nk), pad(v, Nk), pad(o, Nq), pad(do, Nq), slse, scale, 'exact', Nq=Nq, Nk=Nk)
    for mine, ref in ((sdq, dq), (sdk, dk), (sdv, dv)):      # one key => dq, dk are exactly 0: compare absolutely
        assert mine.shape == ref.shape
        assert float((mine - ref).abs().max()) < 1e-11 * max(1.0, float(ref.abs().max()))


@pytest.mark.parametrize('regime', AE.REGIMES)
def test_attn_mma_model_bf16_noise(regime):
    """The 'bf16' model rounds where the kernels do: its outputs are bf16 values (dK / dV only on the packed path), it lands a
    few bf16 ulps from fp64, and the rounding of P and dS adds to the rounding of the outputs alone ('bf16_out')."""
    hd, Nq, Nk, scale = 64, 129, 197, 0.125
    q, k, v, do = AE.make_inputs(2, Nq, Nk, hd, scale, regime, seed=1)
    o, lse, dq, dk, dv = AE.reference(q, k, v, do, scale)
    if regime == 'uniform':
        s = (q @ k.transpose(1, 2)) * scale
        assert float((s - s[:, :, :1]).abs().max()) < 1e-9             # every logit of a row equal: P = 1 / Nk
    if regime == 'max_last':
        s = (q @ k.transpose(1, 2)) * scale
        assert bool((s.argmax(-1) >= (Nk - 1) // 64 * 64).all()) and 26 < float(s.amax()) < 34
    if regime == 'max_first':
        s = (q @ k.transpose(1, 2)) * scale
        assert float((s[:, :, 64:].amax(-1) - s[:, :, :64].amax(-1)).max()) < -90
    b_o, _ = AE.fwd(q, k, v, scale, 'bf16_out')
    m_o, m_lse = AE.fwd(q, k, v, scale, 'bf16')
    assert torch.equal(AE.bf16(m_o), m_o)
    assert float((m_lse - lse).abs().max()) < 1e-10                   # l is summed from the unrounded P
    gq, gk, gv = AE.bwd(q, k, v, m_o, do, m_lse, scale, 'bf16', dkv_bf16=True)
    fq, fk, fv = AE.bwd(q, k, v, m_o, do, m_lse, scale, 'bf16', dkv_bf16=False)
    assert torch.equal(AE.bf16(gq), gq) and torch.equal(AE.bf16(gk), gk) and torch.equal(AE.bf16(gv), gv)
    assert torch.equal(AE.bf16(fk), gk) and torch.equal(AE.bf16(fv), gv) and not torch.equal(fk, gk)
    for got, ref in ((m_o, o), (gq, dq), (gk, dk), (gv, dv)):
        e = AE.row_errors(got, ref)
        assert 1e-4 < e.glob < 0.1, e
    # rounding P costs accuracy on top of the output's rounding, except where P is exactly 1 (uniform rows: exp2(0))
    assert AE.row_errors(b_o, o).glob < AE.row_errors(m_o, o).glob or regime == 'uniform'


# ---- the per-row gate of the attention tests: faults it must catch --------------------------------------------------------
def test_row_gate_catches_one_copied_query_row():
    """At (Bp, N, H) = (64, 197, 12) one head's query row replaced by its neighbour's stays under the whole-tensor 5e-3 gate of
    test_gpu_attention.py but fails the per-row gate against the bf16 model."""
    Bp, N, H, hd, scale = 64, 197, 12, 64, 0.125
    q, k, v, _ = AE.make_inputs(Bp * H, N, N, hd, scale, seed=2)
    o = AE.reference(q, k, v, q, scale)[0]
    model = AE.fwd(q, k, v, scale, 'bf16')[0]
    bad = model.clone()
    bad[5 * H + 7, 100] = bad[5 * H + 7, 101]
    assert AE.within_budget(model, o, model)[0]
    assert rel(bad, o) < 5e-3
    ok, g, m = AE.within_budget(bad, o, model)
    assert not ok and g.where == (5 * H + 7, 0, 100), (g, m)


def test_row_gate_catches_one_wrong_key_tile_of_dk():
    """One 64-key tile of dK 10 % too large at Nk = 1569 is within the 2e-2 whole-tensor gate of test_gpu_mvit.py's
    tensor-core cases, and far outside the per-row gate."""
    P, N, hd, scale = 2, 1569, 64, 0.125
    q, k, v, do = AE.make_inputs(P, N, N, hd, scale, seed=3)
    o, lse, dq, dk, dv = AE.reference(q, k, v, do, scale)
    m_o, m_lse = AE.fwd(q, k, v, scale, 'bf16')
    _, mk, _ = AE.bwd(q, k, v, m_o, do, m_lse, scale, 'bf16')
    bad = mk.clone()
    bad[1, 640:704] *= 1.1
    assert AE.within_budget(mk, dk, mk)[0]
    assert rel(bad, dk) < 2e-2
    ok, g, _ = AE.within_budget(bad, dk, mk)
    assert not ok and g.where[0] == 1 and 640 <= g.where[2] < 704


def test_lse_gate_catches_a_shift_on_a_partial_query_tile():
    """lse off by 1e-3 on the five rows of one problem's partial last query tile (N = 197) passes a whole-tensor 1e-5 gate."""
    P, N, hd, scale = 48, 197, 64, 0.125
    q, k, v, _ = AE.make_inputs(P, N, N, hd, scale, seed=4)
    lse = AE.reference(q, k, v, q, scale)[1]
    bad = lse.clone()
    bad[3, 192:] += 1e-3
    assert AE.lse_error(AE.fwd(q, k, v, scale, 'bf16')[1], lse)[0] < AE.LSE_TOL
    assert rel(bad, lse) < 1e-5
    e, i = AE.lse_error(bad, lse)
    assert e > AE.LSE_TOL and i // N == 3 and i % N >= 192


def test_row_gate_catches_scale_applied_twice_to_dk():
    P, Nq, Nk, hd, scale = 2, 129, 197, 64, 0.125
    q, k, v, do = AE.make_inputs(P, Nq, Nk, hd, scale, seed=5)
    dk = AE.reference(q, k, v, do, scale)[3]
    m_o, m_lse = AE.fwd(q, k, v, scale, 'bf16')
    _, mk, _ = AE.bwd(q, k, v, m_o, do, m_lse, scale, 'bf16')
    assert AE.within_budget(mk, dk, mk)[0]
    assert not AE.within_budget(mk * scale, dk, mk)[0]


def test_row_metric_locates_the_row():
    g = torch.Generator().manual_seed(6)
    ref = torch.randn(2, 3, 70, 8, generator=g, dtype=torch.float64)
    got = ref.clone()
    got[1, 2, 65, 3] += 0.5
    e = AE.row_errors(got, ref)
    assert e.where == (1, 2, 65)
    assert abs(e.worst - 0.5 / float(ref[1, 2, 65].norm())) < 1e-12
    assert abs(e.glob - 0.5 / float(ref.norm())) < 1e-12
    small = ref.clone()
    small[0, 0, 0] *= 1e-6                                             # a near-zero row is measured against the floor
    bumped = small.clone()
    bumped[0, 0, 0, 0] += 1e-3
    rms = float(small.norm(dim=-1).square().mean().sqrt())
    assert abs(AE.row_errors(bumped, small).worst - 1e-3 / (AE.ROW_FLOOR * rms)) < 1e-9
    assert AE.row_errors(torch.full_like(ref, float('nan')), ref).worst == float('inf')
    z = torch.zeros(1, 1, 4, 8, dtype=torch.float64)
    assert AE.row_errors(z + 1e-7, z).worst < 1e-6                    # an all-zero reference is compared absolutely


# ---------------------------------------------------------------------------------------------------------------------
# fp32 residual epilogue on TMA (vt_gemm_common.cuh: epilogue_tile_tma_res): box / segment arithmetic of the affine row maps
# ---------------------------------------------------------------------------------------------------------------------
def _tma_box(tensor3, c_row, c_b, estride, rows=32):
    """rows x D box of the 3-D tensor view [samples, rows in sample, D] starting at row c_row and stepping `estride` rows (the
    map's element stride): out-of-range rows come back as zeros (load) and are dropped (store) — what the TMA unit does in
    tiled mode, negative start coordinates included.  Returns (box, valid, row index of every box row)."""
    import torch
    Bc, Rc, D = tensor3.shape
    box = torch.zeros(rows, D, dtype=tensor3.dtype)
    valid = torch.zeros(rows, dtype=torch.bool)
    where = []
    for i in range(rows):
        r = c_row + i * estride
        where.append(r)
        if 0 <= c_b < Bc and 0 <= r < Rc:
            box[i] = tensor3[c_b, r]
            valid[i] = True
    return box, valid, where


@pytest.mark.parametrize('B,T,P', [(2, 8, 196), (3, 4, 9 * 4), (1, 2, 50), (2, 3, 33)])
@pytest.mark.parametrize('kind', ['temporal', 'spatial'])
def test_residual_epilogue_segments_cover_every_row_once(B, T, P, kind):
    """Walks the epilogue's per-group logic (32-row groups of 128-row tiles; one or two TMA boxes per group; special rows by
    plain stores) for the temporal and spatial maps and checks it against the out_row / aux_row arrays of ops.token_maps."""
    import torch
    from videotransformer_pytorch_b200 import ops
    D = 8
    S = 1 + P * T
    R = B * S
    maps = ops.token_maps(B, T, P, 'cpu')
    aff = ops.affine_row_maps(B, T, P, D)[kind]
    if aff['period'] < 32:
        pytest.skip('periods below 32 rows use the generic epilogue')
    M = B * P * T if kind == 'temporal' else B * T * (P + 1)
    out_row = maps['temporal'] if kind == 'temporal' else maps['sp_out']
    aux_row = maps['temporal'] if kind == 'temporal' else maps['sp_aux']
    g = torch.Generator().manual_seed(0)
    acc = torch.randn(M, D, generator=g)                       # s * (accumulator + bias), already in GEMM row order
    x = torch.randn(R, D, generator=g)                         # residual stream
    rows_total = R + (B * T if kind == 'spatial' else 0)
    got = torch.full((rows_total, D), float('nan'))
    writes = torch.zeros(rows_total, dtype=torch.int32)
    # the 3-D view the tensor maps describe: (sample, row in sample, col); the spatial regrouping walks it with element stride T
    period, skip, tcount = aff['period'], aff['skip'], aff['tcount']
    pc = period - skip
    bc = (M // period + tcount - 1) // tcount
    row_stride = aff['stride_t'] if tcount > 1 else aff['stride_p']
    if tcount > 1:
        assert aff['stride_p'] == tcount * aff['stride_t'] and tcount <= 8      # what res_tma_applicable requires
    def view3(buf):
        return torch.as_strided(buf.reshape(-1), (bc, pc * tcount, D), (aff['stride_b'], row_stride, 1), aff['base'])
    x3 = view3(x if kind == 'temporal' else torch.cat([x, torch.zeros(B * T, D)]))
    n_outer = M // period
    n_direct = n_tma = 0
    for m0 in range(0, (M + 127) // 128 * 128, 32):
        outer0, inner0 = m0 // period, m0 % period
        seg, live = [], []
        for sg in range(2):
            outer = outer0 + sg
            seg_t, seg_p, seg_b = outer % tcount, inner0 - sg * period - skip, outer // tcount
            seg.append((seg_p, seg_t, seg_b))
            live.append(outer < n_outer and seg_p + 31 >= 0 and seg_p < pc and (sg == 0 or inner0 + 32 > period))
        if not (live[0] or live[1]):
            continue
        only = 0 if live[0] else 1
        direct = (live[0] and live[1]) or seg[only][0] < 0
        if direct:                                          # thread = row, addresses from the index arrays
            n_direct += 1
            for lane in range(32):
                row = m0 + lane
                if row >= M:
                    continue
                my_seg = 1 if inner0 + lane >= period else 0
                my_inner = inner0 + lane - my_seg * period
                if my_inner < skip:
                    dst = (aff['special_base'] + (outer0 + my_seg) * aff['special_stride']) // D
                    got[dst] = acc[row]
                    writes[dst] += 1
                    continue
                o, a = int(out_row[row]), int(aux_row[row])
                if o >= 0:
                    got[o] = acc[row] + (x[a] if a >= 0 else 0)
                    writes[o] += 1
            continue
        n_tma += 1
        seg_p, seg_t, seg_b = seg[only]
        assert seg_p >= 0                                   # TMA boxes never start outside the tensor
        box, valid, where = _tma_box(x3, seg_p * tcount + seg_t, seg_b, tcount)
        result = torch.zeros(32, D)
        for lane in range(32):
            row = m0 + lane
            my_seg = 1 if inner0 + lane >= period else 0
            my_inner = inner0 + lane - my_seg * period
            val = (acc[row] if row < M else torch.zeros(D)) + box[lane]
            result[lane] = val
            if row < M and my_inner < skip:                   # next period's special row at the tail of the box
                assert not valid[lane]
                dst = (aff['special_base'] + (outer0 + my_seg) * aff['special_stride']) // D
                got[dst] = val
                writes[dst] += 1
        for lane in range(32):                                # the TMA store clips exactly like the load
            if valid[lane]:
                off = aff['base'] + where[lane] * row_stride + seg_b * aff['stride_b']
                if m0 + lane < M:
                    assert int(out_row[m0 + lane]) == off // D
                got[off // D] = result[lane]
                writes[off // D] += 1
    assert n_tma > 0
    exp = torch.full((rows_total, D), float('nan'))
    add = x[aux_row.long().clamp(min=0)] * (aux_row >= 0)[:, None]
    exp[out_row.long()] = acc + add
    named = torch.zeros(rows_total, dtype=torch.int32)
    named[out_row.long()] = 1
    assert torch.equal(writes, named)                           # every mapped row written exactly once, no other row touched
    assert torch.equal(torch.nan_to_num(got, nan=-1.0), torch.nan_to_num(exp, nan=-1.0))
