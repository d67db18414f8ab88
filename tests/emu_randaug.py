"""CPU twin of vt_rand_augment_u8 (EmuKernels in tests/emu_kernels.py runs it): an fp32 restatement of the kernel's
arithmetic (every product and sum of the warp coordinates rounded separately, in the kernel's
order; the sharpness blur in exact integers; statistics per frame and channel), so the twin gives the kernel's bytes.
TEST INFRASTRUCTURE ONLY."""
from __future__ import annotations

import numpy as np
import torch

from tests.emu_augment import blend_u8, jitter_frames

f32 = np.float32
GEOMETRIC, SHARPNESS = (1, 2, 3, 4, 5), 9
JITTER_OP = {6: 0, 8: 1, 7: 2}            # Brightness, Contrast, Color -> ColorJitter's blend ops in emu_augment


def warp_sources(theta, S):
    """Nearest source (row, col) of every output pixel of an S x S warp, -1 outside: g = (x t0 + y t1) + t2 over the
    pixel centres, source = rint(((g + 1) S - 1) / 2), all in fp32 with separate roundings."""
    t = [f32(v) for v in theta]
    off = f32(0.5) - f32(0.5) * f32(S)
    x = (np.arange(S).astype(f32) + off)[None, :]
    y = (np.arange(S).astype(f32) + off)[:, None]

    def src(a, b, c):
        g = ((x * a).astype(f32) + (y * b).astype(f32)).astype(f32) + c
        u = np.rint((((g.astype(f32) + f32(1)) * f32(S) - f32(1)) * f32(0.5)).astype(f32))
        return np.where((u >= 0) & (u <= S - 1), u, -1).astype(np.int64)
    return src(t[0], t[1], t[2]), src(t[3], t[4], t[5])


def warp_coords64(theta, S):
    """The same source coordinates in fp64 from the same fp32 matrix, before rounding, and the magnitudes the fp32
    evaluations round: (ux, uy, A = max |x t0| + |y t1| + |t2| over both rows, G = max |g|)."""
    t = np.asarray(theta, dtype=np.float64)
    x = (np.arange(S) - S / 2 + 0.5)[None, :]
    y = (np.arange(S) - S / 2 + 0.5)[:, None]
    gx, gy = x * t[0] + y * t[1] + t[2], x * t[3] + y * t[4] + t[5]
    A = max(float((np.abs(x * t[0]) + np.abs(y * t[1]) + abs(t[2])).max()),
            float((np.abs(x * t[3]) + np.abs(y * t[4]) + abs(t[5])).max()))
    G = max(float(np.abs(gx).max()), float(np.abs(gy).max()))
    return ((gx + 1) * S - 1) / 2, ((gy + 1) * S - 1) / 2, A, G


def warp_bound(S, A, G):
    """|fp32 source coordinate - fp64 one| for any evaluation order, with or without FMA, of either unnormalisation
    (((g + 1) S - 1) / 2 or (g + 1) S / 2 - 0.5).  g's three terms and two sums err by at most gamma_3 A < 3.01 eps A,
    scaled by S / 2; adding 1, multiplying by S (or S / 2) and subtracting 1 (or 0.5) each add at most one rounding of a
    value <= S (G + 1).  So 1.51 eps S A + 3 eps S (G + 1) <= eps S (2 A + 4 (G + 1)), eps = 2^-24."""
    return 2.0 ** -24 * S * (2 * A + 4 * (G + 1))


def near_tie_mask(theta, S):
    """Output pixels whose fp64 source coordinate (either axis) lies within warp_bound of a half-integer: the only ones
    where two fp32 evaluations may pick different source pixels."""
    ux, uy, A, G = warp_coords64(theta, S)
    b = warp_bound(S, A, G)
    near = lambda u: np.abs(u - np.floor(u) - 0.5) <= b
    return near(ux) | near(uy), b


def warp(frames, theta):
    """frames uint8 [T, S, S, 3] -> the nearest-sampled warp, zero outside"""
    S = frames.shape[1]
    sx, sy = warp_sources(theta, S)
    ok = torch.from_numpy((sx >= 0) & (sy >= 0))
    out = frames[:, torch.from_numpy(np.maximum(sy, 0)), torch.from_numpy(np.maximum(sx, 0))]
    return torch.where(ok[None, :, :, None], out, torch.zeros_like(out))


def sharpen(frames, r, rc):
    """blend with the rounded [1 1 1; 1 5 1; 1 1 1] / 13 blur over interior pixels, each border pixel with itself"""
    S = frames.shape[1]
    if S <= 2:
        return frames
    x = frames.to(torch.int64)
    n = x[:, 1:-1, 1:-1] * 4
    for dy in (0, 1, 2):
        for dx in (0, 1, 2):
            n = n + x[:, dy:dy + S - 2, dx:dx + S - 2]
    y = x.clone()
    y[:, 1:-1, 1:-1] = torch.div(2 * n + 13, 26, rounding_mode='floor')
    return blend_u8(frames, y.to(torch.float32), r, rc)


def autocontrast(frames):
    x = frames.to(torch.float32)
    mn, mx = x.amin(dim=(1, 2), keepdim=True), x.amax(dim=(1, 2), keepdim=True)
    same = mx == mn
    scale = torch.reciprocal(torch.where(same, torch.ones_like(mx), mx - mn)) * 255.0     # torch's 255 / tensor
    out = ((x - mn) * scale).clamp(0, 255).to(torch.uint8)
    return torch.where(same, frames, out)


def equalize(frames):
    """per frame and channel: torchvision's table, (cumsum + step // 2) // step shifted right by one bin"""
    out = frames.clone()
    for t in range(frames.shape[0]):
        for c in range(3):
            v = frames[t, :, :, c].numpy().reshape(-1)
            hist = np.bincount(v, minlength=256).astype(np.int64)
            step = (v.size - int(hist[np.nonzero(hist)[0][-1]])) // 255
            if step == 0:
                continue
            lut = np.zeros(256, np.int64)
            lut[1:] = np.minimum((np.cumsum(hist)[:-1] + step // 2) // step, 255)
            out[t, :, :, c] = torch.from_numpy(lut[v].astype(np.uint8).reshape(frames.shape[1:3]))
    return out


def randaug_frames(frames, ops):
    """frames uint8 [T, S, S, 3]; ops [(op, arg, one_minus, theta6)] -> uint8, the ops applied in order"""
    x = frames.clone()
    for op, arg, rc, theta in ops:
        if op in GEOMETRIC:
            x = warp(x, theta)
        elif op in JITTER_OP:
            x = jitter_frames(x, [(JITTER_OP[op], arg, rc)])
        elif op == SHARPNESS:
            x = sharpen(x, arg, rc)
        elif op == 10:
            x = x & int(arg)
        elif op == 11:
            x = torch.where(x.to(torch.float32) >= float(arg), 255 - x, x)
        elif op == 12:
            x = autocontrast(x)
        elif op == 13:
            x = equalize(x)
    return x


def desc_ops(d):
    return [(d.op[s], d.arg[s], d.one_minus[s], list(d.theta[s])) for s in range(d.n_ops)]

