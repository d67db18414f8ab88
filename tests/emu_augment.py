"""CPU twin of vt_resized_crop_u8 / vt_color_jitter_u8 (EmuKernels in tests/emu_kernels.py runs it): an fp32
restatement of both kernels' arithmetic (every product, sum and quotient rounded separately, as the kernels do
with __fmul_rn / __fadd_rn / __fdiv_rn), so the twin gives the kernels' bytes.  TEST INFRASTRUCTURE ONLY."""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

f32 = np.float32


def aa_filter(x, filter_id):
    """torch's antialias filter on an fp32 array: bicubic (a = -0.5, PIL's) or bilinear"""
    x = np.abs(x).astype(f32)
    if filter_id == 1:
        return np.where(x < 1, f32(1) - x, f32(0)).astype(f32)
    near = (((f32(1.5) * x - f32(2.5)) * x) * x + f32(1)).astype(f32)
    far = ((((f32(-0.5) * x + f32(2.5)) * x) - f32(4)) * x + f32(2)).astype(f32)
    return np.where(x < 1, near, np.where(x < 2, far, f32(0))).astype(f32)


def axis_weights(idx, n_in, n_out, filter_id, max_taps=32):
    """Taps of the resized-axis indices idx (int array) -> (lo int64 [n], w fp32 [n, max_taps]; taps past each count are
    0).  The fp32 operations of torch's _compute_indices_min_size_weights_aa, in its order."""
    scale = f32(n_in) / f32(n_out)
    half = f32(2.0 if filter_id == 0 else 1.0)
    support = half * scale if scale >= 1 else half
    invscale = f32(1.0 / np.float64(scale)) if scale >= 1 else f32(1.0)
    center = (scale * (np.asarray(idx).astype(f32) + f32(0.5))).astype(f32)
    lo = np.maximum(np.trunc((center - support).astype(f32).astype(np.float64) + 0.5), 0).astype(np.int64)
    hi = np.minimum(np.trunc((center + support).astype(f32).astype(np.float64) + 0.5), n_in).astype(np.int64)
    n = np.clip(hi - lo, 0, min(2 * int(np.ceil(support)) + 1, max_taps))
    j = np.arange(max_taps)
    arg = (((lo[:, None] + j).astype(f32) - center[:, None]).astype(f32).astype(np.float64) + 0.5) * np.float64(invscale)
    w = np.where(j < n[:, None], aa_filter(arg.astype(f32), filter_id), f32(0)).astype(f32)
    total = np.zeros(len(lo), f32)
    for k in range(max_taps):                     # sequential fp32 sum
        total = (total + w[:, k]).astype(f32)
    w = np.where(total[:, None] != 0, (w / np.where(total == 0, f32(1), total)[:, None]).astype(f32), w)
    return lo, n, w


def resize_window(frames, crop, resized, window, S, filter_id, flip):
    """frames uint8 [T, H, W, 3] -> uint8 [T, S, S, 3]: the S x S window at `window` of the crop box resized to `resized`
    (width pass, then height pass, fp32, sequential sums), clamped and rounded half to even, mirrored if flip."""
    cy, cx, ch, cw = crop
    RH, RW = resized
    oy, ox = window
    x = torch.from_numpy(np.ascontiguousarray(frames[:, cy:cy + ch, cx:cx + cw])).float()     # [T, ch, cw, 3]
    lo_x, n_x, w_x = axis_weights(np.arange(ox, ox + S), cw, RW, filter_id)
    lo_y, n_y, w_y = axis_weights(np.arange(oy, oy + S), ch, RH, filter_id)
    h = torch.zeros((x.shape[0], ch, S, 3))
    for j in range(int(n_x.max())):
        cols = torch.from_numpy(np.minimum(lo_x + j, cw - 1))
        h = h + x[:, :, cols] * torch.from_numpy(w_x[:, j])[None, None, :, None]
    acc = torch.zeros((x.shape[0], S, S, 3))
    for i in range(int(n_y.max())):
        rows = torch.from_numpy(np.minimum(lo_y + i, ch - 1))
        acc = acc + h[:, rows] * torch.from_numpy(w_y[:, i])[None, :, None, None]
    out = torch.round(acc.clamp(0, 255)).to(torch.uint8)
    return out.flip(2) if flip else out


def gray_u8(img):
    """torchvision rgb_to_grayscale on uint8 [..., 3] (fp32 ops, truncated)"""
    r, g, b = img[..., 0], img[..., 1], img[..., 2]
    return (0.2989 * r + 0.587 * g + 0.114 * b).to(torch.uint8)


def blend_u8(x, y, r, rc):
    return (torch.tensor(r, dtype=torch.float32) * x + torch.tensor(rc, dtype=torch.float32) * y).clamp(0, 255).to(torch.uint8)


def jitter_frames(frames, ops):
    """frames uint8 [T, S, S, 3]; ops [(op, factor, one_minus)] -> uint8 (ColorJitter's per-frame arithmetic)"""
    x = frames.clone()
    for op, r, rc in ops:
        if op == 0:
            x = blend_u8(x, torch.zeros_like(x), r, rc)
        elif op == 1:
            gs = gray_u8(x).to(torch.int64).sum(dim=(1, 2))                      # exact per-frame sum
            mean = gs.to(torch.float32) / float(x.shape[1] * x.shape[2])
            x = blend_u8(x, mean[:, None, None, None], r, rc)
        else:
            x = blend_u8(x, gray_u8(x)[..., None], r, rc)
    return x


def parse(desc, cls, n):
    raw = desc.cpu().numpy().tobytes()
    return [cls.from_buffer_copy(raw, k * C.sizeof(cls)) for k in range(n)]

