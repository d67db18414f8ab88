"""CPU emulation of the attention-map kernel table (videotransformer_pytorch_b200.attn_maps_lib.CudaAttnMapKernels).

TEST INFRASTRUCTURE ONLY.  `mass_mask_rows` restates vt_attn_mass_mask operation for operation; EmuAttnMapKernels has
the methods of CudaAttnMapKernels (tests/test_attn_maps_abi.py checks this), and the `emu_maps` fixture installs it as
attn_maps_lib.K for host-logic tests, next to the `emu` fixture's EmuKernels.
"""
from __future__ import annotations

import pytest
import torch

from videotransformer_pytorch_b200 import _lib


def mass_mask_rows(rows, thresh):
    """vt_attn_mass_mask restated operation for operation (vt_attn_maps.cu, steps 1-5), on numpy fp32 rows [R, n]:
    1024 threads, thread t owning np / 1024 consecutive sorted positions, xor-butterfly sums and Hillis-Steele scans in
    fp64.  thresh: a Python float, rounded to fp32 as the ABI's float field does.  -> fp32 0 / 1 [R, n]"""
    import numpy as np
    R, n = rows.shape
    npad = max(1024, 1 << (n - 1).bit_length())
    chunk = npad // 1024
    th = np.float32(thresh)
    u = rows.astype(np.float32).view(np.uint32).astype(np.uint64)
    ob = np.where(u & 0x80000000, ~u & 0xffffffff, u | 0x80000000)          # order bits
    keys = (ob << np.uint64(32)) | np.arange(n, dtype=np.uint64)[None, :]
    order = np.argsort(keys, axis=1, kind='stable')                          # keys are distinct: the bitonic sort's order
    xs = np.take_along_axis(rows.astype(np.float32), order, axis=1)
    pad = np.zeros((R, npad - n), dtype=np.float32)
    lanes = np.arange(32)

    def butterfly(a):                       # [..., 32] fp64 -> every lane holds the xor-butterfly sum
        for o in (16, 8, 4, 2, 1):
            a = a + a[..., lanes ^ o]
        return a

    def scan(a):                            # [..., 32] fp64 inclusive Hillis-Steele scan (lane >= o adds lane - o)
        for o in (1, 2, 4, 8, 16):
            b = a.copy()
            b[..., o:] = a[..., o:] + a[..., :-o]
            a = b
        return a

    def seq(vals):                          # [R, 1024, chunk] -> sequential fp64 sums per thread (padding adds 0)
        acc = np.zeros(vals.shape[:2], dtype=np.float64)
        for e in range(chunk):
            acc = acc + vals[:, :, e].astype(np.float64)
        return acc

    xp = np.concatenate([xs, pad], axis=1).reshape(R, 1024, chunk)
    part = butterfly(seq(xp).reshape(R, 32, 32))[:, :, 0]
    s = butterfly(part)[:, 0].astype(np.float32)                             # [R]
    v = (xp / s[:, None, None]).astype(np.float32)                          # fp32 divisions (padding: 0 / s = 0)
    inc = scan(seq(v).reshape(R, 32, 32))                                   # [R, warp, lane]
    winc = scan(inc[:, :, 31])                                              # [R, warp]
    wbase = np.concatenate([np.zeros((R, 1)), winc[:, :-1]], axis=1)
    prev = np.concatenate([np.zeros((R, 32, 1)), inc[:, :, :-1]], axis=2)
    run = (wbase[:, :, None] + prev).reshape(R, 1024)
    c = np.empty((R, 1024, chunk), dtype=np.float32)
    for e in range(chunk):
        run = run + v[:, :, e].astype(np.float64)
        c[:, :, e] = run.astype(np.float32)
    kept = (c.reshape(R, npad)[:, :n] > th).astype(np.float32)
    mask = np.empty_like(kept)
    np.put_along_axis(mask, order, kept, axis=1)
    return mask


class EmuAttnMapKernels:
    name = 'emu'

    def __init__(self):
        self.calls = []

    def attn_cls_probs(self, qkv, Bp, N, H, hd, scale):
        """row 0 of the installed kernel table's attn_fwd probabilities: the emulation models the contract, not the memory"""
        self.calls.append(('attn_cls_probs', N))
        return _lib.K.attn_fwd(qkv, Bp, N, H, hd, scale, want_probs=True, want_lse=False)[2][:, :, 0].contiguous()

    def attn_mass_mask(self, probs, threshold):
        self.calls.append(('attn_mass_mask', probs.shape[-1]))
        n = probs.shape[-1]
        rows = probs.detach().to(torch.float32).reshape(-1, n).cpu().numpy()
        return torch.from_numpy(mass_mask_rows(rows, float(1.0 - threshold))).reshape(probs.shape)


@pytest.fixture
def emu_maps():
    """Swap the attention-map kernel table for the CPU emulation (host-logic tests only)."""
    from videotransformer_pytorch_b200 import attn_maps_lib
    old = attn_maps_lib.K
    attn_maps_lib.K = EmuAttnMapKernels()
    yield attn_maps_lib.K
    attn_maps_lib.K = old
