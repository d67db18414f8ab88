"""ctypes binding of include/vt_attn_maps.h: the cls row of the attention probabilities and show_attn's threshold masks
(libvt_b200.so, sm_90a).  `K` is the table ops.attention_probs and the models' attention_maps call; tests swap in a CPU
emulation with the same methods (tests/emu_attention_maps.py)."""
from __future__ import annotations

import ctypes as C

import torch

from ._lib import _check, _req, _stream, c_f32, c_i32, c_i64, c_vp, load_library


class AttnClsProbsParams(C.Structure):
    _fields_ = [('qkv', c_vp), ('probs', c_vp), ('Bp', c_i32), ('N', c_i32), ('H', c_i32), ('hd', c_i32), ('scale', c_f32)]


class AttnMassMaskParams(C.Structure):
    _fields_ = [('probs', c_vp), ('ld', c_i64), ('mask', c_vp), ('ldm', c_i64), ('rows', c_i32), ('n', c_i32),
                ('thresh', c_f32)]


EXPORTS = ['vt_attn_cls_probs', 'vt_attn_mass_mask']


def library() -> C.CDLL:
    lib = load_library()
    for name in EXPORTS:
        getattr(lib, name).restype = C.c_int
    return lib


class CudaAttnMapKernels:
    """Tensor-level wrappers; every method enqueues on torch's current CUDA stream."""

    name = 'cuda'

    def attn_cls_probs(self, qkv, Bp, N, H, hd, scale):
        """-> fp32 [Bp, H, N]: query row 0 of CudaKernels.attn_fwd's probs for the same qkv, bit for bit, without the
        [Bp, H, N, N] map."""
        _req(qkv, torch.bfloat16, 'attn_cls_probs.qkv')
        if not qkv.is_contiguous() or qkv.numel() != Bp * N * 3 * H * hd:
            raise RuntimeError('attn_cls_probs: qkv must be contiguous [Bp, N, 3, H, hd]')
        probs = torch.empty((Bp, H, N), dtype=torch.float32, device=qkv.device)
        p = AttnClsProbsParams()
        p.qkv, p.probs, p.Bp, p.N, p.H, p.hd, p.scale = qkv.data_ptr(), probs.data_ptr(), Bp, N, H, hd, scale
        _check(library().vt_attn_cls_probs(C.byref(p), _stream()), 'vt_attn_cls_probs')
        return probs

    def attn_mass_mask(self, probs, threshold):
        """show_attn's threshold mask of each row of probs (fp32 [..., n]) -> fp32 0 / 1 of the same shape, contiguous:
        an entry is kept when the cumulative mass of the row sorted ascending, up to and including it, exceeds
        1 - threshold (vt_attn_mass_mask; 1 - threshold is rounded to fp32, as torch compares it).  Rows are read in place
        when they are evenly strided with a unit last stride (a [..., 1:] slice of attn_cls_probs' output is)."""
        _req(probs, torch.float32, 'attn_mass_mask.probs')
        n = probs.shape[-1]
        rows2 = probs.reshape(-1, n)
        if rows2.stride(1) != 1:
            rows2 = rows2.contiguous()
        mask = torch.empty(probs.shape, dtype=torch.float32, device=probs.device)
        p = AttnMassMaskParams()
        ld = rows2.stride(0) if rows2.shape[0] > 1 else n      # a single row's stride is arbitrary
        p.probs, p.ld, p.mask, p.ldm = rows2.data_ptr(), ld, mask.data_ptr(), n
        p.rows, p.n, p.thresh = rows2.shape[0], n, 1.0 - threshold
        _check(library().vt_attn_mass_mask(C.byref(p), _stream()), 'vt_attn_mass_mask')
        return mask


K = CudaAttnMapKernels()
