"""CPU twin of the fp8 inference forms (vt_quant_rows_e4m3, vt_gemm_e4m3; EmuKernels in tests/emu_kernels.py runs it with
fp8_forms=True) for the host-logic tests and as the quantising fp64 model of the GPU tests.  TEST INFRASTRUCTURE ONLY.

The quantiser's scale is a power of two, so x / scale is exact and the only rounding is the cast to e4m3 (round to nearest
even, saturating at +-448).  `quant_rows_twin` takes that cast from torch (clamp first: torch turns values past +-448 into
NaN where the kernel's satfinite saturates); `e4m3_round_fp64` restates it in exact fp64 arithmetic on the e4m3 grid.
"""
from __future__ import annotations

import torch

from videotransformer_pytorch_b200._lib import E4M3

E4M3_MAX = 448.0


def scale_exponent(amax: torch.Tensor) -> torch.Tensor:
    """k with 2^k = 2^ceil(log2(amax / 448)) exactly (frexp: amax = m 2^e, 448 = 0.875 2^9), clamped to [-126, 127];
    0 for an all-zero row."""
    m, e = torch.frexp(amax.to(torch.float64))
    k = e.to(torch.int64) - 9 + (m > 0.875).to(torch.int64)
    k = k.clamp(-126, 127)
    return torch.where(amax > 0, k, torch.zeros_like(k))


def e4m3_round_fp64(v: torch.Tensor) -> torch.Tensor:
    """Round fp64 values to the e4m3 grid, nearest even, saturating at +-448: exact fp64 arithmetic (v / quantum and the
    product back are power-of-two scalings; torch.round rounds half to even)."""
    v = v.to(torch.float64)
    a = v.abs()
    _, e = torch.frexp(torch.where(a > 0, a, torch.ones_like(a)))
    E = (e.to(torch.int64) - 1).clamp(min=-6)                  # exponent of the binade; subnormals share 2^-6
    quantum = torch.ldexp(torch.ones_like(v), E - 3)          # 3 mantissa bits
    r = torch.round(v / quantum) * quantum
    return r.clamp(-E4M3_MAX, E4M3_MAX)


def e4m3_cast(y: torch.Tensor) -> torch.Tensor:
    """cvt.rn.satfinite.e4m3 of fp32 values: torch's cast after clamping to +-448."""
    return y.float().clamp(-E4M3_MAX, E4M3_MAX).to(torch.float8_e4m3fn)


def quant_rows_twin(x: torch.Tensor) -> E4M3:
    """vt_quant_rows_e4m3 on the CPU: bf16 / fp32 rows [M, K] -> E4M3(q float8_e4m3fn, scale fp32).  fp64 rows (the exact
    emulation) are rounded by e4m3_round_fp64."""
    amax = x.abs().amax(dim=1) if x.shape[1] else torch.zeros(x.shape[0], dtype=x.dtype)
    k = scale_exponent(amax)
    inv = torch.ldexp(torch.ones_like(k, dtype=torch.float64), -k)
    if x.dtype == torch.float64:
        q = e4m3_round_fp64(x * inv[:, None]).to(torch.float8_e4m3fn)
    else:
        q = e4m3_cast(x.float() * inv.float()[:, None])       # exact power-of-two scaling, then the one rounding
    return E4M3(q, torch.ldexp(torch.ones_like(k, dtype=torch.float32), k.to(torch.int32)))


def dequant(t: E4M3, dtype=torch.float64) -> torch.Tensor:
    return t.q.to(dtype) * t.scale.to(dtype)[:, None]

