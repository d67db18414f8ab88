"""CPU twin of vt_im2col3d_u8_bf16 for the MaskFeat uint8-input tests: the kernel table of tests/emu_kernels.py plus the
uint8 Conv3d patch operand, with the kernel's rounding points.  TEST INFRASTRUCTURE ONLY."""
from __future__ import annotations

import torch

from tests.emu_kernels import EmuKernels


class EmuKernelsU8(EmuKernels):
    name = 'emu_u8'

    def im2col3d_u8(self, x, mean, std, plan, kernel, stride, padding, kpad):
        """Twin of vt_im2col3d_u8_bf16, with its rounding points: every op below is one fp32 op rounded to nearest (torch
        on the CPU contracts nothing): ToTensor u / 255, Normalize (. - mean) / std, Mixup v*lam + o*(1 - lam) with
        (1 - lam) in fp32, CutMix a copy; then zero padding and one bf16 rounding in im2col3d."""
        f32 = torch.float32
        v = (x.to(f32) / 255.0 - mean.to(f32).view(1, 1, 1, 1, -1)) / std.to(f32).view(1, 1, 1, 1, -1)   # [B,T,H,W,C]
        if plan is not None:
            plan = plan.to('cpu', f32)
            mode = int(plan[0])
            if mode == 1:
                lam = plan[1]
                v = v * lam + v.flip(0) * (torch.ones((), dtype=f32) - lam)
            elif mode == 2:
                yl, yh, xl, xh = (int(t) for t in plan[2:6])
                v = v.clone()
                v[:, :, yl:yh, xl:xh] = v.flip(0)[:, :, yl:yh, xl:xh]
        return self.im2col3d(v.permute(0, 1, 4, 2, 3), kernel, stride, padding, kpad)
