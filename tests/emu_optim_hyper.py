"""CPU kernel table for the capturable optimizer launches: EmuKernels whose fused update takes its per-step scalars the way
vt_opt_sgd / vt_opt_adamw do (include/vt_b200.h, vt_opt_params).

TEST INFRASTRUCTURE ONLY.  The kernels receive clip, first_step, bc1 and bc2 as fp32 struct fields, or, when the table
carries tbl['hyper'] (the static block of a captured step, optim.HyperArena), read them from that fp32 block and ignore
the fields.  This table rounds the field values to fp32 and substitutes the block's values when it is there, then runs
EmuKernels' update, so the two forms can be compared bit for bit on the CPU.
"""
from __future__ import annotations

import torch

from tests.emu_kernels import EmuKernels
from videotransformer_pytorch_b200 import _lib


def f32(x):
    """a scalar as the kernels receive it: an fp32 field of vt_opt_params or a slot of the fp32 hyper block"""
    return float(torch.tensor(float(x), dtype=torch.float32))


class HyperEmuKernels(EmuKernels):
    name = 'emu-hyper'

    def _scalars(self, tbl, **fields):
        hyper = tbl.get('hyper')
        if hyper is None:
            return {k: f32(v) for k, v in fields.items()}
        return {k: float(hyper[_lib.OPT_HYPER[k]]) for k in fields}

    def opt_sgd(self, tbl, clip, momentum, nesterov, first_step):
        sc = self._scalars(tbl, clip=clip or 0.0, first_step=int(first_step))
        super().opt_sgd(tbl, sc['clip'], momentum, nesterov, sc['first_step'] != 0.0)

    def opt_adamw(self, tbl, clip, beta1, beta2, eps, bc1, bc2):
        sc = self._scalars(tbl, clip=clip or 0.0, bc1=bc1, bc2=bc2)
        super().opt_adamw(tbl, sc['clip'], beta1, beta2, eps, sc['bc1'], sc['bc2'])
