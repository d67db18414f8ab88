"""CPU twin of vt_pos_resize_fwd / _bwd for the host-logic tests: the kernel table of tests/emu_kernels.py plus the
bicubic pos_embed resize as fp64 F.interpolate and its autograd.  TEST INFRASTRUCTURE ONLY."""
from __future__ import annotations

import torch

from tests.emu_kernels import EmuKernels


def bicubic_rows(rows, grid, out_grid, scales):
    """fp64 F.interpolate(mode='bicubic', align_corners=False, scale_factor=scales) of the row-major grid
    rows [gh*gw, D] -> [oh*ow, D]"""
    import torch.nn.functional as F
    D = rows.shape[1]
    g = rows.reshape(grid[0], grid[1], D).permute(2, 0, 1)[None]
    y = F.interpolate(g, scale_factor=tuple(scales), mode='bicubic', align_corners=False)
    assert tuple(y.shape[-2:]) == tuple(out_grid), (y.shape, out_grid)
    return y[0].permute(1, 2, 0).reshape(-1, D)


class EmuKernelsResize(EmuKernels):
    def pos_resize_fwd(self, src, grid, out_grid, scales, out=None):
        self.calls.append(('pos_resize_fwd', tuple(grid), tuple(out_grid)))
        y = bicubic_rows(src.double(), grid, out_grid, scales).to(self.f)
        return y if out is None else out.copy_(y)

    def pos_resize_bwd(self, dout, grid, out_grid, scales, out=None):
        self.calls.append(('pos_resize_bwd', tuple(grid), tuple(out_grid)))
        with torch.enable_grad():
            x = torch.zeros(grid[0] * grid[1], dout.shape[1], dtype=torch.float64, requires_grad=True)
            (gx,) = torch.autograd.grad(bicubic_rows(x, grid, out_grid, scales), x, dout.double())
        gx = gx.to(self.f)
        return gx if out is None else out.copy_(gx)
