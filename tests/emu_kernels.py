"""CPU emulation of the C-ABI kernel table (videotransformer_pytorch_b200._lib.CudaKernels).

TEST INFRASTRUCTURE ONLY — lives under tests/ and is installed by the `emu` fixture so that the
host-side logic of ops.py / transformer.py / video_transformer.py (row maps, cls handling, DropPath
bookkeeping, backward formulas, state-dict surface) can be checked against the reference-generated
goldens on a box without a GPU.  It mirrors each kernel's *contract* (include/vt_b200.h) with plain torch
ops; set `exact=True` to skip bf16 rounding (then results match the fp64 goldens to ~1e-6 in fp32 /
1e-12 in fp64, which pins the host logic independent of kernel precision).
The product package never imports this file.

Every method has the name, parameters and defaults of its CudaKernels counterpart (tests/test_abi.py checks this).  The
two capabilities ops.run asks a table for are constructor flags, off by default so that the `emu` fixture's table takes
the saving (autograd) forms: `inference_forms` (the 'gelu_h' epilogue and the calls that leave their backward-only
outputs unwritten) and `fp8_forms` (the e4m3 GEMM and row quantiser).  Calls that tests inspect are appended to `calls`,
one record per call, led by the method's name; a forward form's record carries whether the backward-only outputs were
asked for as its second field.
"""
from __future__ import annotations

import math

import torch

from tests.emu_augment import jitter_frames, parse, resize_window
from tests.emu_fp8 import dequant, quant_rows_twin
from tests.emu_randaug import desc_ops, randaug_frames
from videotransformer_pytorch_b200 import _lib


def bicubic_rows(rows, grid, out_grid, scales):
    """fp64 F.interpolate(mode='bicubic', align_corners=False, scale_factor=scales) of the row-major grid
    rows [gh*gw, D] -> [oh*ow, D]"""
    import torch.nn.functional as F
    D = rows.shape[1]
    g = rows.reshape(grid[0], grid[1], D).permute(2, 0, 1)[None]
    y = F.interpolate(g, scale_factor=tuple(scales), mode='bicubic', align_corners=False)
    assert tuple(y.shape[-2:]) == tuple(out_grid), (y.shape, out_grid)
    return y[0].permute(1, 2, 0).reshape(-1, D)


class EmuKernels:
    name = 'emu'

    def __init__(self, exact=False, dtype=torch.float32, *, inference_forms=False, fp8_forms=False):
        self.exact = exact
        self.f = dtype          # "fp32" storage type of the emulation (float64 for exact host-logic checks)
        self.inference_forms = inference_forms
        self.fp8_forms = fp8_forms
        self.calls = []

    # storage type standing in for bf16
    def _h(self, t):
        if self.exact:
            return t.to(self.f)
        return t.to(torch.bfloat16)

    def _up(self, t):
        return t.to(self.f)

    def _idx(self, t):
        return t.to(torch.int64)

    def gemm(self, a, b, M, N, Kdim, *, a_mn=False, b_mn=False, epi='bf16', bias=None, bias2=None, out=None, aux=None,
             out_row=None, aux_row=None, row_scale=None, out_rows=None, split_ok=False,
             force_splits=0, force_bn=0, row_map=None, tag=None):
        self.calls.append(('gemm', M, N, Kdim, a_mn, b_mn, epi))
        if row_map is not None:
            # the affine description handed to the TMA residual epilogue must be the out_row / aux_row arrays in closed form
            assert epi == 'f32' and aux is not None and out_row is not None and aux_row is not None
            ld = out.stride(0)
            m = torch.arange(M, dtype=torch.int64)
            outer, inner = m // row_map['period'], m % row_map['period']
            special = inner < row_map['skip']
            elem = (row_map['base'] + (outer % row_map['tcount']) * row_map['stride_t'] +
                    (inner - row_map['skip']) * row_map['stride_p'] + (outer // row_map['tcount']) * row_map['stride_b'])
            assert bool((elem % ld == 0).all()) and M % row_map['period'] == 0
            rows = elem // ld
            exp_out = torch.where(special, (row_map.get('special_base', -1) + outer * row_map.get('special_stride', 0)) // ld, rows)
            exp_aux = torch.where(special, torch.full_like(rows, -1), rows)
            assert torch.equal(exp_out, out_row.cpu().to(torch.int64)), 'row_map does not reproduce out_row'
            assert torch.equal(exp_aux, aux_row.cpu().to(torch.int64)), 'row_map does not reproduce aux_row'
            assert aux.stride(0) == ld
        A = self._up(a).t() if a_mn else self._up(a)
        Bm = self._up(b) if b_mn else self._up(b).t()
        assert A.shape == (M, Kdim) and Bm.shape == (Kdim, N), (A.shape, Bm.shape, M, N, Kdim)
        acc = A @ Bm
        if bias is not None:
            acc = acc + self._up(bias)
        assert epi in ('bf16', 'f32', 'gelu_h') and (aux is None or epi == 'f32'), epi
        if row_scale is not None:
            acc = acc * self._up(row_scale)[:, None]
        if bias2 is not None:
            assert epi == 'f32' and aux is not None
            acc = acc + self._up(bias2)
        if epi == 'f32' and aux is not None:
            if aux_row is not None:
                ar = self._idx(aux_row)
                add = torch.zeros_like(acc)
                ok = ar >= 0
                add[ok] = self._up(aux)[ar[ok]]
                acc = acc + add
            else:
                acc = acc + self._up(aux)
        val = acc.to(self.f) if epi == 'f32' else self._h(acc)
        dst = None if epi == 'gelu_h' else out          # gelu_h: h from the bf16-rounded z, like the kernel
        if dst is None:
            rows = out_rows if out_rows is not None else M
            dst = torch.empty((rows, N), dtype=val.dtype)
        if out_row is not None:
            orow = self._idx(out_row)
            ok = orow >= 0
            dst[orow[ok]] = val[ok].to(dst.dtype)
        else:
            dst[:M] = val.to(dst.dtype)
        if epi == 'gelu_h':
            h = self._gelu(dst)
            return h if out is None else out.copy_(h)
        return dst

    def gemm_e4m3(self, a, b, M, N, Kdim, *, epi='bf16', bias=None, bias2=None, out=None, aux=None, out_row=None,
                  aux_row=None, row_scale=None, out_rows=None, force_bn=0, row_map=None, tag=None):
        """Dequantises both operands (exact: e4m3 values times powers of two) and runs the emulated GEMM with the same
        epilogue."""
        assert isinstance(a, _lib.E4M3) and isinstance(b, _lib.E4M3) and epi in ('bf16', 'f32', 'gelu_h')
        out = self.gemm(dequant(a, self.f), dequant(b, self.f), M, N, Kdim, epi=epi, bias=bias, bias2=bias2, out=out, aux=aux,
                        out_row=out_row, aux_row=aux_row, row_scale=row_scale, out_rows=out_rows, force_bn=force_bn,
                        row_map=row_map, tag=tag)
        self.calls[-1] = ('gemm_e4m3',) + self.calls[-1][1:]
        return out

    def quant_rows_e4m3(self, x):
        self.calls.append(('quant_rows_e4m3',) + tuple(x.shape))
        return quant_rows_twin(x)

    def ln_fwd(self, x2d, gamma, beta, eps, in_row=None, rows=None, out_fp32=False, stats=True):
        self.calls.append(('ln_fwd', stats))
        x = self._up(x2d)
        if in_row is not None:
            x = x[self._idx(in_row)]
        elif rows is not None:
            x = x[:rows]
        mu = x.mean(-1, keepdim=True)
        var = ((x - mu) ** 2).mean(-1, keepdim=True)
        rstd = torch.rsqrt(var + eps)
        y = (x - mu) * rstd * self._up(gamma) + self._up(beta)
        y = y.to(self.f) if out_fp32 else self._h(y)
        return (y, mu[:, 0].to(self.f), rstd[:, 0].to(self.f)) if stats else (y, None, None)

    def ln_bwd(self, dy, x2d, mean, rstd, gamma, in_row=None, out_row=None, dres=None, dx=None, n_aux=0):
        x = self._up(x2d)
        xs = x[self._idx(in_row)] if in_row is not None else x[:dy.shape[0]]
        d = self._up(dy)
        xh = (xs - self._up(mean)[:, None]) * self._up(rstd)[:, None]
        g = d * self._up(gamma)
        m1 = g.mean(-1, keepdim=True)
        m2 = (g * xh).mean(-1, keepdim=True)
        val = self._up(rstd)[:, None] * (g - m1 - xh * m2)
        D = d.shape[1]
        if dx is None:
            dx = torch.empty((x2d.shape[0], D), dtype=self.f)
        aux = torch.empty((n_aux, D), dtype=self.f) if n_aux else None
        if out_row is not None:
            t = self._idx(out_row)
            pos = t >= 0
            add = val[pos]
            if dres is not None:
                add = add + self._up(dres)[t[pos]]
            dx[t[pos]] = add.to(dx.dtype)
            if (~pos).any():
                aux[(-t[~pos] - 1)] = val[~pos].to(aux.dtype)
        else:
            add = val
            if dres is not None:
                add = add + self._up(dres)[:val.shape[0]]
            dx[:val.shape[0]] = add.to(dx.dtype)
        return dx, aux, (d * xh).sum(0).to(self.f), d.sum(0).to(self.f)

    def colsum(self, x):
        return self._up(x).sum(0).to(self.f)

    def cast_bf16(self, x):
        return self._h(x)

    def gather_cast(self, src2d, in_row=None, row_scale=None, rows=None):
        s = self._up(src2d)
        if in_row is not None:
            ir = self._idx(in_row)
            v = torch.zeros((ir.numel(), s.shape[1]), dtype=s.dtype)
            ok = ir >= 0
            v[ok] = s[ir[ok]]
        else:
            v = s if rows is None else s[:rows]
        if row_scale is not None:
            v = v * self._up(row_scale)[:, None]
        return self._h(v)

    def gelu(self, z):
        self.calls.append(('gelu',))
        return self._gelu(z)

    def _gelu(self, z):
        zz = self._up(z)
        return self._h(0.5 * zz * (1 + torch.erf(zz / math.sqrt(2.0))))

    def cls_rows(self, dst, src, extra=None, scale=1.0):
        v = self._up(src)
        if extra is not None:
            v = v + scale * self._up(extra).sum(dim=1)
        dst.copy_(v.to(dst.dtype))
        return dst

    def gather_cast_colsum(self, src2d, in_row=None, row_scale=None, rows=None, unscaled_sums=False):
        out = self.gather_cast(src2d, in_row=in_row, row_scale=row_scale, rows=rows)
        if unscaled_sums:
            return out, self.colsum(out), self.colsum(self.gather_cast(src2d, in_row=in_row, rows=rows))
        return out, self.colsum(out)

    def dgelu_colsum(self, dh, z):
        out = self.dgelu(dh, z)
        return out, self.colsum(out)

    def dgelu(self, dh, z):
        zz = self._up(z)
        cdf = 0.5 * (1 + torch.erf(zz / math.sqrt(2.0)))
        pdf = torch.exp(-0.5 * zz * zz) / math.sqrt(2 * math.pi)
        return self._h(self._up(dh) * (cdf + zz * pdf))

    def attn_fwd(self, qkv, Bp, N, H, hd, scale, want_probs=False, impl=0, want_lse=True):
        self.calls.append(('attn_fwd', want_lse, N))
        q = self._up(qkv).reshape(Bp, N, 3, H, hd).permute(2, 0, 3, 1, 4)
        s = (q[0] @ q[1].transpose(-1, -2)) * scale
        lse = torch.logsumexp(s, dim=-1)
        p = torch.exp(s - lse[..., None])
        o = (p @ q[2]).transpose(1, 2).reshape(Bp * N, H * hd)
        return self._h(o), (lse.to(self.f) if want_lse else None), (p.to(self.f) if want_probs else None)

    def attn_bwd(self, qkv, ctx, dctx, lse, Bp, N, H, hd, scale, impl=0):
        self.calls.append(('attn_bwd', N))
        q = self._up(qkv).reshape(Bp, N, 3, H, hd).permute(2, 0, 3, 1, 4)
        Q, Kk, V = q[0], q[1], q[2]
        O = self._up(ctx).reshape(Bp, N, H, hd).transpose(1, 2)
        dO = self._up(dctx).reshape(Bp, N, H, hd).transpose(1, 2)
        s = (Q @ Kk.transpose(-1, -2)) * scale
        p = torch.exp(s - self._up(lse)[..., None])
        dV = p.transpose(-1, -2) @ dO
        dP = dO @ V.transpose(-1, -2)
        delta = (dO * O).sum(-1, keepdim=True)
        dS = p * (dP - delta) * scale
        dQ = dS @ Kk
        dK = dS.transpose(-1, -2) @ Q
        d = torch.stack((dQ, dK, dV), dim=0).permute(1, 3, 0, 2, 4).reshape(qkv.shape)
        return self._h(d)

    def im2col(self, x, tube, ph, pw):
        B, T, C, H, W = x.shape
        Tp, Hp, Wp = T // tube, H // ph, W // pw
        xx = self._up(x).reshape(B, Tp, tube, C, Hp, ph, Wp, pw).permute(0, 1, 4, 6, 3, 2, 5, 7)
        return self._h(xx.reshape(B * Tp * Hp * Wp, C * tube * ph * pw))

    def im2col_u8(self, x, scale, shift, tube, ph, pw):
        xf = x.to(self.f).permute(0, 1, 4, 2, 3) * self._up(scale).view(1, 1, -1, 1, 1) + self._up(shift).view(1, 1, -1, 1, 1)
        return self.im2col(xf, tube, ph, pw)

    def im2col_u8_mix(self, x, scale, shift, plan, tube, ph, pw):
        xf = x.to(self.f).permute(0, 1, 4, 2, 3) * self._up(scale).view(1, 1, -1, 1, 1) + self._up(shift).view(1, 1, -1, 1, 1)
        mode, lam = int(plan[0]), float(plan[1])
        yl, yh, xl, xh = (int(v) for v in plan[2:6])
        if mode == 1:
            xf = xf * lam + xf.flip(0) * (1.0 - lam)
        elif mode == 2:
            xf = xf.clone()
            xf[..., yl:yh, xl:xh] = xf.flip(0)[..., yl:yh, xl:xh]
        return self.im2col(xf, tube, ph, pw)

    def linear_small_fwd(self, x, w, b):
        y = self._up(x) @ self._up(w).t()
        return (y + self._up(b) if b is not None else y).to(torch.float32)

    def linear_small_bwd(self, dy, x, w, need_dx=True, need_dw=True):
        dy_, x_, w_ = self._up(dy), self._up(x), self._up(w)
        dx = (dy_ @ w_).to(torch.float32) if need_dx else None
        dw = (dy_.t() @ x_).to(torch.float32) if need_dw else None
        db = dy_.sum(0).to(torch.float32) if need_dw else None
        return dx, dw, db

    def softmax_ce(self, logits, labels=None, soft_targets=None):
        z = self._up(logits)
        M, N = z.shape
        t = torch.nn.functional.one_hot(labels, N).to(z.dtype) if labels is not None else self._up(soft_targets)
        lse = torch.logsumexp(z, dim=-1)
        ts = t.sum(-1)
        row = lse * ts - (t * z).sum(-1)
        dz = (z.softmax(-1) * ts[:, None] - t) / M
        return row.mean().reshape(1).to(torch.float32), dz.to(torch.float32), row.to(torch.float32)

    def scale_by_scalar(self, t, scalar):
        return (self._up(t) * self._up(scalar)[0]).to(torch.float32)

    def col2im(self, cols, shape, tube, ph, pw):
        B, T, C, H, W = shape
        Tp, Hp, Wp = T // tube, H // ph, W // pw
        xx = self._up(cols).reshape(B, Tp, Hp, Wp, C, tube, ph, pw).permute(0, 1, 5, 4, 2, 6, 3, 7)
        return xx.reshape(shape).to(self.f)

    def topk_hits(self, logits, labels, views, ks, hits, samples, probs=None):
        self.calls.append(('topk_hits', views, tuple(ks)))
        B = labels.numel()
        C = logits.shape[1]
        z = logits.float().reshape(B, views, C)
        m = z[:, 0]
        for v in range(1, views):                           # views summed in order, then scaled by fp32 1/V (as the kernel does)
            m = m + z[:, v]
        m = m * torch.tensor(1.0 / views, dtype=torch.float32)
        ok = (labels >= 0) & (labels < C)
        ml = m.gather(1, labels.clamp(0, C - 1).reshape(B, 1))
        rank = (m > ml).sum(1)
        rank = torch.where(ok & ~torch.isnan(ml[:, 0]), rank, torch.full_like(rank, C))
        for i, k in enumerate(ks):
            hits[i] += int((rank < k).sum())
        samples[0] += B
        if probs is not None:
            probs.copy_(m.softmax(-1))

    def forward_only_calls(self):
        """The recorded calls that show a forward-only form: gelu_h GEMMs and calls without their statistics."""
        return [c for c in self.calls if (c[0] == 'gemm' and c[-1] == 'gelu_h') or
                (c[0] in ('ln_fwd', 'attn_fwd', 'xattn_fwd', 'pool_fwd', 'maxpool_fwd') and c[1] is False)]

    # ------------------------------------------------------------------------------------------
    # positional-embedding resize: fp64 F.interpolate and its autograd
    # ------------------------------------------------------------------------------------------
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

    # ------------------------------------------------------------------------------------------
    # clip transforms: the fp32 restatements of tests/emu_augment.py and tests/emu_randaug.py
    # ------------------------------------------------------------------------------------------
    def resized_crop_u8(self, src, desc, out, err=None):
        n, T, S = out.shape[:3]
        self.calls.append(('resized_crop_u8', n, T, S))
        flat = src.cpu().numpy()
        for k, d in enumerate(parse(desc, _lib.CropDesc, n)):
            frames = flat[d.src_offset:d.src_offset + T * d.H * d.W * 3].reshape(T, d.H, d.W, 3)
            out[k] = resize_window(frames, (d.crop_y, d.crop_x, d.crop_h, d.crop_w), (d.RH, d.RW), (d.oy, d.ox), S,
                                   d.filter, d.flip)
        return out

    def color_jitter_u8(self, frames, desc):
        n = frames.shape[0]
        self.calls.append(('color_jitter_u8', n))
        for k, d in enumerate(parse(desc, _lib.JitterDesc, n)):
            ops = [(d.op[s], d.factor[s], d.one_minus[s]) for s in range(d.n_ops)]
            frames[k] = jitter_frames(frames[k], ops)
        return frames

    def rand_augment_u8(self, frames, desc, err=None):
        n = frames.shape[0]
        self.calls.append(('rand_augment_u8', n))
        for k, d in enumerate(parse(desc, _lib.RandAugDesc, n)):
            if not 0 <= d.n_ops <= _lib.RANDAUG_MAX_OPS or any(not 0 <= d.op[s] < 14 for s in range(d.n_ops)):
                frames[k] = 0
                if err is not None:
                    err.fill_(1)
                continue
            frames[k] = randaug_frames(frames[k], desc_ops(d))
        return frames

    # ------------------------------------------------------------------------------------------
    # MViT / MaskFeat kernels (include/vt_b200.h, second half)
    # ------------------------------------------------------------------------------------------
    @staticmethod
    def pool_out_thw(thw, stride):
        return tuple((n + 2 - 3) // s + 1 for n, s in zip(thw, stride))

    @staticmethod
    def maxpool_out_thw(thw, kernel, stride):
        return tuple((n + 2 * (k // 2) - k) // s + 1 for n, k, s in zip(thw, kernel, stride))

    def _pool_core(self, x, H, hd, thw, stride, w, gamma, beta, eps):
        """x: [B, N, H*hd] (float) -> (normalised [B,H,1+Lo,hd], pooled, mean, rstd)"""
        import torch.nn.functional as F
        B, N1, _ = x.shape
        T, Hin, Win = thw
        t = x.reshape(B, N1, H, hd).permute(0, 2, 1, 3)
        cls, body = t[:, :, :1], t[:, :, 1:]
        vol = body.reshape(B * H, T, Hin, Win, hd).permute(0, 4, 1, 2, 3)
        pv = F.conv3d(vol, w.reshape(hd, 1, 3, 3, 3), None, stride=tuple(stride), padding=1, groups=hd)
        pooled = torch.cat([cls, pv.reshape(B, H, hd, -1).transpose(2, 3)], dim=2)
        mu = pooled.mean(-1, keepdim=True)
        var = ((pooled - mu) ** 2).mean(-1, keepdim=True)
        rstd = torch.rsqrt(var + eps)
        out = (pooled - mu) * rstd * gamma + beta
        return out, pooled, mu, rstd

    def pool_fwd(self, src, H, hd, thw, stride, w, gamma, beta, eps, stats=True):
        self.calls.append(('pool_fwd', stats))
        out, pooled, mu, rstd = self._pool_core(self._up(src), H, hd, thw, stride, self._up(w), self._up(gamma),
                                                self._up(beta), eps)
        thw_o = self.pool_out_thw(thw, stride)
        if not stats:
            return self._h(out), None, None, None, thw_o
        return self._h(out), pooled.to(self.f), mu.reshape(-1).to(self.f), rstd.reshape(-1).to(self.f), thw_o

    def pool_bwd(self, dout, pooled, mean, rstd, gamma, src, w, din, H, hd, thw, stride):
        shp = pooled.shape[:-1] + (1,)
        xh = (self._up(pooled) - self._up(mean).reshape(shp)) * self._up(rstd).reshape(shp)
        d = self._up(dout)
        g = d * self._up(gamma)
        m1 = g.mean(-1, keepdim=True)
        m2 = (g * xh).mean(-1, keepdim=True)
        dpooled = self._up(rstd).reshape(shp) * (g - m1 - xh * m2)            # LayerNorm backward, closed form
        with torch.enable_grad():                                              # conv adjoint by autograd
            xs = self._up(src).detach().clone().requires_grad_(True)
            ws = self._up(w).detach().clone().requires_grad_(True)
            one, zero = torch.ones(hd, dtype=self.f), torch.zeros(hd, dtype=self.f)
            pooled_r = self._pool_core(xs, H, hd, thw, stride, ws, one, zero, 0.0)[1]
            gx, gw = torch.autograd.grad(pooled_r, (xs, ws), dpooled)
        din.copy_(self._h(gx).to(din.dtype))
        return gw.reshape(hd, 27).to(self.f), (d * xh).sum((0, 1, 2)).to(self.f), d.sum((0, 1, 2)).to(self.f)

    def xattn_fwd(self, q, k, v, scale, impl=0, want_lse=True):
        self.calls.append(('xattn_fwd', want_lse, tuple(q.shape), k.shape[2]))
        Q, Kk, V = self._up(q), self._up(k), self._up(v)
        B, H, Nq, hd = Q.shape
        s = (Q @ Kk.transpose(-1, -2)) * scale
        lse = torch.logsumexp(s, dim=-1)
        p = torch.exp(s - lse[..., None])
        o = (p @ V).transpose(1, 2).reshape(B, Nq, H * hd)
        return self._h(o), (lse.to(self.f) if want_lse else None)

    def xattn_bwd(self, q, k, v, o, dout, lse, scale, dq, impl=0):
        Q, Kk, V = self._up(q), self._up(k), self._up(v)
        B, H, Nq, hd = Q.shape
        O = self._up(o).reshape(B, Nq, H, hd).transpose(1, 2)
        dO = self._up(dout).reshape(B, Nq, H, hd).transpose(1, 2)
        s = (Q @ Kk.transpose(-1, -2)) * scale
        p = torch.exp(s - self._up(lse)[..., None])
        dV = p.transpose(-1, -2) @ dO
        dP = dO @ V.transpose(-1, -2)
        delta = (dO * O).sum(-1, keepdim=True)
        dS = p * (dP - delta) * scale
        dq.copy_(self._h(dS @ Kk).to(dq.dtype))
        return (dS.transpose(-1, -2) @ Q).to(self.f), dV.to(self.f)

    def maxpool_fwd(self, x, thw, kernel, stride, want_idx=True):
        import torch.nn.functional as F
        self.calls.append(('maxpool_fwd', want_idx))
        B, L1, D = x.shape
        T, H, W = thw
        xx = self._up(x)
        vol = xx[:, 1:].reshape(B, T, H, W, D).permute(0, 4, 1, 2, 3)
        y, idx = F.max_pool3d(vol, tuple(kernel), tuple(stride), tuple(k // 2 for k in kernel), return_indices=True)
        out_thw = tuple(y.shape[2:])
        yy = torch.cat([xx[:, :1], y.reshape(B, D, -1).transpose(1, 2)], dim=1)
        return yy.to(self.f), (idx.reshape(B, D, -1) if want_idx else None), out_thw        # idx is opaque to the host logic

    def maxpool_bwd(self, dy, idx, thw, kernel, stride):
        B, Lo1, D = dy.shape
        T, H, W = thw
        d = self._up(dy)
        vol = torch.zeros((B, D, T * H * W), dtype=d.dtype)
        vol.scatter_add_(2, idx, d[:, 1:].transpose(1, 2))
        return torch.cat([d[:, :1], vol.transpose(1, 2)], dim=1).to(self.f)

    def im2col3d(self, x, kernel, stride, padding, kpad):
        import torch.nn.functional as F
        B, T, C, H, W = x.shape
        xp = F.pad(self._up(x).permute(0, 2, 1, 3, 4), (padding[2], padding[2], padding[1], padding[1], padding[0], padding[0]))
        u = xp.unfold(2, kernel[0], stride[0]).unfold(3, kernel[1], stride[1]).unfold(4, kernel[2], stride[2])
        To, Ho, Wo = u.shape[2:5]
        cols = u.permute(0, 2, 3, 4, 1, 5, 6, 7).reshape(B * To * Ho * Wo, -1)
        cols = F.pad(cols, (0, kpad - cols.shape[1]))
        return self._h(cols), (To, Ho, Wo)

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

    def mvit_tokens_fwd(self, t, wmask, mask_token, cls_token, pos_s, pos_t, pos_cls, B, T, HW):
        C = t.shape[1]
        tt = self._up(t).reshape(B, T * HW, C)
        if wmask is not None:
            w = self._up(wmask).reshape(B, T * HW, 1)
            tt = tt * (1 - w) + self._up(mask_token).reshape(1, 1, C) * w
        pos = self._up(pos_s).reshape(1, HW, C).repeat(1, T, 1) + \
            torch.repeat_interleave(self._up(pos_t).reshape(1, T, C), HW, dim=1)
        cls = (self._up(cls_token).reshape(1, 1, C) + self._up(pos_cls).reshape(1, 1, C)).expand(B, 1, C)
        return torch.cat([cls, tt + pos], dim=1).to(self.f)

    def mvit_tokens_bwd(self, dx, wmask, B, T, HW):
        d = self._up(dx)[:, 1:]
        if wmask is not None:
            d = d * (1 - self._up(wmask).reshape(B, T * HW, 1))
        return self._h(d.reshape(B * T * HW, -1))

    def _mse_pred(self, pred, dims):
        B, t, dt, h, w, dc = dims
        p = self._up(pred).reshape(B, 1 + t * h * w, dt * dc)[:, 1:]
        return p.reshape(B, t, h, w, dt, dc).permute(0, 1, 4, 2, 3, 5).reshape(B, t * dt, h, w, dc)

    def mse_fwd(self, pred, target, mask, dims):
        B, t, dt, h, w, dc = dims
        p = self._mse_pred(pred, dims)
        e = ((p - self._up(target).reshape(p.shape)) ** 2).mean(-1) * self._up(mask).reshape(B, t * dt, h, w)
        num = torch.zeros(4, dtype=torch.float64 if target.dtype == torch.float64 else self.f)
        num[0] = e.sum()
        return num

    def mse_bwd(self, pred, target, mask, coef, dims):
        B, t, dt, h, w, dc = dims
        p = self._mse_pred(pred, dims)
        g = self._up(coef)[0] * self._up(mask).reshape(B, t * dt, h, w, 1) * (p - self._up(target).reshape(p.shape))
        g = g.reshape(B, t, dt, h, w, dc).permute(0, 1, 3, 4, 2, 5).reshape(B, t * h * w, dt * dc)
        g = torch.cat([torch.zeros((B, 1, dt * dc), dtype=g.dtype), g], dim=1)
        return self._h(g.reshape(B * (1 + t * h * w), dt * dc))

    # ------------------------------------------------------------------------------------------
    # fused clip + optimizer: the emulation works on the tensor lists of optim.TensorTable
    # ------------------------------------------------------------------------------------------
    def _opt_tensors(self, tbl):
        return tbl['_params'], tbl['_grads'](), tbl['_state']

    def opt_norm2(self, tbl):
        _, grads, _ = self._opt_tensors(tbl)
        tbl['norm2'].copy_(torch.stack([(g.double() ** 2).sum() for g in grads]).to(tbl['norm2'].dtype))
        return tbl['norm2']

    def _coef(self, tbl, clip, i):
        if not clip:
            return 1.0
        c = clip / (float(tbl['norm2'][i]) ** 0.5 + 1e-6)
        return min(c, 1.0)

    def opt_sgd(self, tbl, clip, momentum, nesterov, first_step):
        params, grads, state = self._opt_tensors(tbl)
        for i, (p, g) in enumerate(zip(params, grads)):
            d = g * self._coef(tbl, clip, i) + float(tbl['wd'][i]) * p
            buf = state[0][i]
            buf.copy_(d if first_step else momentum * buf + d)
            d = d + momentum * buf if nesterov else buf
            p.add_(d, alpha=-float(tbl['lr'][i]))

    def opt_adamw(self, tbl, clip, beta1, beta2, eps, bc1, bc2):
        params, grads, state = self._opt_tensors(tbl)
        for i, (p, g) in enumerate(zip(params, grads)):
            g = g * self._coef(tbl, clip, i)
            lr, wd = float(tbl['lr'][i]), float(tbl['wd'][i])
            p.mul_(1 - lr * wd)
            state[0][i].mul_(beta1).add_(g, alpha=1 - beta1)
            state[1][i].mul_(beta2).addcmul_(g, g, value=1 - beta2)
            p.addcdiv_(state[0][i], state[1][i].sqrt() / bc2 ** 0.5 + eps, value=-lr / bc1)
