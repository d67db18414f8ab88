"""CPU twin of the forward-only kernel forms for the host-logic tests: the kernel table of tests/emu_pos_resize.py plus
the 'gelu_h' GEMM epilogue, NULL statistics outputs (stats=False / want_lse=False / want_idx=False) and vt_topk_hits.
Every call that has a forward-only form is recorded with whether it was given its backward-only outputs, so the tests
can see which form a forward took.  TEST INFRASTRUCTURE ONLY."""
from __future__ import annotations

import torch

from tests.emu_kernels import EmuKernels
from tests.emu_pos_resize import EmuKernelsResize


class EmuKernelsEval(EmuKernelsResize):
    inference_forms = True

    def gemm(self, a, b, M, N, Kdim, *, epi='bf16', out=None, **kw):
        if epi != 'gelu_h':
            return super().gemm(a, b, M, N, Kdim, epi=epi, out=out, **kw)
        z = super().gemm(a, b, M, N, Kdim, epi='bf16', **kw)       # h from the bf16-rounded z, like the kernel
        self.calls[-1] = self.calls[-1][:-1] + ('gelu_h',)
        h = EmuKernels.gelu(self, z)
        return h if out is None else out.copy_(h)

    def gelu(self, z):
        self.calls.append(('gelu',))
        return super().gelu(z)

    def ln_fwd(self, x2d, gamma, beta, eps, in_row=None, rows=None, out_fp32=False, stats=True):
        self.calls.append(('ln_fwd', stats))
        y, mu, rstd = super().ln_fwd(x2d, gamma, beta, eps, in_row=in_row, rows=rows, out_fp32=out_fp32)
        return (y, mu, rstd) if stats else (y, None, None)

    def attn_fwd(self, qkv, Bp, N, H, hd, scale, want_probs=False, impl=0, want_lse=True):
        self.calls.append(('attn_fwd', want_lse))
        o, lse, p = super().attn_fwd(qkv, Bp, N, H, hd, scale, want_probs=want_probs, impl=impl)
        return o, (lse if want_lse else None), p

    def xattn_fwd(self, q, k, v, scale, impl=0, want_lse=True):
        self.calls.append(('xattn_fwd', want_lse))
        o, lse = super().xattn_fwd(q, k, v, scale, impl=impl)
        return o, (lse if want_lse else None)

    def pool_fwd(self, src, H, hd, thw, stride, w, gamma, beta, eps, stats=True):
        self.calls.append(('pool_fwd', stats))
        out, pooled, mu, rstd, thw_o = super().pool_fwd(src, H, hd, thw, stride, w, gamma, beta, eps)
        return (out, pooled, mu, rstd, thw_o) if stats else (out, None, None, None, thw_o)

    def maxpool_fwd(self, x, thw, kernel, stride, want_idx=True):
        self.calls.append(('maxpool_fwd', want_idx))
        y, idx, thw_o = super().maxpool_fwd(x, thw, kernel, stride)
        return y, (idx if want_idx else None), thw_o

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
