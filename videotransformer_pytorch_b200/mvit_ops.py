"""Autograd functions of the MaskFeat / MViT path (SURVEY §8 a13-a15), as fixed sequences of C-ABI kernel launches.

  ConvTokensFn  <- MaskFeat.forward_features head: Conv3d patch embed + mask-token mixing + cls / positional encoding
                   (reference video_transformer.py:911-919, :585-618; pytorchvideo SpatioTemporalClsPositionalEncoding)
  PoolAttnFn    <- first half of pytorchvideo MultiScaleBlock.forward: x_res + proj(attention(pool(q), pool(k), pool(v)))
  MlpFn         <- second half: (x | proj(norm2 x)) + fc2(gelu(fc1(norm2 x)))
  MaskedMSEFn   <- MaskFeat.forward tail: decoder_pred + masked MSE on the cube centre frames (:878-901)

Data layout: the token stream stays fp32 [B, 1+T*H*W, dim] (cls first, tokens t-major) like the reference.  The fused
q/k/v projection writes one bf16 [B*N, 3*dim] buffer; pooling and attention read their q/k/v slices of it in place
through strides, and the backward kernels write the matching slices of the gradient buffer, so the reference's
reshape/permute/contiguous copies (pytorchvideo _attention_pool) never materialise.

Forward-only calls go through ops.run like the transformer blocks: ctx=None, no statistics, FC1 through 'gelu_h', and
with e4m3 weight shadows (fp8 inference precision) every block linear through ops._gemm.
"""
from __future__ import annotations

import torch

from . import _lib
from .ops import _act, _dgrad, _fc1_gelu, _gemm, _lse, _stats, _wgrad


def K():
    return _lib.K


def _slots(buf, B, N1, d):
    """q/k/v slices of a fused [B*N1, 3d] buffer as [B, N1, d] views."""
    v = buf.view(B, N1, 3 * d)
    return [v[:, :, s * d:(s + 1) * d] for s in range(3)]


def _bhnd(view, H, hd):
    """[B, N, H*hd] view -> [B, H, N, hd] view (no copy)."""
    B, N = view.shape[0], view.shape[1]
    return view.view(B, N, H, hd).permute(0, 2, 1, 3)


class ConvTokensFn(torch.autograd.Function):
    """x0[b,0] = cls + pos_cls;  x0[b,1+l] = conv3d(x)[b,l]*(1-w) + mask_token*w + pos_s[l%HW] + pos_t[l//HW].

    x is the float clip [B, T, C, H, W], or the decoder's uint8 clip [B, T, H, W, C] with norm = (mean, std) device
    tensors and an optional Mixup / CutMix plan (mixup.MixedClip.plan): the operand kernel then normalises and mixes."""

    @staticmethod
    def forward(ctx, x, conv_w, conv_b, mask_token, cls_token, pos_s, pos_t, pos_cls, wmask, conv_wh, geom, norm=None,
                plan=None):
        k = K()
        kernel, stride, padding = geom
        C0 = conv_w.shape[0]
        kpad = conv_wh.shape[1]
        if x.dtype == torch.uint8:
            cols, (To, Ho, Wo) = k.im2col3d_u8(x, norm[0], norm[1], plan, kernel, stride, padding, kpad)
        else:
            cols, (To, Ho, Wo) = k.im2col3d(x.float(), kernel, stride, padding, kpad)
        B = x.shape[0]
        M = cols.shape[0]
        t = k.gemm(cols, conv_wh, M, C0, kpad, bias=conv_b, epi='f32')
        x0 = k.mvit_tokens_fwd(t, wmask, mask_token.reshape(C0), cls_token.reshape(C0), pos_s.reshape(-1, C0),
                               pos_t.reshape(-1, C0), pos_cls.reshape(C0), B, To, Ho * Wo)
        if ctx is None:
            return x0
        ctx.save_for_backward(cols, wmask if wmask is not None else torch.empty(0, device=x.device))
        ctx.meta = (tuple(conv_w.shape), tuple(mask_token.shape), tuple(cls_token.shape), tuple(pos_s.shape),
                    tuple(pos_t.shape), tuple(pos_cls.shape), wmask is not None, B, To, Ho * Wo)
        return x0

    @staticmethod
    def backward(ctx, dx0):
        k = K()
        cols, wmask = ctx.saved_tensors
        wshape, mshape, cshape, psshape, ptshape, pcshape, has_mask, B, To, HW = ctx.meta
        wmask = wmask if has_mask else None
        C0 = wshape[0]
        kreal = wshape[1] * wshape[2] * wshape[3] * wshape[4]
        dx0 = dx0.contiguous()
        dt = k.mvit_tokens_bwd(dx0, wmask, B, To, HW)
        M = cols.shape[0]
        d_w = _wgrad(dt, cols, C0, cols.shape[1], M)[:, :kreal].reshape(wshape)
        d_b = k.colsum(dt)
        # parameter tables: plain reductions of the token gradient (96 columns)
        body = dx0[:, 1:].view(B, To, HW, C0)
        d_pos_s = body.sum(dim=(0, 1)).reshape(psshape)
        d_pos_t = body.sum(dim=(0, 2)).reshape(ptshape)
        d_cls = dx0[:, 0].sum(dim=0)
        if has_mask:
            d_mask = (body * wmask.view(B, To, HW, 1)).sum(dim=(0, 1, 2)).reshape(mshape)
        else:
            d_mask = torch.zeros(mshape, dtype=dx0.dtype, device=dx0.device)
        return (None, d_w.contiguous(), d_b, d_mask, d_cls.reshape(cshape).clone(), d_pos_s, d_pos_t,
                d_cls.reshape(pcshape).clone(), None, None, None, None, None)


class PoolAttnFn(torch.autograd.Function):
    """y = skip(x) + proj(softmax(Qp Kp^T / sqrt(hd)) Vp),  (Q,K,V) = Linear_{q,k,v}(LayerNorm(x)),
    Xp = LayerNorm_hd(depthwise_conv3d(X without cls) ++ cls)  (pool_first=False, conv pooling, cls kept)."""

    @staticmethod
    def forward(ctx, x, n1w, n1b, qw, qb, kw, kb, vw, vb, pw, pb, pq_w, nq_w, nq_b, pk_w, nk_w, nk_b, pv_w, nv_w, nv_b,
                qkv_wh, proj_wh, meta):
        k = K()
        heads, thw, stride_q, stride_kv, eps_block, eps_pool = meta
        x = x.contiguous()
        B, N1, d = x.shape
        H, hd = heads, d // heads
        M = B * N1
        scale = hd ** -0.5
        x2 = x.view(M, d)
        save = ctx is not None
        st = _stats(save)
        xn, mean, rstd = k.ln_fwd(x2, n1w, n1b, eps_block, **st)
        qkv = _gemm(k, xn, qkv_wh, M, 3 * d, d, bias=torch.cat([qb, kb, vb]), epi='bf16')
        sq, sk, sv = _slots(qkv, B, N1, d)
        if stride_q is not None:
            q4, q_pooled, q_mean, q_rstd, q_thw = k.pool_fwd(sq, H, hd, thw, stride_q, pq_w.reshape(hd, 27), nq_w, nq_b, eps_pool,
                                                             **st)
        else:
            q4, q_thw = _bhnd(sq, H, hd), tuple(thw)
            q_pooled = q_mean = q_rstd = torch.empty(0, device=x.device)
        k4, k_pooled, k_mean, k_rstd, _ = k.pool_fwd(sk, H, hd, thw, stride_kv, pk_w.reshape(hd, 27), nk_w, nk_b, eps_pool, **st)
        v4, v_pooled, v_mean, v_rstd, _ = k.pool_fwd(sv, H, hd, thw, stride_kv, pv_w.reshape(hd, 27), nv_w, nv_b, eps_pool, **st)
        o, lse = k.xattn_fwd(q4, k4, v4, scale, **_lse(save))
        Nq = q4.shape[2]
        Mq = B * Nq
        if stride_q is not None:
            kernel_skip = tuple(s + 1 if s > 1 else s for s in stride_q)
            x_res, idx, _ = k.maxpool_fwd(x, thw, kernel_skip, stride_q, **({} if save else {'want_idx': False}))
        else:
            x_res, idx = x, torch.empty(0, device=x.device)
        y = _gemm(k, o.view(Mq, d), proj_wh, Mq, d, d, bias=pb, epi='f32', aux=x_res.view(Mq, d))
        if not save:
            return y.view(B, Nq, d)
        ctx.save_for_backward(x, n1w, mean, rstd, xn, qkv, o, lse, idx, q4 if stride_q is not None else torch.empty(0, device=x.device),
                              q_pooled, q_mean, q_rstd, k4, k_pooled, k_mean, k_rstd, v4, v_pooled, v_mean, v_rstd,
                              pq_w if stride_q is not None else torch.empty(0, device=x.device), nq_w if stride_q is not None else torch.empty(0, device=x.device),
                              pk_w, nk_w, pv_w, nv_w, qkv_wh, proj_wh)
        ctx.meta = meta
        return y.view(B, Nq, d)

    @staticmethod
    def backward(ctx, dy):
        k = K()
        (x, n1w, mean, rstd, xn, qkv, o, lse, idx, q4s, q_pooled, q_mean, q_rstd, k4, k_pooled, k_mean, k_rstd,
         v4, v_pooled, v_mean, v_rstd, pq_w, nq_w, pk_w, nk_w, pv_w, nv_w, qkv_wh, proj_wh) = ctx.saved_tensors
        heads, thw, stride_q, stride_kv, eps_block, eps_pool = ctx.meta
        B, N1, d = x.shape
        H, hd = heads, d // heads
        M = B * N1
        scale = hd ** -0.5
        dy = dy.contiguous()
        Nq = dy.shape[1]
        Mq = B * Nq
        dy2 = dy.view(Mq, d)
        g, d_pb = k.gather_cast_colsum(dy2)
        d_pw = _wgrad(g, o.view(Mq, d), d, d, Mq)
        do = _dgrad(g, proj_wh, Mq, d, d, epi='bf16')
        sq, sk, sv = _slots(qkv, B, N1, d)
        dqkv = torch.empty_like(qkv)                      # every element is written by the kernels below
        dsq, dsk, dsv = _slots(dqkv, B, N1, d)
        if stride_q is not None:
            q4 = q4s
            dq4 = torch.empty((B, H, Nq, hd), dtype=qkv.dtype, device=x.device)
        else:
            q4 = _bhnd(sq, H, hd)
            dq4 = _bhnd(dsq, H, hd)
        dk, dv = k.xattn_bwd(q4, k4, v4, o, do, lse, scale, dq4)
        d_pq = d_nqw = d_nqb = None
        if stride_q is not None:
            d_pq, d_nqw, d_nqb = k.pool_bwd(dq4, q_pooled, q_mean, q_rstd, nq_w, sq, pq_w.reshape(hd, 27), dsq, H, hd, thw, stride_q)
            d_pq = d_pq.reshape(pq_w.shape)
        d_pk, d_nkw, d_nkb = k.pool_bwd(dk, k_pooled, k_mean, k_rstd, nk_w, sk, pk_w.reshape(hd, 27), dsk, H, hd, thw, stride_kv)
        d_pv, d_nvw, d_nvb = k.pool_bwd(dv, v_pooled, v_mean, v_rstd, nv_w, sv, pv_w.reshape(hd, 27), dsv, H, hd, thw, stride_kv)
        d_qkv_w = _wgrad(dqkv, xn, 3 * d, d, M)
        d_qkv_b = k.colsum(dqkv)
        dxn = _dgrad(dqkv, qkv_wh, M, d, 3 * d, epi='bf16')
        if stride_q is not None:
            kernel_skip = tuple(s + 1 if s > 1 else s for s in stride_q)
            dres = k.maxpool_bwd(dy, idx, thw, kernel_skip, stride_q).view(M, d)
        else:
            dres = dy2
        dx = torch.empty_like(x)
        _, _, d_n1w, d_n1b = k.ln_bwd(dxn, x.view(M, d), mean, rstd, n1w, dres=dres, dx=dx.view(M, d))
        return (dx, d_n1w, d_n1b, d_qkv_w[:d], d_qkv_b[:d], d_qkv_w[d:2 * d], d_qkv_b[d:2 * d], d_qkv_w[2 * d:], d_qkv_b[2 * d:],
                d_pw, d_pb, d_pq, d_nqw, d_nqb, d_pk.reshape(pk_w.shape), d_nkw, d_nkb, d_pv.reshape(pv_w.shape), d_nvw, d_nvb,
                None, None, None)


class MlpFn(torch.autograd.Function):
    """y = r + fc2(gelu(fc1(xn))),  xn = LayerNorm(x),  r = x  (dim == dim_out)  or  proj(xn)  (dim != dim_out)."""

    @staticmethod
    def forward(ctx, x, n2w, n2b, w1, b1, w2, b2, pjw, pjb, w1h, w2h, pjh, eps):
        k = K()
        x = x.contiguous()
        B, N, d = x.shape
        M = B * N
        Dh, do = w1h.shape[0], w2h.shape[0]
        x2 = x.view(M, d)
        save = ctx is not None
        xn, mean, rstd = k.ln_fwd(x2, n2w, n2b, eps, **_stats(save))
        xn = _act(k, xn, w1h)              # fp8: quantised once for FC1 and the width-changing proj
        z, h = _fc1_gelu(k, xn, w1h, b1, M, Dh, d, save)
        has_proj = pjh is not None
        r = _gemm(k, xn, pjh, M, do, d, bias=pjb, epi='f32') if has_proj else x2
        y = _gemm(k, h, w2h, M, do, Dh, bias=b2, epi='f32', aux=r)
        if not save:
            return y.view(B, N, do)
        ctx.save_for_backward(x, n2w, mean, rstd, xn, z, h, w1h, w2h, pjh if has_proj else torch.empty(0, device=x.device))
        ctx.has_proj = has_proj
        return y.view(B, N, do)

    @staticmethod
    def backward(ctx, dy):
        k = K()
        x, n2w, mean, rstd, xn, z, h, w1h, w2h, pjh = ctx.saved_tensors
        B, N, d = x.shape
        M = B * N
        Dh, do = w1h.shape[0], w2h.shape[0]
        dy = dy.contiguous()
        dy2 = dy.view(M, do)
        g, d_b2 = k.gather_cast_colsum(dy2)
        d_w2 = _wgrad(g, h, do, Dh, M)
        dz, d_b1 = k.dgelu_colsum(_dgrad(g, w2h, M, Dh, do, epi='bf16'), z)
        d_w1 = _wgrad(dz, xn, Dh, d, M)
        dx = torch.empty_like(x)
        d_pjw = d_pjb = None
        if ctx.has_proj:
            d_pjw = _wgrad(g, xn, do, d, M)
            d_pjb = d_b2.clone()
            dxn = _dgrad(dz, w1h, M, d, Dh, epi='f32')
            dxn = _dgrad(g, pjh, M, d, do, epi='f32', aux=dxn)
            _, _, d_nw, d_nb = k.ln_bwd(dxn, x.view(M, d), mean, rstd, n2w, dx=dx.view(M, d))
        else:
            dxn = _dgrad(dz, w1h, M, d, Dh, epi='bf16')
            _, _, d_nw, d_nb = k.ln_bwd(dxn, x.view(M, d), mean, rstd, n2w, dres=dy2, dx=dx.view(M, d))
        return dx, d_nw, d_nb, d_w1, d_b1, d_w2, d_b2, d_pjw, d_pjb, None, None, None, None


class MaskedMSEFn(torch.autograd.Function):
    """pred = decoder_pred(feats);  loss = sum(mask * mean_dc (pred' - target)^2) / (sum(mask) + 1e-5) with pred' the
    'b (t h w) (dt dc) -> b (t dt) h w dc' regrouping of pred without its cls row (video_transformer.py:878-901).
    `mask` is already restricted to the cube centre frames.  Returns (pred fp32 [B, 1+thw, dt*dc], loss)."""

    @staticmethod
    def forward(ctx, feats, dec_w, dec_b, dec_wh, target, mask, dims):
        k = K()
        B, N1, D = feats.shape
        M = B * N1
        F_out = dec_wh.shape[0]
        f = k.gather_cast(feats.contiguous().view(M, D))
        pred = k.gemm(f, dec_wh, M, F_out, D, bias=dec_b, epi='f32')
        num = k.mse_fwd(pred, target, mask, dims)            # fp64 when the targets are (reference: numpy fp64, dataset.py:190)
        denom = mask.sum() + 1e-5
        loss = num[0] / denom.to(num.dtype)
        ctx.save_for_backward(f, pred, target, mask, denom, dec_wh)
        ctx.dims = dims
        pred3 = pred.view(B, N1, F_out)
        ctx.mark_non_differentiable(pred3)
        return pred3, loss

    @staticmethod
    def backward(ctx, _dpred, dloss):
        k = K()
        f, pred, target, mask, denom, dec_wh = ctx.saved_tensors
        dims = ctx.dims
        M, D = f.shape
        F_out = dec_wh.shape[0]
        coef = (dloss.float() * (2.0 / dims[5]) / denom.float()).reshape(1).contiguous()
        dp = k.mse_bwd(pred, target, mask, coef, dims)
        d_w = _wgrad(dp, f, F_out, D, M)
        d_b = k.colsum(dp)
        B = dims[0]
        dfeats = _dgrad(dp, dec_wh, M, D, F_out, epi='f32').view(B, M // B, D)
        return dfeats, d_w, d_b, None, None, None, None
