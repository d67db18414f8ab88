"""MaskFeat (MViT-B encoder + HOG-regression head) on the sm_90a kernels, behind the reference's module surface.

Mirrors (reference file:line):
  MaskFeat                          video_transformer.py:803-922   (ctor kwargs, forward, forward_features)
  create_conv_patch_embed           video_transformer.py:585-618   -> .patch_embed.patch_model
  create_multiscale_vision_transformers  video_transformer.py:621-800 -> .mvit (block configuration logic)
and the pytorchvideo classes it instantiates (MultiScaleBlock, MultiScaleAttention, Mlp,
SpatioTemporalClsPositionalEncoding, MultiscaleVisionTransformers; 0.1.3-era signatures, see oracle/mvit_oracle.py):
parameter names and shapes are identical (`mvit.blocks.{i}.attn.{q,k,v,proj,pool_q,norm_q,...}`, `mvit.norm_embed`,
`mvit.cls_positional_encoding.*`, `patch_embed.patch_model.*`, `decoder_pred.*`, `mask_token`), so reference
checkpoints load with strict=True and optimizer.py's layer-decay parser (:100-111) sees the prefixes it expects.

The nn.Linear / nn.Conv3d / nn.LayerNorm children are parameter holders only; every forward goes through
mvit_ops.py -> libvt_b200.so.  No eager / CPU fallback.
"""
from __future__ import annotations

import torch
import torch.nn as nn

from . import mvit_ops, ops
from .ops import RowsNormFn
from .transformer import InferencePrecision, ShadowWeights, _f32
from .video_transformer import _ByteClipInput

HEAD_DIM = 96   # the kernels are specialised for MViT-B's head width (patch_embed_dim 96, heads double with dim)


def _round_width(width, multiplier, min_width=8, divisor=8):
    """Channel rounding rule of the MViT factory: scale, round to the nearest multiple of `divisor`, never lose >10 %."""
    if not multiplier:
        return int(width)
    scaled = float(width) * float(multiplier)
    floor = min_width or divisor
    rounded = max(floor, int(scaled + divisor / 2) // divisor * divisor)
    if rounded < 0.9 * scaled:
        rounded += divisor
    return int(rounded)


def mvit_block_plan(depth, patch_embed_dim, num_heads, embed_dim_mul, atten_head_mul, pool_q_stride_size,
                    pool_kv_stride_adaptive, pool_kvq_kernel, mlp_ratio=4.0):
    """Per-block (dim, dim_out, heads, stride_q | None, stride_kv) as the reference factory derives them
    (video_transformer.py:707-761): widths/heads multiply at the listed block indices, Q is pooled at the listed
    blocks, and the K/V stride shrinks by the accumulated Q stride so K/V keep a constant token count per stage."""
    dim_mul = {int(i): float(m) for i, m in (embed_dim_mul or [])}
    head_mul = {int(i): float(m) for i, m in (atten_head_mul or [])}
    q_stride = {int(r[0]): tuple(int(s) for s in r[1:]) for r in (pool_q_stride_size or [])}
    kernel = tuple(pool_kvq_kernel)
    if kernel != (3, 3, 3):
        raise NotImplementedError(f'pool_kvq_kernel={kernel}: the pooling kernels implement the 3x3x3 depthwise filter')
    plan = []
    kv = tuple(pool_kv_stride_adaptive)
    heads, dim = num_heads, patch_embed_dim
    for i in range(depth):
        if i in q_stride:
            kv = tuple(max(kv[a] // q_stride[i][a], 1) for a in range(3))
        heads = _round_width(heads, head_mul.get(i, 1.0), min_width=1, divisor=1)
        dim = _round_width(dim, dim_mul.get(i, 1.0), divisor=heads)
        dim_out = _round_width(dim, dim_mul.get(i + 1, 1.0), divisor=_round_width(heads, head_mul.get(i + 1, 1.0)))
        plan.append(dict(dim=dim, dim_out=dim_out, heads=heads, stride_q=q_stride.get(i), stride_kv=kv,
                         hidden=int(dim * mlp_ratio)))
    return plan


class PatchEmbeding(nn.Module):
    """Holder of the Conv3d patch filter (reference class name and spelling, video_transformer.py:563-581)."""

    def __init__(self, *, patch_model=None):
        super().__init__()
        assert patch_model is not None
        self.patch_model = patch_model


class SpatioTemporalClsPositionalEncoding(nn.Module):
    def __init__(self, embed_dim, patch_embed_shape, sep_pos_embed=True, has_cls=True):
        super().__init__()
        if not (sep_pos_embed and has_cls):
            raise NotImplementedError('only the separable positional encoding with a cls token is on the hot path')
        self.patch_embed_shape = tuple(patch_embed_shape)
        T, H, W = self.patch_embed_shape
        self.cls_token = nn.Parameter(torch.zeros(1, 1, embed_dim))
        self.pos_embed_spatial = nn.Parameter(torch.zeros(1, H * W, embed_dim))
        self.pos_embed_temporal = nn.Parameter(torch.zeros(1, T, embed_dim))
        self.pos_embed_class = nn.Parameter(torch.zeros(1, 1, embed_dim))


class Mlp(nn.Module):
    def __init__(self, in_features, hidden_features, out_features):
        super().__init__()
        self.fc1 = nn.Linear(in_features, hidden_features)
        self.fc2 = nn.Linear(hidden_features, out_features)


class MultiScaleAttention(nn.Module):
    def __init__(self, dim, num_heads, qkv_bias, stride_q, stride_kv):
        super().__init__()
        hd = dim // num_heads
        if hd != HEAD_DIM:
            raise NotImplementedError(f'head dim {hd}: the pooling-attention kernels are built for {HEAD_DIM}')
        if not qkv_bias:
            raise NotImplementedError('qkv_bias=False is not used by the reference (video_transformer.py:640)')
        self.num_heads = num_heads
        self.q = nn.Linear(dim, dim)
        self.k = nn.Linear(dim, dim)
        self.v = nn.Linear(dim, dim)
        self.proj = nn.Linear(dim, dim)

        def pool(stride):
            conv = nn.Conv3d(hd, hd, (3, 3, 3), stride=tuple(stride), padding=(1, 1, 1), groups=hd, bias=False)
            return conv, nn.LayerNorm(hd)        # eps 1e-5: the reference leaves attn_norm_layer at its default (:773)

        if stride_q is not None:
            self.pool_q, self.norm_q = pool(stride_q)
        else:
            self.pool_q = self.norm_q = None
        self.pool_k, self.norm_k = pool(stride_kv)
        self.pool_v, self.norm_v = pool(stride_kv)


class MultiScaleBlock(nn.Module):
    inference_precision = 'bf16'       # InferencePrecision.set_inference_precision

    def __init__(self, dim, dim_out, num_heads, hidden, stride_q, stride_kv, norm_eps=1e-6, qkv_bias=True):
        super().__init__()
        self.dim, self.dim_out = dim, dim_out
        self.stride_q = None if stride_q is None else tuple(stride_q)
        self.stride_kv = tuple(stride_kv)
        self.norm1 = nn.LayerNorm(dim, eps=norm_eps)
        self.attn = MultiScaleAttention(dim, num_heads, qkv_bias, self.stride_q, self.stride_kv)
        self.norm2 = nn.LayerNorm(dim, eps=norm_eps)
        self.mlp = Mlp(dim, hidden, dim_out)
        if dim != dim_out:
            self.proj = nn.Linear(dim, dim_out)
        self._shadow = ShadowWeights()

    def out_thw(self, thw):
        if self.stride_q is None:
            return tuple(thw)
        return tuple((n + 2 - 3) // s + 1 for n, s in zip(thw, self.stride_q))

    def _shadows(self, fp8):
        """(qkv, proj, fc1, fc2, width-changing proj or None) weight shadows: bf16, or e4m3 for the fp8 forward-only form."""
        a, sh, has_proj = self.attn, self._shadow, self.dim != self.dim_out
        if fp8:
            e = lambda name, *ps: sh.get_e4m3(name + ':e4m3', ps)
            return (e('qkv', a.q.weight, a.k.weight, a.v.weight), e('proj', a.proj.weight), e('fc1', self.mlp.fc1.weight),
                    e('fc2', self.mlp.fc2.weight), e('blkproj', self.proj.weight) if has_proj else None)
        return (sh.get_cat('qkv', [a.q.weight, a.k.weight, a.v.weight]), sh.get('proj', a.proj.weight),
                sh.get('fc1', self.mlp.fc1.weight), sh.get('fc2', self.mlp.fc2.weight),
                sh.get('blkproj', self.proj.weight) if has_proj else None)

    def forward(self, x, thw):
        a = self.attn
        qkv_wh, proj_wh, fc1_wh, fc2_wh, blkproj_wh = self._shadows(ops.fp8_form(self, x))
        f = _f32
        pq = (f(a.pool_q.weight), f(a.norm_q.weight), f(a.norm_q.bias)) if self.stride_q is not None else (None, None, None)
        meta = (a.num_heads, tuple(thw), self.stride_q, self.stride_kv, self.norm1.eps, a.norm_k.eps)
        x = ops.run(
            mvit_ops.PoolAttnFn, x, f(self.norm1.weight), f(self.norm1.bias), f(a.q.weight), f(a.q.bias), f(a.k.weight), f(a.k.bias),
            f(a.v.weight), f(a.v.bias), f(a.proj.weight), f(a.proj.bias), *pq,
            f(a.pool_k.weight), f(a.norm_k.weight), f(a.norm_k.bias), f(a.pool_v.weight), f(a.norm_v.weight), f(a.norm_v.bias),
            qkv_wh, proj_wh, meta)
        has_proj = self.dim != self.dim_out
        x = ops.run(
            mvit_ops.MlpFn, x, f(self.norm2.weight), f(self.norm2.bias), f(self.mlp.fc1.weight), f(self.mlp.fc1.bias),
            f(self.mlp.fc2.weight), f(self.mlp.fc2.bias),
            f(self.proj.weight) if has_proj else None, f(self.proj.bias) if has_proj else None,
            fc1_wh, fc2_wh, blkproj_wh, self.norm2.eps)
        return x, self.out_thw(thw)


class MultiscaleVisionTransformers(nn.Module):
    """Token stream [B, 1+T*H*W, 96] (already positional-encoded) -> [B, 1+T'*H'*W', dim_out]."""

    def __init__(self, cls_positional_encoding, blocks, norm_embed):
        super().__init__()
        self.cls_positional_encoding = cls_positional_encoding
        self.blocks = blocks
        self.norm_embed = norm_embed

    def forward(self, x):
        thw = self.cls_positional_encoding.patch_embed_shape
        for blk in self.blocks:
            x, thw = blk(x, thw)
        B, N, D = x.shape
        y = ops.run(RowsNormFn, x, _f32(self.norm_embed.weight), _f32(self.norm_embed.bias), self.norm_embed.eps, None)
        return y.view(B, N, D)


def create_multiscale_vision_transformers(*, spatial_size, temporal_size, depth=16, patch_embed_dim=96,
                                          conv_patch_embed_stride=(2, 4, 4), num_heads=1, mlp_ratio=4.0, qkv_bias=True,
                                          embed_dim_mul=None, atten_head_mul=None, pool_q_stride_size=None,
                                          pool_kv_stride_adaptive=None, pool_kvq_kernel=None, head=None, **unused):
    if head is not None:
        raise NotImplementedError('MaskFeat builds the MViT without a head (video_transformer.py:798)')
    if pool_kv_stride_adaptive is None or pool_kvq_kernel is None:
        raise NotImplementedError('the reference always sets pool_kv_stride_adaptive and pool_kvq_kernel (:822-823)')
    if isinstance(spatial_size, int):
        spatial_size = (spatial_size, spatial_size)
    dims = (temporal_size, spatial_size[0], spatial_size[1])
    shape = tuple(dims[i] // conv_patch_embed_stride[i] for i in range(3))
    plan = mvit_block_plan(depth, patch_embed_dim, num_heads, embed_dim_mul, atten_head_mul, pool_q_stride_size,
                           pool_kv_stride_adaptive, pool_kvq_kernel, mlp_ratio)
    blocks = nn.ModuleList(MultiScaleBlock(b['dim'], b['dim_out'], b['heads'], b['hidden'], b['stride_q'], b['stride_kv'],
                                           qkv_bias=qkv_bias) for b in plan)
    pos = SpatioTemporalClsPositionalEncoding(patch_embed_dim, shape, sep_pos_embed=True, has_cls=True)
    return MultiscaleVisionTransformers(pos, blocks, nn.LayerNorm(plan[-1]['dim_out'], eps=1e-6))


class MaskFeat(_ByteClipInput, InferencePrecision, nn.Module):
    """forward(x[B,T,3,H,W], target_x[B,T,h,w,dc], mask[B,t,h,w], cube_marker) -> (pred[B,T,h,w,dc], loss);
    forward_features(x, mask=None) -> [B, 1+t*h*w, embed_dims].

    x may also be the decoder's uint8 clip [B, T, H, W, 3] on the device, or a mixup.MixedClip wrapping one: ToTensor,
    Normalize (set_input_normalization) and Mixup / CutMix then happen inside the Conv3d patch-operand kernel."""

    def __init__(self, img_size=224, num_frames=16, input_channels=3, feature_dim=10, patch_embed_dim=96,
                 conv_patch_embed_kernel=(3, 7, 7), conv_patch_embed_stride=(2, 4, 4), conv_patch_embed_padding=(1, 3, 3),
                 embed_dim_mul=[[1, 2.0], [3, 2.0], [14, 2.0]], atten_head_mul=[[1, 2.0], [3, 2.0], [14, 2.0]],
                 pool_q_stride_size=[[1, 1, 2, 2], [3, 1, 2, 2], [14, 1, 2, 2]], pool_kv_stride_adaptive=[1, 8, 8],
                 pool_kvq_kernel=[3, 3, 3], head=None, pretrain_pth=None, **kwargs):
        super().__init__()
        self.num_frames = num_frames
        self.img_size = img_size
        self.stride = tuple(conv_patch_embed_stride)
        self.kernel = tuple(conv_patch_embed_kernel)
        self.padding = tuple(conv_patch_embed_padding)
        self.downsample_rate = 2 ** len(pool_q_stride_size)
        self.embed_dims = 2 ** len(embed_dim_mul) * patch_embed_dim
        self.patch_embed = PatchEmbeding(patch_model=nn.Conv3d(input_channels, patch_embed_dim, self.kernel,
                                                               stride=self.stride, padding=self.padding, bias=True))
        self.mvit = create_multiscale_vision_transformers(
            spatial_size=img_size, temporal_size=num_frames, patch_embed_dim=patch_embed_dim,
            conv_patch_embed_stride=self.stride, embed_dim_mul=embed_dim_mul, atten_head_mul=atten_head_mul,
            pool_q_stride_size=pool_q_stride_size, pool_kv_stride_adaptive=pool_kv_stride_adaptive,
            pool_kvq_kernel=pool_kvq_kernel, head=head)
        in_features = self.mvit.norm_embed.normalized_shape[0]
        self.decoder_pred = nn.Linear(in_features, feature_dim, bias=True)
        self.mask_token = nn.Parameter(torch.zeros(1, 1, patch_embed_dim))
        # reference init (video_transformer.py:847-853)
        w = self.patch_embed.patch_model.weight.data
        nn.init.xavier_uniform_(w.view([w.shape[0], -1]))
        nn.init.xavier_uniform_(self.decoder_pred.weight)
        nn.init.constant_(self.decoder_pred.bias, 0)
        nn.init.trunc_normal_(self.mask_token, std=.02)
        self._shadow = ShadowWeights()
        if pretrain_pth is not None:
            self.init_weights(pretrain_pth)

    def init_weights(self, pretrain_pth):
        """reference video_transformer.py:866-870"""
        from .weight_init import init_from_kinetics_pretrain_
        init_from_kinetics_pretrain_(self, pretrain_pth)

    @torch.jit.ignore
    def no_weight_decay_keywords(self):
        return {'pos_embed', 'cls_token', 'mask_token'}

    # ------------------------------------------------------------------------------------------
    def forward_features(self, x, mask=None):
        x, norm, plan = self._unwrap_clip(x, mean_std=True)
        conv = self.patch_embed.patch_model
        n, s, c = self.num_frames, self.img_size, conv.in_channels
        if norm is not None:
            if x.dim() != 5 or tuple(x.shape[1:]) != (n, s, s, c):
                raise RuntimeError(f'MaskFeat: expected a uint8 clip [B, {n}, {s}, {s}, {c}], got {tuple(x.shape)}')
        elif x.dim() != 5 or x.shape[1] != n or x.shape[-1] != s or x.shape[-2] != s:
            raise RuntimeError(f'MaskFeat: expected [B, {n}, C, {s}, {s}], got {tuple(x.shape)}')
        pos = self.mvit.cls_positional_encoding
        T, H, W = pos.patch_embed_shape
        B = x.shape[0]
        wmask = None
        if mask is not None:
            r = self.downsample_rate
            dense = mask.repeat_interleave(r, dim=2).repeat_interleave(r, dim=3)          # nearest resize (:917)
            wmask = dense.reshape(B, T * H * W).to(device=x.device, dtype=torch.float32).contiguous()
        kreal = conv.weight[0].numel()
        kpad = (kreal + 63) // 64 * 64
        x0 = ops.run(
            mvit_ops.ConvTokensFn, x, _f32(conv.weight), _f32(conv.bias), _f32(self.mask_token), _f32(pos.cls_token), _f32(pos.pos_embed_spatial),
            _f32(pos.pos_embed_temporal), _f32(pos.pos_embed_class), wmask,
            self._shadow.get_padded('conv', conv.weight, kpad), (self.kernel, self.stride, self.padding), norm, plan)
        return self.mvit(x0)

    def center_frame_mask(self, mask, cube_marker):
        """mask repeated over dt, zeroed outside each sample's cube centre frames (video_transformer.py:889-896)."""
        dt = self.stride[0]
        B = mask.shape[0]
        keep = torch.zeros(B, self.num_frames, dtype=torch.float32)
        for i, cubes in enumerate(cube_marker):
            for start, span in cubes:
                keep[i, int(start) * dt + int(span) * dt // 2] = 1.0
        keep = keep.to(mask.device, non_blocking=True)
        m = mask.to(torch.float32).repeat_interleave(dt, dim=1)
        return (m * keep[:, :, None, None]).contiguous()

    def forward(self, x, target_x, mask, cube_marker, visualize=False):
        if visualize:
            raise NotImplementedError('visualize=True is a debugging path of the reference ("need to update", :903)')
        return self.forward_with_center_mask(x, target_x, mask, self.center_frame_mask(mask.to(x.device), cube_marker))

    def forward_with_center_mask(self, x, target_x, mask, center_mask):
        """forward() after its host-side loop over `cube_marker`: device work only, so a whole training step can be
        captured in a CUDA graph (graph.GraphedTrainStep).  center_mask = self.center_frame_mask(mask, cube_marker)."""
        feats = self.forward_features(x, mask)
        dt = self.stride[0]
        t = self.num_frames // dt
        h = self.img_size // (self.stride[1] * self.downsample_rate)
        w = self.img_size // (self.stride[2] * self.downsample_rate)
        fdim = self.decoder_pred.out_features
        dc = fdim // dt
        B = x.shape[0]
        # the reference's targets are fp64 numpy arrays (dataset.py:190), which makes its loss fp64 (:899-901): fp64 targets
        # are kept and the loss kernel then works in fp64; anything else is taken in fp32
        tdt = torch.float64 if target_x.dtype == torch.float64 else torch.float32
        target = target_x.to(device=x.device, dtype=tdt).contiguous()
        m = center_mask.to(device=x.device, dtype=torch.float32).contiguous()
        pred, loss = mvit_ops.MaskedMSEFn.apply(feats, _f32(self.decoder_pred.weight), _f32(self.decoder_pred.bias),
                                                self._shadow.get('dec', self.decoder_pred.weight), target, m,
                                                (B, t, dt, h, w, dc))
        pred = pred[:, 1:].reshape(B, t, h, w, dt, dc).permute(0, 1, 4, 2, 3, 5).reshape(B, t * dt, h, w, dc)
        return pred, loss
