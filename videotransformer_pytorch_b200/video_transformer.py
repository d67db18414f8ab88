"""Model surface: TimeSformer and ViViT with the reference's constructor signatures, attribute names
and state-dict keys (reference video_transformer.py:20-268 and :270-557), forward/backward on the
sm_90a kernels.

Covered configurations (SURVEY.md §8a, §8f rank 4): TimeSformer `divided_space_time`, `space_only` (197-token joint
attention per frame) and `joint_space_time` (one 1569-token attention per clip, tiled tensor-core kernels); ViViT
`fact_encoder` (model 2), `joint_space_time` (model 1) and `divided_space_time` (model 3).  TimeSformer also takes clips
whose patch grid differs from img_size's (interpolate_pos_encoding, reference :171-191).  Nothing falls back to eager
PyTorch.
"""
from __future__ import annotations

import math

import torch
import torch.nn as nn

from . import ops
from .mixup import MixedClip
from .transformer import InferencePrecision, PatchEmbed, TransformerContainer, get_sine_cosine_pos_emb, _f32
from .weight_init import init_from_kinetics_pretrain_, init_from_vit_pretrain_, trunc_normal_


def _load_pretrained(module, **vit_kwargs):
    """reference video_transformer.py:154-165 / :434-451: image (ViT) or kinetics checkpoint by `weights_from`."""
    if module.pretrain_pth is None:
        return
    if module.weights_from == 'imagenet':
        init_from_vit_pretrain_(module, module.pretrain_pth, module.conv_type, module.attention_type, module.copy_strategy,
                                **vit_kwargs)
    elif module.weights_from == 'kinetics':
        init_from_kinetics_pretrain_(module, module.pretrain_pth)
    else:
        raise TypeError(f'not support the pretrained weight {module.pretrain_pth}')


class _ByteClipInput:
    """Models fed the decoder's uint8 clip [B, T, H, W, 3] (optionally wrapped in a mixup.MixedClip): ToTensor + Normalize
    (+ Mixup / CutMix) are folded into the patch-operand kernel."""

    def set_input_normalization(self, mean, std):
        """Normalisation applied when the model is fed the decoder's uint8 clip [B, T, H, W, 3] directly (the reference
        does it on the CPU: data_transform.py ToTensor + Normalize with data_trainer.py:69-73's mean / std)."""
        self._input_norm = (tuple(float(m) for m in mean), tuple(float(s) for s in std))
        self._input_norm_dev = None
        self._input_mean_std_dev = None

    def input_normalization(self):
        """(mean, std) tuples applied to uint8 clips; (0.45,) * 3 and (0.225,) * 3 until set_input_normalization."""
        return getattr(self, '_input_norm', ((0.45, 0.45, 0.45), (0.225, 0.225, 0.225)))

    def _norm_tensors(self, device):
        cached = getattr(self, '_input_norm_dev', None)
        if cached is None or cached[0].device != device:
            mean, std = self.input_normalization()
            scale = torch.tensor([1.0 / (255.0 * s) for s in std], dtype=torch.float32, device=device)
            shift = torch.tensor([-m / s for m, s in zip(mean, std)], dtype=torch.float32, device=device)
            cached = self._input_norm_dev = (scale, shift)
        return cached

    def input_mean_std(self, device):
        """The normalisation as fp32 device tensors (mean [C], std [C]), for kernels that apply the reference's
        (u / 255 - mean) / std op by op."""
        cached = getattr(self, '_input_mean_std_dev', None)
        if cached is None or cached[0].device != device:
            mean, std = self.input_normalization()
            cached = self._input_mean_std_dev = (torch.tensor(mean, dtype=torch.float32, device=device),
                                                 torch.tensor(std, dtype=torch.float32, device=device))
        return cached

    def _unwrap_clip(self, x, mean_std=False):
        """-> (tensor, (scale, shift) | None, mix plan | None); (mean, std) in place of (scale, shift) when mean_std"""
        plan = None
        if isinstance(x, MixedClip):
            x, plan = x.clip, x.plan
        norm = None
        if x.dtype == torch.uint8:
            norm = self.input_mean_std(x.device) if mean_std else self._norm_tensors(x.device)
        if plan is not None and norm is None:
            raise RuntimeError('MixedClip must wrap a uint8 clip (float clips are mixed by Mixup.__call__ itself)')
        return x, norm, plan


class _AttentionMaps:
    """The cls query's attention in the last attention layer, the product visualize_attention.py consumes
    (attentions[:, 0, 1:], :71, turned into heatmaps and threshold masks by show_attn, :66-102).  The model supplies
    _last_attention(x, return_attention) and _map_layout()."""

    def cls_attention(self, x):
        """get_last_selfattention(x)[:, :, 0, :], bit for bit: fp32 [B', H, N], without the [B', H, N, N] map.  Always the
        forward-only form: every block before the last runs as under no_grad (nothing saved), and the last runs only its
        LayerNorm, the qkv GEMM and vt_attn_cls_probs, where the reference's return_attention stops as well."""
        with torch.no_grad():
            return self._last_attention(x, 'cls')

    def attention_maps(self, x, threshold=0.6):
        """(heatmaps, masks) of the cls query over the patch tokens, per head, from cls_attention(x).

        Spatial maps use show_attn's own axis order: reshape(nh, w_featmap, h_featmap) with w_featmap = H // p and
        h_featmap = W // p for a clip of H x W pixels, kept as is.  Per-frame attention (divided_space_time, space_only)
        gives one map per frame, [B * T, nh, w_featmap, h_featmap] (frames in get_last_selfattention's order); joint
        attention (joint_space_time, token 1 + p * T + t) gives [B, nh, T, w_featmap, h_featmap] per clip.  ViViT's
        fact_encoder ends in the temporal encoder, whose 1 + T tokens are the cls and one token per frame: its result is
        the per-frame weight row [B, nh, T], not a spatial map.

        masks (None when threshold is None) has the heatmaps' shape: show_attn's float 0 / 1 mask keeping the largest
        probabilities of each (frame or clip, head) row until their mass exceeds threshold (vt_attn_mass_mask; a joint
        clip's row covers all its T * P patches).  Upsampling by the patch size is left to the caller
        (repeat_interleave on the last two axes is show_attn's nearest interpolation)."""
        cls = self.cls_attention(x)
        pat = cls[:, :, 1:]
        nh = pat.shape[1]
        kind, grid = self._map_layout(x)
        with torch.no_grad():
            masks = None if threshold is None else ops.maps_K().attn_mass_mask(pat, threshold)
            out = []
            for t in (pat, masks):
                if t is None:
                    out.append(None)
                elif kind == 'frame':
                    out.append(t.reshape(t.shape[0], nh, *grid))
                elif kind == 'clip':
                    T = t.shape[-1] // (grid[0] * grid[1])
                    out.append(t.reshape(t.shape[0], nh, grid[0] * grid[1], T).transpose(2, 3).reshape(t.shape[0], nh, T, *grid))
                else:
                    out.append(t.contiguous())
        return out[0], out[1]

    def _featmap(self, x):
        """(w_featmap, h_featmap) of show_attn: (H // p, W // p) of the clip"""
        clip = x.clip if isinstance(x, MixedClip) else x
        h, w = (clip.shape[2], clip.shape[3]) if clip.dtype == torch.uint8 else (clip.shape[3], clip.shape[4])
        p = self.patch_embed.patch_size
        return h // p[0], w // p[1]


class TimeSformer(_AttentionMaps, _ByteClipInput, InferencePrecision, nn.Module):
    """TimeSformer (divided space-time attention).  forward(x[B,T,3,H,W]) -> [B, embed_dims]."""

    supported_attention_types = ['divided_space_time', 'space_only', 'joint_space_time']

    def __init__(self, num_frames, img_size=224, patch_size=16, pretrain_pth=None, weights_from='imagenet',
                 embed_dims=768, num_heads=12, num_transformer_layers=12, in_channels=3, conv_type='Conv2d',
                 dropout_p=0., attention_type='divided_space_time', norm_layer=nn.LayerNorm, copy_strategy='repeat',
                 use_learnable_pos_emb=True, return_cls_token=True, **kwargs):
        super().__init__()
        assert attention_type in self.supported_attention_types, f'Unsupported Attention Type {attention_type}!'
        if dropout_p:
            raise NotImplementedError('dropout_p > 0 is not on the reference hot path (always 0.)')
        self.num_frames = num_frames
        self.pretrain_pth = pretrain_pth
        self.weights_from = weights_from
        self.embed_dims = embed_dims
        self.num_transformer_layers = num_transformer_layers
        self.attention_type = attention_type
        self.copy_strategy = copy_strategy
        self.conv_type = conv_type
        self.use_learnable_pos_emb = use_learnable_pos_emb
        self.return_cls_token = return_cls_token

        self.patch_embed = PatchEmbed(img_size=img_size, patch_size=patch_size, in_channels=in_channels,
                                      embed_dims=embed_dims, conv_type=conv_type)
        num_patches = self.patch_embed.num_patches
        operator_order = ['time_attn', 'space_attn', 'ffn'] if attention_type == 'divided_space_time' else ['self_attn', 'ffn']
        self.transformer_layers = TransformerContainer(
            num_transformer_layers=num_transformer_layers, embed_dims=embed_dims, num_heads=num_heads,
            num_frames=num_frames, norm_layer=norm_layer, hidden_channels=embed_dims * 4,
            operator_order=operator_order)
        self.norm = norm_layer(embed_dims, eps=1e-6)

        self.cls_token = nn.Parameter(torch.zeros(1, 1, embed_dims))
        self.use_cls_token_temporal = operator_order[-2] == 'time_attn'     # False: cls lives in pos_embed
        num_patches = num_patches + 1
        if use_learnable_pos_emb:
            self.pos_embed = nn.Parameter(torch.zeros(1, num_patches, embed_dims))
        else:
            self.pos_embed = get_sine_cosine_pos_emb(num_patches, embed_dims)
        self.drop_after_pos = nn.Dropout(p=dropout_p)
        if attention_type != 'space_only':          # space_only has no temporal embedding (reference :137-142)
            if use_learnable_pos_emb:
                self.time_embed = nn.Parameter(torch.zeros(1, num_frames, embed_dims))
            else:
                self.time_embed = get_sine_cosine_pos_emb(num_frames, embed_dims)
            self.drop_after_time = nn.Dropout(p=dropout_p)
        self.init_weights()

    def init_weights(self):
        if self.use_learnable_pos_emb:
            nn.init.trunc_normal_(self.pos_embed, std=.02)
            if self.attention_type != 'space_only':
                nn.init.trunc_normal_(self.time_embed, std=.02)
        trunc_normal_(self.cls_token, std=.02)
        _load_pretrained(self)

    @torch.jit.ignore
    def no_weight_decay_keywords(self):
        return {'pos_embed', 'cls_token', 'mask_token'}

    def interpolate_pos_encoding(self, x, w, h):
        """reference video_transformer.py:171-191.  x: the tokens, or any tensor whose dim 1 is 1 + the input's patch
        count; w, h: the clip's width and height."""
        return self._interpolate(self.pos_embed, x.shape[1] - 1, w, h)

    def _interpolate(self, pos, npatch, w, h):
        """pos unchanged when the input has the training grid, else its patch rows (a sqrt(N) x sqrt(N) grid) resized
        bicubically to (w // p) rows x (h // p) columns with the reference's scale factors ((n + 0.1) / sqrt(N)).  The
        resized grid is flattened row-major and added to patch tokens in Conv2d order (h // p rows of w // p): for w != h
        token i takes cell (i // (h // p), i % (h // p)), the reference's axis order, reproduced as is."""
        N = pos.shape[1] - 1
        if npatch == N and w == h:
            return pos
        g = math.isqrt(N)
        if g * g != N:
            raise ValueError(f'pos_embed holds {N} patch rows, which is not a square grid: it cannot be interpolated')
        p = self.patch_embed.patch_size[0]
        w0, h0 = w // p, h // p
        scales = ((w0 + 0.1) / math.sqrt(N), (h0 + 0.1) / math.sqrt(N))
        out_grid = (math.floor(g * scales[0]), math.floor(g * scales[1]))      # F.interpolate's output size
        if out_grid != (w0, h0) or w0 < 1 or h0 < 1:
            raise ValueError(f'cannot resize the {g}x{g} position grid to {w0}x{h0}')
        return ops.PosResizeFn.apply(pos, (g, g), out_grid, scales)

    def _embeds(self, x):
        pos = self.pos_embed
        tim = self.time_embed if self.attention_type != 'space_only' else None
        if not self.use_learnable_pos_emb:
            pos = pos.to(x.device).detach()
            tim = None if tim is None else tim.to(x.device).detach()
        return pos, tim

    def prepare_tokens(self, x):
        x, norm, plan = self._unwrap_clip(x)
        if norm is not None:                # [B, T, H, W, C] bytes
            b, t, h, w, c = x.shape
        else:
            b, t, c, h, w = x.shape
        ps = self.patch_embed.patch_size
        if h % ps[0] or w % ps[1]:
            raise ValueError(f'clip sides {h}x{w} must be multiples of the patch size {ps[0]}x{ps[1]}')
        if self.attention_type != 'space_only' and t != self.num_frames:
            raise ValueError(f'{self.attention_type} model of {self.num_frames} frames fed a clip of {t} frames')
        pos, tim = self._embeds(x)
        pos = self._interpolate(pos, (h // ps[0]) * (w // ps[1]), w, h)
        pe = self.patch_embed
        mode = 'frames' if self.attention_type == 'space_only' else 'timesformer'   # space_only: per-frame tokens
        tok = ops.run(ops.PatchTokensFn, x, _f32(pe.projection.weight), _f32(pe.projection.bias), self.cls_token, pos, tim,
                                      pe.shadow(), mode, 1, norm, plan)
        return tok, b

    def forward(self, x):
        x, b = self.prepare_tokens(x)
        x = self.transformer_layers(x)
        if self.attention_type == 'space_only':      # '(b t) p d -> b p d' mean over frames (reference :247-249)
            x = x.view(b, x.shape[0] // b, x.shape[1], x.shape[2]).mean(dim=1)
        S = x.shape[1]
        if self.return_cls_token:
            if self.attention_type == 'space_only':
                rows = (torch.arange(b, device=x.device, dtype=torch.int32) * S).contiguous()
                return ops.run(ops.RowsNormFn, x, _f32(self.norm.weight), _f32(self.norm.bias), self.norm.eps, rows)
            rows = ops.token_maps(b, self.num_frames, (S - 1) // self.num_frames, str(x.device))['cls_rows']
            return ops.run(ops.RowsNormFn, x, _f32(self.norm.weight), _f32(self.norm.bias), self.norm.eps, rows)
        y = ops.run(ops.RowsNormFn, x, _f32(self.norm.weight), _f32(self.norm.bias), self.norm.eps, None)
        return y.view(b, S, -1)[:, 1:].mean(1)

    def get_last_selfattention(self, x):
        """fp32 [B', H, N, N] probabilities of the last attention layer.  Without autograd recording (no_grad /
        inference_mode, or nothing requiring grad) the blocks take their forward-only form and the last layer stops
        after its probabilities; the result is the same either way."""
        return self._last_attention(x, True)

    def _last_attention(self, x, return_attention):
        x, b = self.prepare_tokens(x)
        return self.transformer_layers(x, return_attention=return_attention)

    def _map_layout(self, x):
        return ('clip' if self.attention_type == 'joint_space_time' else 'frame'), self._featmap(x)


def get_vit_base_patch16_224(**kwargs):
    return TimeSformer(num_frames=kwargs['num_frames'], pretrain_pth=kwargs['pretrain_pth'],
                       weights_from=kwargs['weights_from'], img_size=kwargs['img_size'],
                       attention_type=kwargs['attention_type'], patch_size=16, embed_dims=768, num_heads=12,
                       in_channels=3, num_transformer_layers=12, conv_type='Conv2d', dropout_p=0.,
                       norm_layer=nn.LayerNorm, copy_strategy='repeat', use_learnable_pos_emb=True,
                       return_cls_token=True)


class ViViT(_AttentionMaps, _ByteClipInput, InferencePrecision, nn.Module):
    """ViViT factorised encoder (model 2): tubelet embed -> 12 spatial layers per frame ->
    frame tokens (+ the reference's `x[:b,0,:]` cls gather) -> 4 temporal layers."""

    supported_attention_types = ['fact_encoder', 'joint_space_time', 'divided_space_time']

    def __init__(self, num_frames, img_size=224, patch_size=16, pretrain_pth=None, weights_from='imagenet',
                 embed_dims=768, num_heads=12, num_transformer_layers=12, in_channels=3, dropout_p=0., tube_size=2,
                 conv_type='Conv3d', attention_type='fact_encoder', norm_layer=nn.LayerNorm, copy_strategy='repeat',
                 extend_strategy='temporal_avg', use_learnable_pos_emb=True, return_cls_token=True, **kwargs):
        super().__init__()
        assert attention_type in self.supported_attention_types, f'Unsupported Attention Type {attention_type}!'
        if dropout_p:
            raise NotImplementedError('dropout_p > 0 is not on the reference hot path (always 0.)')
        if conv_type != 'Conv3d':
            raise NotImplementedError('ViViT hot path uses the Conv3d tubelet embedding')
        num_frames = num_frames // tube_size
        self.num_frames = num_frames
        self.pretrain_pth = pretrain_pth
        self.weights_from = weights_from
        self.embed_dims = embed_dims
        self.num_transformer_layers = num_transformer_layers
        self.attention_type = attention_type
        self.conv_type = conv_type
        self.copy_strategy = copy_strategy
        self.extend_strategy = extend_strategy
        self.tube_size = tube_size
        self.num_time_transformer_layers = 4 if attention_type == 'fact_encoder' else 0
        self.use_learnable_pos_emb = use_learnable_pos_emb
        self.return_cls_token = return_cls_token

        self.patch_embed = PatchEmbed(img_size=img_size, patch_size=patch_size, in_channels=in_channels,
                                      embed_dims=embed_dims, tube_size=tube_size, conv_type=conv_type)
        num_patches = self.patch_embed.num_patches
        mk = lambda n, order: TransformerContainer(
            num_transformer_layers=n, embed_dims=embed_dims, num_heads=num_heads, num_frames=num_frames,
            norm_layer=norm_layer, hidden_channels=embed_dims * 4, operator_order=order)
        if attention_type == 'divided_space_time':          # model 3 (reference :349-360)
            self.transformer_layers = mk(num_transformer_layers, ['time_attn', 'space_attn', 'ffn'])
        elif attention_type == 'joint_space_time':          # model 1 (:361-373): one 1+P*T' token attention per clip
            self.transformer_layers = mk(num_transformer_layers, ['self_attn', 'ffn'])
        else:                                               # model 2, factorised encoder (:374-400)
            self.transformer_layers = nn.ModuleList([mk(num_transformer_layers, ['self_attn', 'ffn']),
                                                     mk(self.num_time_transformer_layers, ['self_attn', 'ffn'])])
        self.norm = norm_layer(embed_dims, eps=1e-6)
        self.cls_token = nn.Parameter(torch.zeros(1, 1, embed_dims))
        # reference :405-416: only fact_encoder has a cls slot in time_embed; operator_order[-2] is never 'time_attn'
        self.use_cls_token_temporal = False
        n_time = num_frames + 1 if attention_type == 'fact_encoder' else num_frames
        if use_learnable_pos_emb:
            self.pos_embed = nn.Parameter(torch.zeros(1, num_patches + 1, embed_dims))
            self.time_embed = nn.Parameter(torch.zeros(1, n_time, embed_dims))
        else:
            self.pos_embed = get_sine_cosine_pos_emb(num_patches + 1, embed_dims)
            self.time_embed = get_sine_cosine_pos_emb(n_time, embed_dims)
        self.drop_after_pos = nn.Dropout(p=dropout_p)
        self.drop_after_time = nn.Dropout(p=dropout_p)
        self.init_weights()

    def init_weights(self):
        if self.use_learnable_pos_emb:
            nn.init.trunc_normal_(self.pos_embed, std=.02)
            nn.init.trunc_normal_(self.time_embed, std=.02)
        trunc_normal_(self.cls_token, std=.02)
        _load_pretrained(self, extend_strategy=self.extend_strategy, tube_size=self.tube_size,
                         num_time_transformer_layers=self.num_time_transformer_layers)

    @torch.jit.ignore
    def no_weight_decay_keywords(self):
        return {'pos_embed', 'cls_token', 'mask_token'}

    def prepare_tokens(self, x):
        x, norm, plan = self._unwrap_clip(x)
        b = x.shape[0]
        h, w = (x.shape[2], x.shape[3]) if norm is not None else (x.shape[3], x.shape[4])
        ps = self.patch_embed.patch_size
        if (h // ps[0]) * (w // ps[1]) != self.patch_embed.num_patches:
            # no pos_embed interpolation in ViViT: the reference fails on `x + self.pos_embed` (:464-473)
            raise ValueError(f'ViViT built for img_size {self.patch_embed.img_size} got a {h}x{w} clip')
        pos = self.pos_embed if self.use_learnable_pos_emb else self.pos_embed.to(x.device).detach()
        pe = self.patch_embed
        if self.attention_type == 'fact_encoder':
            tok = ops.run(ops.PatchTokensFn, x, _f32(pe.projection.weight), _f32(pe.projection.bias), self.cls_token, pos, None,
                                          pe.shadow(), 'frames', self.tube_size, norm, plan)
        else:
            # reference :476-499 with use_cls_token_temporal False == TimeSformer's assembly on tubelets: one cls,
            # tokens 'b (p t) d', pos_embed per patch + time_embed per tubelet (fused into the patch GEMM epilogue)
            tim = self.time_embed if self.use_learnable_pos_emb else self.time_embed.to(x.device).detach()
            tok = ops.run(ops.PatchTokensFn, x, _f32(pe.projection.weight), _f32(pe.projection.bias), self.cls_token, pos, tim,
                                          pe.shadow(), 'timesformer', self.tube_size, norm, plan)
        cls_tokens = self.cls_token.expand(tok.shape[0], -1, -1)
        return tok, cls_tokens, b

    def _temporal_tokens(self, x, b):
        # reference video_transformer.py:515-523.  NOTE the quirk at :515: `x[:b, 0, :]` indexes the
        # (b t)-major tensor, i.e. it takes the cls of sample 0 / frames 0..b-1 — reproduced, not fixed.
        cls_tokens = x[:b, 0, :].unsqueeze(1)
        tim = self.time_embed if self.use_learnable_pos_emb else self.time_embed.to(x.device).detach()
        frames = x[:, 1:, :].reshape(b, x.shape[0] // b, x.shape[1] - 1, x.shape[2]).mean(dim=2)
        return torch.cat((cls_tokens, frames), dim=1) + tim

    def forward(self, x):
        x, cls_tokens, b = self.prepare_tokens(x)
        if self.attention_type != 'fact_encoder':
            x = self.transformer_layers(x)
        else:
            spatial, temporal = self.transformer_layers
            x = spatial(x)
            x = self._temporal_tokens(x, b)
            x = temporal(x)
        if self.return_cls_token:
            S = x.shape[1]
            rows = (torch.arange(b, device=x.device, dtype=torch.int32) * S).contiguous()
            return ops.run(ops.RowsNormFn, x, _f32(self.norm.weight), _f32(self.norm.bias), self.norm.eps, rows)
        y = ops.run(ops.RowsNormFn, x, _f32(self.norm.weight), _f32(self.norm.bias), self.norm.eps, None)
        return y.view(x.shape)[:, 1:].mean(1)

    def get_last_selfattention(self, x):
        """fp32 [B', H, N, N] probabilities of the last attention layer (fact_encoder: the temporal encoder's); forward-only
        without autograd recording, as TimeSformer.get_last_selfattention."""
        return self._last_attention(x, True)

    def _last_attention(self, x, return_attention):
        x, cls_tokens, b = self.prepare_tokens(x)
        if self.attention_type != 'fact_encoder':
            return self.transformer_layers(x, return_attention=return_attention)
        spatial, temporal = self.transformer_layers
        x = spatial(x)
        x = self._temporal_tokens(x, b)
        return temporal(x, return_attention=return_attention)

    def _map_layout(self, x):
        kind = {'fact_encoder': 'row', 'joint_space_time': 'clip'}.get(self.attention_type, 'frame')
        return kind, self._featmap(x)
