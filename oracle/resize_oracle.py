"""Plain-torch CPU restatement of TimeSformer at input sizes other than img_size.

TEST INFRASTRUCTURE (see oracle/__init__.py).  TimeSformer.prepare_tokens sends every input through
interpolate_pos_encoding (reference video_transformer.py:171-191, :207-211): when the clip's patch grid is not the one
img_size built, the patch rows of pos_embed are resized bicubically.  The forwards below are those of
``oracle/vt_oracle.py`` with that resize restated; at the training grid they compute exactly what vt_oracle does.  The
blocks, containers and primitives are vt_oracle's own.

Pinned against the real reference class by ``oracle/make_resize_golden.py``; the vectors live in
``tests/golden/resize_*.npz``.
"""
from __future__ import annotations

import math

import torch

from oracle.vt_oracle import container, layer_norm, patch_embed

Tensor = torch.Tensor


def interpolate_pos_encoding(pos: Tensor, npatch: int, w: int, h: int, patch: int) -> Tensor:
    """TimeSformer.interpolate_pos_encoding, video_transformer.py:171-191.  Computed in the table's own dtype, as the
    reference does (its fixed sine-cosine table is fp32 and is cast after the resize, :211)."""
    N = pos.shape[1] - 1
    if npatch == N and w == h:                                            # :174-175
        return pos
    dim = pos.shape[-1]
    w0, h0 = w // patch + 0.1, h // patch + 0.1                           # :179-183
    g = int(math.sqrt(N))
    grid = pos[:, 1:].reshape(1, g, g, dim).permute(0, 3, 1, 2)
    grid = torch.nn.functional.interpolate(grid, scale_factor=(w0 / math.sqrt(N), h0 / math.sqrt(N)),
                                           mode='bicubic')               # :184-188
    assert int(w0) == grid.shape[-2] and int(h0) == grid.shape[-1]
    return torch.cat((pos[:, :1], grid.permute(0, 2, 3, 1).reshape(1, -1, dim)), dim=1)   # :190-191


def pos_for(sd, x, npatch):
    """pos_embed as prepare_tokens adds it (:207-211) for a clip x [B, T, C, H, W]."""
    return interpolate_pos_encoding(sd['pos_embed'], npatch, x.shape[-1], x.shape[-2],
                                    sd['patch_embed.projection.weight'].shape[-2]).to(x.dtype)


def timesformer_tokens(sd, x, cfg):
    """TimeSformer.prepare_tokens (divided / joint space-time), video_transformer.py:193-240, any input size."""
    B = x.shape[0]
    tok = patch_embed(x, sd['patch_embed.projection.weight'], sd['patch_embed.projection.bias'])
    BT, P, D = tok.shape
    T = BT // B
    cls = sd['cls_token'].expand(BT, 1, D)
    tok = torch.cat((cls, tok), dim=1) + pos_for(sd, x, P)                # :207-211
    cls_tokens = tok[:B, 0, :].unsqueeze(1)                               # :216
    tok = tok[:, 1:, :].reshape(B, T, P, D).permute(0, 2, 1, 3).reshape(B * P, T, D)  # :231
    tok = tok + sd['time_embed']                                          # :233 (T must be num_frames)
    tok = tok.reshape(B, P * T, D)                                        # :236
    return torch.cat((cls_tokens, tok), dim=1)                            # :237


def timesformer_forward(sd, x, cfg, training=False):
    """TimeSformer.forward, attention_type='divided_space_time' (video_transformer.py:242-256)."""
    tok = timesformer_tokens(sd, x, cfg)
    tok = container(tok, sd, 'transformer_layers.', cfg['num_transformer_layers'], ['time_attn', 'space_attn', 'ffn'],
                    cfg['num_frames'], cfg['num_heads'], training)
    return layer_norm(tok, sd['norm.weight'], sd['norm.bias'], 1e-6)[:, 0]


def timesformer_joint_forward(sd, x, cfg, training=False):
    """TimeSformer.forward, attention_type='joint_space_time'."""
    tok = timesformer_tokens(sd, x, cfg)
    tok = container(tok, sd, 'transformer_layers.', cfg['num_transformer_layers'], ['self_attn', 'ffn'],
                    cfg['num_frames'], cfg['num_heads'], training)
    return layer_norm(tok, sd['norm.weight'], sd['norm.bias'], 1e-6)[:, 0]


def timesformer_space_only_forward(sd, x, cfg, training=False):
    """TimeSformer.forward, attention_type='space_only': per-frame tokens, no time embedding, mean over frames
    (video_transformer.py:193-212, :242-256)."""
    B, T = x.shape[0], x.shape[1]
    tok = patch_embed(x, sd['patch_embed.projection.weight'], sd['patch_embed.projection.bias'])
    BT, P, D = tok.shape
    tok = torch.cat((sd['cls_token'].expand(BT, 1, D), tok), dim=1) + pos_for(sd, x, P)        # :207-211
    tok = container(tok, sd, 'transformer_layers.', cfg['num_transformer_layers'], ['self_attn', 'ffn'],
                    cfg['num_frames'], cfg['num_heads'], training)
    tok = tok.reshape(B, T, P + 1, D).mean(dim=1)                                               # :248-249
    return layer_norm(tok, sd['norm.weight'], sd['norm.bias'], 1e-6)[:, 0]


def timesformer_last_selfattention(sd, x, cfg):
    """TimeSformer.get_last_selfattention (divided space-time), video_transformer.py:258-261, any input size."""
    tok = timesformer_tokens(sd, x, cfg)
    return container(tok, sd, 'transformer_layers.', cfg['num_transformer_layers'], ['time_attn', 'space_attn', 'ffn'],
                     cfg['num_frames'], cfg['num_heads'], False, return_attention=True)


FORWARD = {'divided_space_time': timesformer_forward, 'space_only': timesformer_space_only_forward,
           'joint_space_time': timesformer_joint_forward}
