"""Batch-level Mixup / CutMix (reference mixup.py:58-126, used at model_trainer.py:87-89, :142-143).

Same constructor and call surface as the reference's `Mixup`, same numpy RNG stream (the draws happen in the same order:
`rand()` apply?, `rand()` cutmix?, `beta()`, and for CutMix `randint()` cy, cx), so for equal `np.random.seed` the lambda,
the box and the soft targets are identical to the reference's.

Two input kinds:
  * float clips [B,T,C,H,W] / [B,C,H,W] (the reference's path, after CPU normalisation): mixed in place with the same
    tensor ops as the reference; returns (x, soft_target).
  * uint8 clips [B,T,H,W,3] straight from the decoder (SURVEY §8f rank 2): nothing is touched here — the draw is
    packaged as a `MixedClip` (clip + a 6-float device plan) that TimeSformer / ViViT / MaskFeat consume; the blend with
    the flipped batch then happens inside the patch-operand kernel (`vt_im2col_u8_mix_bf16`, `vt_im2col3d_u8_bf16`)
    together with ToTensor + Normalize, so the mixed fp32 clip never exists in memory.
"""
from __future__ import annotations

import numpy as np
import torch


def one_hot(x, num_classes, on_value=1., off_value=0., device='cuda'):
    x = x.long().view(-1, 1)
    return torch.full((x.size()[0], num_classes), off_value, device=device).scatter_(1, x, on_value)


def mixup_target(target, num_classes, lam=1., smoothing=0.0, device='cuda'):
    """lam * smooth_one_hot(target) + (1 - lam) * smooth_one_hot(target.flip(0))   (mixup.py:19-24)"""
    off = smoothing / num_classes
    on = 1. - smoothing + off
    y1 = one_hot(target, num_classes, on_value=on, off_value=off, device=device)
    y2 = one_hot(target.flip(0), num_classes, on_value=on, off_value=off, device=device)
    return y1 * lam + y2 * (1. - lam)


def rand_bbox(img_shape, lam, margin=0., count=None):
    """CutMix box with side ratio sqrt(1 - lam) around a uniformly drawn centre, clipped to the image (mixup.py:26-48)."""
    ratio = np.sqrt(1 - lam)
    img_h, img_w = img_shape[-2:]
    cut_h, cut_w = int(img_h * ratio), int(img_w * ratio)
    margin_y, margin_x = int(margin * cut_h), int(margin * cut_w)
    cy = np.random.randint(0 + margin_y, img_h - margin_y, size=count)
    cx = np.random.randint(0 + margin_x, img_w - margin_x, size=count)
    yl = np.clip(cy - cut_h // 2, 0, img_h)
    yh = np.clip(cy + cut_h // 2, 0, img_h)
    xl = np.clip(cx - cut_w // 2, 0, img_w)
    xh = np.clip(cx + cut_w // 2, 0, img_w)
    return yl, yh, xl, xh


def cutmix_bbox_and_lam(img_shape, lam, correct_lam=True, count=None):
    yl, yu, xl, xu = rand_bbox(img_shape, lam, count=count)
    if correct_lam:
        lam = 1. - (yu - yl) * (xu - xl) / float(img_shape[-2] * img_shape[-1])
    return (yl, yu, xl, xu), lam


class MixedClip:
    """uint8 clip [B,T,H,W,3] + this step's mix draw.  `plan` = fp32 [6] {mode (0 none / 1 mixup / 2 cutmix), lam, yl, yh,
    xl, xh}; kept in a caller-provided device buffer when given, so a captured CUDA graph sees every step's values."""

    def __init__(self, clip, mode, lam, box, plan_out=None):
        self.clip = clip
        self.mode, self.lam, self.box = mode, float(lam), tuple(int(v) for v in box)
        host = torch.tensor([float(mode), float(lam), *[float(v) for v in self.box]], dtype=torch.float32)
        if plan_out is not None:
            plan_out.copy_(host, non_blocking=True)
            self.plan = plan_out
        else:
            self.plan = host.to(clip.device, non_blocking=True)

    @property
    def shape(self):
        return self.clip.shape

    @property
    def device(self):
        return self.clip.device

    @property
    def dtype(self):
        return self.clip.dtype


class Mixup:
    def __init__(self, mixup_alpha=0.8, cutmix_alpha=1.0, prob=1.0, switch_prob=0.5, mode='batch', correct_lam=True,
                 label_smoothing=0.1, num_classes=1000):
        if mode != 'batch':
            raise NotImplementedError("only mode='batch' exists in the reference (mixup.py:102-114)")
        self.mixup_alpha = mixup_alpha
        self.cutmix_alpha = cutmix_alpha
        self.mix_prob = prob
        self.switch_prob = switch_prob
        self.label_smoothing = label_smoothing
        self.num_classes = num_classes
        self.mode = mode
        self.correct_lam = correct_lam
        self.mixup_enabled = True

    def _params_per_batch(self):
        lam, use_cutmix = 1., False
        if self.mixup_enabled and np.random.rand() < self.mix_prob:
            if self.mixup_alpha > 0. and self.cutmix_alpha > 0.:
                use_cutmix = np.random.rand() < self.switch_prob
                a = self.cutmix_alpha if use_cutmix else self.mixup_alpha
            elif self.mixup_alpha > 0.:
                a = self.mixup_alpha
            elif self.cutmix_alpha > 0.:
                use_cutmix, a = True, self.cutmix_alpha
            else:
                assert False, 'One of mixup_alpha > 0., cutmix_alpha > 0.'
            lam = float(np.random.beta(a, a))
        return lam, use_cutmix

    def draw(self, img_hw):
        """This step's (mode, lam, (yl, yh, xl, xh)) for images of size img_hw, consuming the numpy RNG like the reference."""
        lam, use_cutmix = self._params_per_batch()
        if lam == 1.:
            return 0, 1., (0, 0, 0, 0)
        if use_cutmix:
            (yl, yh, xl, xh), lam = cutmix_bbox_and_lam(tuple(img_hw), lam, correct_lam=self.correct_lam)
            return 2, float(lam), (int(yl), int(yh), int(xl), int(xh))
        return 1, lam, (0, 0, 0, 0)

    def __call__(self, x, target, plan_out=None):
        assert len(x) % 2 == 0, 'Batch size should be even when using this'
        if x.dtype == torch.uint8:                      # [B, T, H, W, 3] bytes: mixed inside the patch-operand kernel
            if x.ndim != 5 or x.shape[-1] != 3:
                raise RuntimeError('Mixup: uint8 clips must be [B, T, H, W, 3]')
            mode, lam, box = self.draw(x.shape[2:4])
            mixed = MixedClip(x, mode, lam, box, plan_out)
        else:
            shape = x.shape
            if x.ndim == 5:
                b, t, c, h, w = shape
                x = x.view(b, t * c, h, w)
            mode, lam, (yl, yh, xl, xh) = self.draw(x.shape[-2:])
            if mode == 2:
                x[:, :, yl:yh, xl:xh] = x.flip(0)[:, :, yl:yh, xl:xh]
            elif mode == 1:
                x_flipped = x.flip(0).mul_(1. - lam)
                x.mul_(lam).add_(x_flipped)
            mixed = x.view(shape)
        return mixed, mixup_target(target, self.num_classes, lam, self.label_smoothing, x.device)
