#!/usr/bin/env python
"""MaskFeat / MViT fed the decoder's uint8 clip: the Conv3d patch operand from bytes (vt_im2col3d_u8_bf16) against the
float route it replaces, and the graphed steps built on each.

    python tools/mvit_u8_input.py [--iters 50] [--rounds 5] [--steps 10]

Prints one JSON line per measurement, after a line with the card's name and power limit read in the same run.
  * operand: ms per call at 16 x 224^2 (batch 16 and 8) of the new kernel (no plan, Mixup, CutMix) and of the float route
    (ATen normalise as bench.py's maskfeat arm does it, permute copy, vt_im2col3d_bf16), CUDA events around `iters`
    back-to-back calls, arms alternating, median of `rounds`; with the bytes each moves and the multiple of the data-sheet
    byte floor (3.35 TB/s).
  * pretrain_step: GraphedTrainStep of the MaskFeat pre-training step (batch 16) fed the uint8 clip, and fed the clip
    normalised as bench.py does it (the normalisation inside the timed window, like bench's prepare); step_peak_gb is the
    peak allocation each arm adds (its input, its capture and a replay) over what was allocated before it.
  * mixup_step: GraphedTrainStep of the MViT-B + 400-class head Mixup step (batch 8): Mixup on the uint8 batch (the draw
    through plan_out) against the reference's float Mixup on the normalised clip.
"""
from __future__ import annotations

import argparse
import json
import os
import random
import statistics
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))

from resolution_step import card  # noqa: E402

MEAN, STD = (0.45,) * 3, (0.225,) * 3
FILTER = ((3, 7, 7), (2, 4, 4), (1, 3, 3))
KPAD = 448
HBM = 3.35e12
MASKFEAT_KW = dict(pool_q_stride_size=[[1, 1, 2, 2], [3, 1, 2, 2]], feature_dim=2 * 2 * 2 * 3 * 9)


def timed(fn, iters):
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(iters):
        fn()
    t1.record()
    torch.cuda.synchronize()
    return t0.elapsed_time(t1) / iters


def alternate(arms, iters, rounds):
    """ms per call of each arm: the arms take turns within every round; median and range over the rounds."""
    for fn in arms.values():
        fn()
    torch.cuda.synchronize()
    res = {k: [] for k in arms}
    for _ in range(rounds):
        for k, fn in arms.items():
            res[k].append(timed(fn, iters))
    return {k: dict(ms=statistics.median(v), lo=min(v), hi=max(v)) for k, v in res.items()}


def bench_normalise(u8):
    """bench.py's maskfeat arm: ToTensor + Normalize with ATen ops on the device, then the [B, T, C, H, W] copy."""
    return ((u8.float() * (1.0 / (255.0 * 0.225)) - 0.45 / 0.225)).permute(0, 1, 4, 2, 3).contiguous()


def operand(B, iters, rounds):
    from videotransformer_pytorch_b200 import _lib
    K = _lib.K
    u8 = torch.randint(0, 256, (B, 16, 224, 224, 3), dtype=torch.uint8, device='cuda')
    mean, std = torch.tensor(MEAN, device='cuda'), torch.tensor(STD, device='cuda')
    plans = {'mixup': torch.tensor([1, 0.37, 0, 0, 0, 0], device='cuda'),
             'cutmix': torch.tensor([2, 0.6, 40, 182, 30, 172], device='cuda')}
    arms = {'u8': lambda: K.im2col3d_u8(u8, mean, std, None, *FILTER, KPAD),
            'u8_mixup': lambda: K.im2col3d_u8(u8, mean, std, plans['mixup'], *FILTER, KPAD),
            'u8_cutmix': lambda: K.im2col3d_u8(u8, mean, std, plans['cutmix'], *FILTER, KPAD),
            'float_route': lambda: K.im2col3d(bench_normalise(u8), *FILTER, KPAD)}
    times = alternate(arms, iters, rounds)
    clip = u8.numel()
    cols = B * 8 * 56 * 56 * KPAD * 2
    moved = {'u8': clip + cols, 'u8_mixup': 2 * clip + cols, 'u8_cutmix': 2 * clip + cols,
             # u8 read + fp32 write, fp32 read + fp32 write (permute copy), fp32 read + cols write
             'float_route': clip + 4 * clip + 8 * clip + 4 * clip + cols}
    for k, t in times.items():
        floor_ms = moved[k] / HBM * 1e3
        print(json.dumps(dict(measure='operand', batch=B, arm=k, ms=round(t['ms'], 4), lo=round(t['lo'], 4),
                              hi=round(t['hi'], 4), bytes=moved[k], floor_ms=round(floor_ms, 4),
                              x_floor=round(t['ms'] / floor_ms, 2))), flush=True)


class Pretrain(torch.nn.Module):
    def __init__(self, net):
        super().__init__()
        self.net = net

    def forward(self, x, target, mask, cmask):
        return self.net.forward_with_center_mask(x, target, mask, cmask)[1]


def pretrain_step(steps, rounds):
    from videotransformer_pytorch_b200 import MaskFeat
    from videotransformer_pytorch_b200.graph import GraphedTrainStep
    from videotransformer_pytorch_b200.hog import hog_targets_batch
    from videotransformer_pytorch_b200.mask_generator import CubeMaskGenerator
    B = 16
    torch.manual_seed(0)
    net = MaskFeat(**MASKFEAT_KW).cuda().train()
    net.set_input_normalization(MEAN, STD)
    gen = CubeMaskGenerator((8, 14, 14), min_num_patches=16)
    random.seed(0)
    masks, markers = zip(*(gen() for _ in range(B)))
    mask = torch.from_numpy(np.stack(masks)).float().cuda()
    u8 = torch.randint(0, 256, (B, 16, 224, 224, 3), dtype=torch.uint8, device='cuda')
    target = hog_targets_batch(u8, markers)
    cmask = net.center_frame_mask(mask, markers)
    step = {}
    peak = {}
    for arm in ('u8', 'float'):
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        x0 = u8 if arm == 'u8' else bench_normalise(u8)
        step[arm] = GraphedTrainStep(Pretrain(net), (x0, target, mask, cmask))
        step[arm](x0, target, mask, cmask)
        torch.cuda.synchronize()
        peak[arm] = torch.cuda.max_memory_allocated() - base       # what this arm's capture and replay add
    arms = {'u8': lambda: step['u8'](u8, target, mask, cmask),
            'float': lambda: step['float'](bench_normalise(u8), target, mask, cmask)}
    times = alternate(arms, steps, rounds)
    for k, t in times.items():
        print(json.dumps(dict(measure='pretrain_step', batch=B, arm=k, ms=round(t['ms'], 3), lo=round(t['lo'], 3),
                              hi=round(t['hi'], 3), step_peak_gb=round(peak[k] / 1e9, 2))), flush=True)


class MixStep(torch.nn.Module):
    def __init__(self, net, head):
        super().__init__()
        self.net, self.head = net, head

    def forward(self, x, plan, y):
        from videotransformer_pytorch_b200 import MixedClip
        if plan is not None and x.dtype == torch.uint8:
            mc = MixedClip.__new__(MixedClip)                 # the static clip + plan the graph reads
            mc.clip, mc.plan = x, plan
            x = mc
        return self.head.loss(self.net.forward_features(x)[:, 0], y)


def mixup_step(steps, rounds):
    from videotransformer_pytorch_b200 import ClassificationHead, MaskFeat, Mixup
    from videotransformer_pytorch_b200.graph import GraphedTrainStep
    B = 8
    torch.manual_seed(0)
    net = MaskFeat(**MASKFEAT_KW).cuda().train()
    net.set_input_normalization(MEAN, STD)
    head = ClassificationHead(400, net.mvit.norm_embed.normalized_shape[0]).cuda()
    mod = MixStep(net, head)
    mix = Mixup(num_classes=400)
    u8 = torch.randint(0, 256, (B, 16, 224, 224, 3), dtype=torch.uint8, device='cuda')
    labels = torch.randint(0, 400, (B,), device='cuda')
    np.random.seed(0)
    plan = torch.zeros(6, device='cuda')
    _, y = mix(u8, labels, plan_out=plan)
    used = [p for n, p in mod.named_parameters() if not n.startswith('net.decoder_pred')]   # not in forward_features
    g8 = GraphedTrainStep(mod, (u8, plan, y), params=used)
    dummy = torch.zeros(6, device='cuda')
    xf, yf = mix(bench_normalise(u8), labels)
    gf = GraphedTrainStep(mod, (xf, dummy, yf), params=used)
    sp = g8.static_inputs[1]

    def run_u8():
        _, y = mix(u8, labels, plan_out=sp)
        g8(u8, sp, y)

    def run_float():
        xm, y = mix(bench_normalise(u8), labels)
        gf(xm, dummy, y)

    times = alternate({'u8': run_u8, 'float': run_float}, steps, rounds)
    for k, t in times.items():
        print(json.dumps(dict(measure='mixup_step', batch=B, arm=k, ms=round(t['ms'], 3), lo=round(t['lo'], 3),
                              hi=round(t['hi'], 3))), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=50)
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--steps', type=int, default=10)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('mvit_u8_input.py measures on a CUDA device; none is visible')
    print(json.dumps(dict(card=card())), flush=True)
    for B in (16, 8):
        operand(B, args.iters, args.rounds)
    pretrain_step(args.steps, args.rounds)
    mixup_step(args.steps, args.rounds)


if __name__ == '__main__':
    main()
