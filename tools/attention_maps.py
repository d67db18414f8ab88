#!/usr/bin/env python
"""Attention maps of the cls query, as visualize_attention.py draws them, and what they cost.

    python tools/attention_maps.py [--out DIR] [--reps 10] [--rounds 3] [--skip-images] [--skip-table]

1. Images: a TimeSformer-B (8 x 224^2, divided space-time, random weights) on a synthetic clip; per frame the
   attn_img{i}.png of visualize_attention.py: the frame, the frame with the threshold masks of heads 0-5 drawn in colour
   (show_attn_color), and the per-head heatmaps side by side.  Heatmaps and masks come from model.attention_maps and are
   upsampled to pixels with repeat_interleave (show_attn's nearest interpolation); PIL writes the files, with a
   viridis-like colour ramp in place of matplotlib's.
2. Table: peak allocation above the resident model and inputs (torch.cuda.max_memory_allocated after
   reset_peak_memory_stats, after a warm-up call) and time per call (CUDA events: median over --rounds of the mean of
   --reps calls, the three arms alternated) of cls_attention against get_last_selfattention, forward-only (no_grad) and
   with autograd recording, for TimeSformer-B
   divided and joint space-time at 8 x 224^2 and 16 x 448^2, batch 1.  A call that fails is reported with its error.
The card's name and power limit are read with a read-only nvidia-smi query and printed with the numbers.  Needs a CUDA
device.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))

from eval_step import card  # noqa: E402


def model(kind, frames, side):
    from videotransformer_pytorch_b200 import TimeSformer
    torch.manual_seed(0)
    m = TimeSformer(num_frames=frames, img_size=side, patch_size=16, attention_type=kind)
    return m.cuda().eval()


def clip(frames, side):
    """a smooth synthetic clip [1, T, 3, S, S]: moving blobs, normalised like the reference's inputs"""
    t = torch.arange(frames, dtype=torch.float32)[:, None, None]
    yy, xx = torch.meshgrid(torch.linspace(0, 1, side), torch.linspace(0, 1, side), indexing='ij')
    chans = []
    for c, (cy, cx) in enumerate(((0.3, 0.3), (0.6, 0.7), (0.5, 0.4))):
        cyt, cxt = cy + 0.02 * t, cx - 0.015 * t
        chans.append(torch.exp(-((yy - cyt) ** 2 + (xx - cxt) ** 2) / 0.02))
    x = torch.stack(chans, dim=1)                   # [T, 3, S, S]
    return ((x - 0.45) / 0.225)[None].cuda()


def ramp(v):
    """[H, W] in [0, 1] -> uint8 [H, W, 3], a viridis-like ramp (dark blue -> green -> yellow)"""
    stops = np.array([[68, 1, 84], [59, 82, 139], [33, 145, 140], [94, 201, 98], [253, 231, 37]], dtype=np.float64)
    pos = np.clip(v, 0, 1) * (len(stops) - 1)
    i = np.minimum(pos.astype(int), len(stops) - 2)
    f = (pos - i)[..., None]
    return (stops[i] * (1 - f) + stops[i + 1] * f).astype(np.uint8)


def images(out):
    from PIL import Image
    m = model('divided_space_time', 8, 224)
    x = clip(8, 224)
    p = 16
    heat, mask = m.attention_maps(x, threshold=0.6)              # [8, 12, 14, 14] each
    heat = heat.repeat_interleave(p, -2).repeat_interleave(p, -1).cpu().numpy()
    mask = mask.repeat_interleave(p, -2).repeat_interleave(p, -1).cpu().numpy()
    frames = x[0].permute(0, 2, 3, 1).cpu().numpy()
    nh = heat.shape[1]
    rng = np.random.default_rng(0)
    colours = rng.uniform(0.3, 1.0, (nh, 3))
    for i in range(heat.shape[0]):
        f = frames[i]
        f = ((f - f.min()) / (f.max() - f.min() + 1e-12) * 255).astype(np.uint8)
        # show_attn_color: a faded grey frame with heads 0-5's masks blended in their colours
        grey = (f.astype(np.float64) - f.min()) / (f.max() - f.min() + 1e-12) * 64 + 192
        grey = np.repeat(grey.mean(axis=2)[:, :, None], 3, axis=2)
        for h in range(min(6, nh)):
            a = mask[i, h][:, :, None] * 0.5
            grey = grey * (1 - a) + a * 255 * colours[h]
        heads = np.concatenate([ramp(heat[i, h] / (heat[i, h].max() + 1e-12)) for h in range(nh)], axis=1)
        canvas = np.concatenate([f, grey.astype(np.uint8), heads], axis=1)
        Image.fromarray(canvas).save(os.path.join(out, f'attn_img{i}.png'))
    return heat.shape[0]


def peak(fn):
    """peak bytes above the allocation before one call (after a warm-up call: shadows, index maps, kernel attributes),
    or the call's error"""
    try:
        fn()
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        fn()
        torch.cuda.synchronize()
        return {'peak_MB': (torch.cuda.max_memory_allocated() - base) / 2 ** 20}
    except (RuntimeError, torch.cuda.OutOfMemoryError) as e:
        torch.cuda.synchronize()
        return {'error': str(e).splitlines()[0][:160]}


def time_arms(arms, reps, rounds):
    """ms per call of each arm that ran: the median over `rounds` of the mean of `reps` calls, arms alternated"""
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ms = {name: [] for name in arms}
    for _ in range(rounds):
        for name, fn in arms.items():
            t0.record()
            for _ in range(reps):
                fn()
            t1.record()
            torch.cuda.synchronize()
            ms[name].append(t0.elapsed_time(t1) / reps)
    return {name: sorted(v)[len(v) // 2] for name, v in ms.items()}


def table(reps, rounds):
    rows = []
    for frames, side in ((8, 224), (16, 448)):
        for kind in ('divided_space_time', 'joint_space_time'):
            m = model(kind, frames, side)
            x = torch.randn(1, frames, 3, side, side, device='cuda')

            def full_no_grad():
                with torch.no_grad():
                    return m.get_last_selfattention(x)

            arms = {'cls_attention': lambda: m.cls_attention(x),
                    'get_last_selfattention (no_grad)': full_no_grad,
                    'get_last_selfattention (autograd)': lambda: m.get_last_selfattention(x)}
            row = {'config': f'{kind} {frames}x{side}^2', 'N': int(m.cls_attention(x).shape[-1])}
            row.update({name: peak(fn) for name, fn in arms.items()})
            ran = {name: fn for name, fn in arms.items() if 'error' not in row[name]}
            for name, t in time_arms(ran, reps, rounds).items():
                row[name]['ms'] = t
            rows.append(row)
            del m, arms, ran
            torch.cuda.empty_cache()
    return rows


def cell(r):
    return r['error'] if 'error' in r else f"{r['peak_MB']:.0f} MB, {r['ms']:.1f} ms"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default='attention_maps_out', help='directory for the images and attention_maps.json')
    ap.add_argument('--reps', type=int, default=10)
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--skip-images', action='store_true')
    ap.add_argument('--skip-table', action='store_true')
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'tools/attention_maps.py needs a CUDA device'
    os.makedirs(args.out, exist_ok=True)
    print('card:', card())
    if not args.skip_images:
        print(f'wrote {images(args.out)} attn_img*.png to {args.out}')
    if not args.skip_table:
        rows = table(args.reps, args.rounds)
        cols = ['cls_attention', 'get_last_selfattention (no_grad)', 'get_last_selfattention (autograd)']
        print('| TimeSformer-B, batch 1 | N | ' + ' | '.join(f'`{c}`' for c in cols) + ' |')
        print('|---|---|' + '---|' * len(cols))
        for r in rows:
            print(f"| {r['config']} | {r['N']} | " + ' | '.join(cell(r[c]) for c in cols) + ' |')
        with open(os.path.join(args.out, 'attention_maps.json'), 'w') as fh:
            json.dump({'card': card(), 'rows': rows}, fh, indent=1)


if __name__ == '__main__':
    main()
