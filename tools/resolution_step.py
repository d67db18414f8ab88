#!/usr/bin/env python
"""TimeSformer-B (img_size 224) trained on larger clips: graphed train-step time and peak memory per input size, the
pos_embed resize kernels in situ, and the spatial attention kernels at 16 x 448^2 (N = 785).

    python tools/resolution_step.py [--steps 20] [--warmup 5] [--out DIR]

Prints one JSON line per configuration, with the card's name and power limit read in the same run.  A step is the
forward, cross-entropy loss and full backward of TimeSformer-B + a 400-class head, replayed as one CUDA graph; kernel
times come from one eager step under torch.profiler (CUDA activities), written under --out when given.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

CONFIGS = [('8x224', 8, 224, 8), ('8x320', 8, 320, 4), ('16x448', 16, 448, 1)]     # (name, frames, side, batch)


def card():
    q = subprocess.run(['nvidia-smi', '-i', str(torch.cuda.current_device()),
                        '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True)
    return q.stdout.strip() if q.returncode == 0 else torch.cuda.get_device_name()


class Net(torch.nn.Module):
    def __init__(self, frames):
        super().__init__()
        from videotransformer_pytorch_b200 import ClassificationHead, TimeSformer
        self.model = TimeSformer(num_frames=frames, img_size=224, patch_size=16, embed_dims=768, num_heads=12,
                                 num_transformer_layers=12)
        self.head = ClassificationHead(400, 768)

    def forward(self, x, y):
        return torch.nn.functional.cross_entropy(self.head(self.model(x)), y)


def kernel_times(net, x, y, trace_path=None):
    """us per kernel-name group over one eager step"""
    from torch.profiler import ProfilerActivity, profile
    net(x, y).backward()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        net(x, y).backward()
        torch.cuda.synchronize()
    if trace_path:
        prof.export_chrome_trace(trace_path)
    groups = {'pos_resize_fwd': 0.0, 'pos_resize_bwd': 0.0, 'spatial_attn_mma': 0.0, 'temporal_attn': 0.0, 'all': 0.0}
    for ev in prof.key_averages():
        t = ev.device_time_total if hasattr(ev, 'device_time_total') else ev.cuda_time_total
        name = ev.key
        groups['all'] += t
        if 'pos_resize_fwd' in name:
            groups['pos_resize_fwd'] += t
        elif 'pos_resize_bwd' in name:
            groups['pos_resize_bwd'] += t
        elif 'attn_mma' in name:
            groups['spatial_attn_mma'] += t      # spatial pass: tensor-core flash kernels
        elif 'attn' in name and 'probs' not in name:
            groups['temporal_attn'] += t         # temporal pass: warp-per-problem / generic kernels
    return {k: round(v, 1) for k, v in groups.items()}


def resize_times(model, side, reps=200):
    """us per call of vt_pos_resize_fwd / _bwd from Python, launch overhead included (an upper bound on the kernel time),
    on the model's pos_embed for a side x side input (CUDA events over
    `reps` back-to-back launches); empty at the training grid, where nothing is resized."""
    from videotransformer_pytorch_b200 import _lib
    g = round((model.pos_embed.shape[1] - 1) ** 0.5)
    n = side // 16
    if n == g:
        return {}
    src = model.pos_embed.detach()[0, 1:]
    grid, out_grid, sc = (g, g), (n, n), ((n + 0.1) / g, (n + 0.1) / g)
    out = _lib.K.pos_resize_fwd(src, grid, out_grid, sc)
    dsrc = torch.empty_like(src)
    res = {}
    for label, fn in (('fwd', lambda: _lib.K.pos_resize_fwd(src, grid, out_grid, sc, out=out)),
                      ('bwd', lambda: _lib.K.pos_resize_bwd(out, grid, out_grid, sc, out=dsrc))):
        fn()
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0.record()
        for _ in range(reps):
            fn()
        t1.record()
        torch.cuda.synchronize()
        res[label] = round(t0.elapsed_time(t1) * 1000 / reps, 2)
    return res


def run(name, frames, side, batch, steps, warmup, out):
    from videotransformer_pytorch_b200.graph import GraphedTrainStep
    torch.manual_seed(0)
    dev = torch.device('cuda')
    net = Net(frames).to(dev).train()
    x = torch.randn(batch, frames, 3, side, side, device=dev)
    y = torch.randint(0, 400, (batch,), device=dev)
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats(dev)
    step = GraphedTrainStep(net, (x, y))
    for _ in range(warmup):
        step(x, y)
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    times = []
    for _ in range(3):                       # three windows of `steps` replays
        t0.record()
        for _ in range(steps):
            step(x, y)
        t1.record()
        torch.cuda.synchronize()
        times.append(t0.elapsed_time(t1) / steps)
    peak = torch.cuda.max_memory_allocated(dev) / 2 ** 30
    del step
    trace = os.path.join(out, f'trace_{name}.json') if out else None
    kt = kernel_times(net, x, y, trace)
    P = (side // 16) ** 2
    res = dict(config=name, frames=frames, side=side, batch=batch, spatial_tokens=P + 1,
               ms_per_step=round(sorted(times)[1], 3), ms_range=[round(min(times), 3), round(max(times), 3)],
               clips_per_s=round(batch * 1000 / sorted(times)[1], 2), peak_mem_gib=round(peak, 2),
               eager_kernel_us=kt, resize_call_us=resize_times(net.model, side))
    del net
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=5)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('resolution_step.py measures on a CUDA device; none found')
    if args.out:
        os.makedirs(args.out, exist_ok=True)
    info = dict(card=card(), torch=torch.__version__)
    print(json.dumps(info), flush=True)
    for name, frames, side, batch in CONFIGS:
        print(json.dumps(run(name, frames, side, batch, args.steps, args.warmup, args.out)), flush=True)


if __name__ == '__main__':
    main()
