#!/usr/bin/env python
"""Evaluation step time of TimeSformer-B, ViViT-B and MViT-B (+ a 400-class head) on the three forward paths.

    python tools/eval_step.py [--reps 5] [--warmup 2] [--rounds 3] [--workloads timesformer,vivit,mvit] [--json OUT]

Sizes: batch 1 (one clip: BASELINE config 1 on the GPU), validation at batch 8, and the 3-view test step at 8 clips
(24 views, logits averaged per clip before the softmax).  Every call is the model forward plus the top-k counter update
(metrics.TopKAccuracy, top-1 / top-5) of model_trainer.py's validation / test step.  Arms:
  grad  : the forward as it ran before the forward-only path existed: grad mode on, model in eval mode (Function.apply,
          every backward-only output written and saved until the output is dropped)
  eager : the same forward under torch.no_grad(): forward-only kernel forms, launched one by one from Python
  graph : graph.GraphedForward of the no_grad forward, one replay per call
The arms alternate in this one process, `--rounds` times each; each cell is the median over the rounds of the mean of
`--reps` timed calls (CUDA events), with the spread (max - min) beside it.  Kernel launches per call are counted with
vt_launch_count.  The card's name and power limit are read with a read-only nvidia-smi query and printed with the numbers.
Needs a CUDA device; there is no CPU path.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

NUM_CLASSES = 400
SIZES = [('batch 1', 1, 1), ('val batch 8', 8, 1), ('test 8 clips x 3 views', 8, 3)]     # (name, clips, views)
ARMS = ('grad', 'eager', 'graph')


def card():
    q = subprocess.run(['nvidia-smi', '-i', str(torch.cuda.current_device()),
                        '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True)
    return q.stdout.strip() if q.returncode == 0 else torch.cuda.get_device_name()


class Net(torch.nn.Module):
    """backbone + ClassificationHead -> logits"""

    def __init__(self, workload):
        super().__init__()
        from videotransformer_pytorch_b200 import ClassificationHead, MaskFeat, TimeSformer, ViViT
        self.workload = workload
        if workload == 'timesformer':
            self.model = TimeSformer(num_frames=8, img_size=224, patch_size=16, embed_dims=768, num_heads=12,
                                     num_transformer_layers=12, attention_type='divided_space_time')
            dim, self.frames = 768, 8
        elif workload == 'vivit':
            self.model = ViViT(num_frames=16, img_size=224, patch_size=16, embed_dims=768, num_heads=12,
                               num_transformer_layers=12, attention_type='fact_encoder')
            dim, self.frames = 768, 16
        else:
            self.model = MaskFeat(pool_q_stride_size=[[1, 1, 2, 2], [3, 1, 2, 2]], feature_dim=2 * 2 * 2 * 3 * 9)
            dim, self.frames = self.model.mvit.norm_embed.normalized_shape[0], 16
        self.head = ClassificationHead(NUM_CLASSES, dim)
        if workload != 'mvit':
            with torch.no_grad():       # temporal_fc is zero-init: make the branch live
                for n, p in self.model.named_parameters():
                    if 'temporal_fc' in n:
                        p.normal_(std=0.02)

    def forward(self, x):
        f = self.model.forward_features(x)[:, 0] if self.workload == 'mvit' else self.model(x)
        return self.head(f)


def time_calls(fn, reps):
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(reps):
        fn()
    t1.record()
    torch.cuda.synchronize()
    return t0.elapsed_time(t1) / reps


def measure(workload, clips, views, args):
    from videotransformer_pytorch_b200 import _lib
    from videotransformer_pytorch_b200.graph import GraphedForward
    from videotransformer_pytorch_b200.metrics import TopKAccuracy
    torch.manual_seed(0)
    net = Net(workload).cuda().eval()
    x = torch.randn(clips * views, net.frames, 3, 224, 224, device='cuda')
    y = torch.randint(0, NUM_CLASSES, (clips,), device='cuda')
    acc = TopKAccuracy(top_k=(1, 5), views=views, device='cuda')

    def step(xx, yy):
        logits = net(xx)
        acc.update(logits.detach(), yy)
        return logits

    def no_grad_step(xx, yy):
        with torch.no_grad():
            return step(xx, yy)

    fns = {'grad': lambda: step(x, y), 'eager': lambda: no_grad_step(x, y)}
    launches = {}
    for arm, fn in fns.items():
        fn()
        torch.cuda.synchronize()
        l0 = _lib.launch_count()
        fn()
        torch.cuda.synchronize()
        launches[arm] = _lib.launch_count() - l0
    g = GraphedForward(no_grad_step, (x, y))
    fns['graph'] = lambda: g(x, y)
    launches['graph'] = g.kernels_per_replay
    res = {a: [] for a in ARMS}
    for _ in range(args.rounds):
        for arm in ARMS:
            for _ in range(args.warmup):
                fns[arm]()
            torch.cuda.synchronize()
            res[arm].append(time_calls(fns[arm], args.reps))
    out = dict(workload=workload, clips=clips, views=views)
    for arm in ARMS:
        ms = statistics.median(res[arm])
        out[arm] = dict(ms=round(ms, 3), spread_ms=round(max(res[arm]) - min(res[arm]), 3),
                        clips_per_s=round(clips / ms * 1e3, 1), launches=launches[arm])
    out['eager_speedup'] = round(out['grad']['ms'] / out['eager']['ms'], 3)
    out['graph_speedup'] = round(out['grad']['ms'] / out['graph']['ms'], 3)
    del g, fns
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument('--reps', type=int, default=5)
    ap.add_argument('--warmup', type=int, default=2)
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--workloads', default='timesformer,vivit,mvit')
    ap.add_argument('--json', default=None, help='also write the rows as JSON to this file')
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit('eval_step: no CUDA device; these are GPU timings and there is no CPU fallback')
    info = card()
    print(json.dumps({'card': info}))
    rows = []
    for workload in args.workloads.split(','):
        for name, clips, views in SIZES:
            try:
                r = measure(workload, clips, views, args)
            except torch.cuda.OutOfMemoryError as exc:
                r = dict(workload=workload, clips=clips, views=views, error=f'out of memory: {str(exc)[:120]}')
            r['size'] = name
            rows.append(r)
            print(json.dumps(r), flush=True)
            torch.cuda.empty_cache()
    print(f'\ncard: {info}')
    print(f'{"workload":12s} {"size":24s} ' + ' '.join(f'{a + " ms":>10s} {a + " clip/s":>13s}' for a in ARMS) +
          f' {"launches g/e/graph":>20s}')
    for r in rows:
        if 'error' in r:
            print(f'{r["workload"]:12s} {r["size"]:24s} {r["error"]}')
            continue
        cells = ' '.join(f'{r[a]["ms"]:10.2f} {r[a]["clips_per_s"]:13.1f}' for a in ARMS)
        ln = '/'.join(str(r[a]['launches']) for a in ARMS)
        print(f'{r["workload"]:12s} {r["size"]:24s} {cells} {ln:>20s}')
    print(json.dumps({'card_after': card()}))
    if args.json:
        with open(args.json, 'w') as fh:
            json.dump({'card': info, 'rows': rows}, fh, indent=1)


if __name__ == '__main__':
    main()
