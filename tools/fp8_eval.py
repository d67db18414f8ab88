#!/usr/bin/env python
"""FP8 against bf16 inference on the forward-only path of TimeSformer-B, ViViT-B and MViT-B (+ a 400-class head).

    python tools/fp8_eval.py [--reps 20] [--rounds 3] [--workloads timesformer,vivit,mvit] [--skip-steps] [--json OUT]

1. Per GEMM: every distinct block-linear GEMM of the fp8 forward at validation batch 8 (shapes and epilogues recorded from
   one fp8 forward), timed stand-alone as the bf16 GEMM (bf16 operands), the e4m3 GEMM (operands already quantised) and
   the activation quantiser (vt_quant_rows_e4m3 of the bf16 A operand), arms alternated.
2. The eval step of tools/eval_step.py (model forward + top-k update) as GraphedForward replays with the model at 'bf16'
   and at 'fp8', the two graphs alternated, at batch 1, validation batch 8 and the 8 x 3-view test step.
Each cell is the median over --rounds of the mean of --reps calls (CUDA events), with the spread (max - min) beside it.
The card's name and power limit are read with a read-only nvidia-smi query and printed with the numbers.  Needs a CUDA
device; there is no CPU path.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))

from eval_step import NUM_CLASSES, SIZES, Net, card, time_calls  # noqa: E402


def gemm_shapes(workload):
    """(M, N, K, epi) of every e4m3 GEMM of one fp8 forward at batch 8, in first-seen order, with their counts."""
    from videotransformer_pytorch_b200 import _lib
    net = Net(workload).cuda().eval()
    net.model.set_inference_precision('fp8')
    x = torch.randn(8, net.frames, 3, 224, 224, device='cuda')
    seen = {}
    k = _lib.K
    orig = k.gemm_e4m3

    def rec(a, b, M, N, Kd, *, epi='bf16', **kw):
        key = (M, N, Kd, epi)
        seen[key] = seen.get(key, 0) + 1
        return orig(a, b, M, N, Kd, epi=epi, **kw)
    k.gemm_e4m3 = rec
    try:
        with torch.no_grad():
            net(x)
    finally:
        del k.gemm_e4m3
    del net
    torch.cuda.empty_cache()
    return seen


def time_gemm(M, N, Kd, epi, reps, rounds):
    from videotransformer_pytorch_b200 import _lib
    k = _lib.K
    a = torch.randn(M, Kd, device='cuda').to(torch.bfloat16)
    w = (torch.randn(N, Kd, device='cuda') * 0.02)
    wh = w.to(torch.bfloat16)
    bias = torch.randn(N, device='cuda')
    kw = dict(bias=bias)
    if epi == 'f32':
        kw['aux'] = torch.randn(M, N, device='cuda')
    a8, w8 = k.quant_rows_e4m3(a), k.quant_rows_e4m3(w)
    out16 = k.gemm(a, wh, M, N, Kd, epi=epi, **kw)
    out8 = k.gemm_e4m3(a8, w8, M, N, Kd, epi=epi, **kw)
    fns = {'bf16': lambda: k.gemm(a, wh, M, N, Kd, epi=epi, out=out16, **kw),
           'fp8': lambda: k.gemm_e4m3(a8, w8, M, N, Kd, epi=epi, out=out8, **kw),
           'quant': lambda: k.quant_rows_e4m3(a)}
    res = {arm: [] for arm in fns}
    for _ in range(rounds):
        for arm, fn in fns.items():
            fn()
            torch.cuda.synchronize()
            res[arm].append(time_calls(fn, reps) * 1e3)
    out = {arm: dict(us=round(statistics.median(v), 1), spread_us=round(max(v) - min(v), 1)) for arm, v in res.items()}
    flops = 2.0 * M * N * Kd
    out['bf16']['tflops'] = round(flops / out['bf16']['us'] * 1e-6, 1)
    out['fp8']['tflops'] = round(flops / out['fp8']['us'] * 1e-6, 1)
    out['fp8_plus_quant_vs_bf16'] = round((out['fp8']['us'] + out['quant']['us']) / out['bf16']['us'], 3)
    return out


def time_steps(workload, clips, views, reps, rounds):
    from videotransformer_pytorch_b200.graph import GraphedForward
    from videotransformer_pytorch_b200.metrics import TopKAccuracy
    torch.manual_seed(0)
    net = Net(workload).cuda().eval()
    x = torch.randn(clips * views, net.frames, 3, 224, 224, device='cuda')
    y = torch.randint(0, NUM_CLASSES, (clips,), device='cuda')
    acc = TopKAccuracy(top_k=(1, 5), views=views, device='cuda')

    def step(xx, yy):
        logits = net(xx)
        acc.update(logits, yy)
        return logits
    graphs, logits = {}, {}
    for prec in ('bf16', 'fp8'):
        net.model.set_inference_precision(prec)
        graphs[prec] = GraphedForward(step, (x, y))
        logits[prec] = graphs[prec](x, y).clone()
    res = {p: [] for p in graphs}
    for _ in range(rounds):
        for prec, g in graphs.items():
            g(x, y)
            torch.cuda.synchronize()
            res[prec].append(time_calls(lambda: g(x, y), reps))
    out = dict(workload=workload, clips=clips, views=views)
    for prec in graphs:
        ms = statistics.median(res[prec])
        out[prec] = dict(ms=round(ms, 3), spread_ms=round(max(res[prec]) - min(res[prec]), 3),
                         clips_per_s=round(clips / ms * 1e3, 1), launches=graphs[prec].kernels_per_replay)
    out['speedup'] = round(out['bf16']['ms'] / out['fp8']['ms'], 3)
    l16, l8 = logits['bf16'].double(), logits['fp8'].double()
    out['logits_rel_l2'] = round(float((l8 - l16).norm() / l16.norm()), 4)
    out['top1_agreement'] = round(float((l8.argmax(1) == l16.argmax(1)).double().mean()), 3)
    del graphs
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument('--reps', type=int, default=20)
    ap.add_argument('--step-reps', type=int, default=5)
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--workloads', default='timesformer,vivit,mvit')
    ap.add_argument('--skip-steps', action='store_true')
    ap.add_argument('--json', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit('fp8_eval: no CUDA device; these are GPU timings and there is no CPU fallback')
    info = card()
    print(json.dumps({'card': info}), flush=True)
    report = {'card': info, 'gemms': [], 'steps': []}
    for wl in args.workloads.split(','):
        for (M, N, Kd, epi), count in gemm_shapes(wl).items():
            r = dict(workload=wl, M=M, N=N, K=Kd, epi=epi, per_forward=count, **time_gemm(M, N, Kd, epi, args.reps, args.rounds))
            report['gemms'].append(r)
            print(json.dumps(r), flush=True)
    if not args.skip_steps:
        for wl in args.workloads.split(','):
            for name, clips, views in SIZES:
                try:
                    r = time_steps(wl, clips, views, args.step_reps, args.rounds)
                except torch.cuda.OutOfMemoryError as exc:
                    r = dict(workload=wl, clips=clips, views=views, error=f'out of memory: {str(exc)[:120]}')
                r['size'] = name
                report['steps'].append(r)
                print(json.dumps(r), flush=True)
                torch.cuda.empty_cache()
    print(f'\ncard: {info}')
    print(f'{"workload":12s} {"M x N x K":20s} {"epi":7s} {"bf16 us":>9s} {"fp8 us":>9s} {"quant us":>9s} {"(fp8+q)/bf16":>13s}')
    for r in report['gemms']:
        print(f'{r["workload"]:12s} {f"{r["M"]}x{r["N"]}x{r["K"]}":20s} {r["epi"]:7s} {r["bf16"]["us"]:9.1f} {r["fp8"]["us"]:9.1f} '
              f'{r["quant"]["us"]:9.1f} {r["fp8_plus_quant_vs_bf16"]:13.3f}')
    for r in report['steps']:
        if 'error' in r:
            print(f'{r["workload"]:12s} {r["size"]:24s} {r["error"]}')
            continue
        print(f'{r["workload"]:12s} {r["size"]:24s} bf16 {r["bf16"]["ms"]:8.2f} ms  fp8 {r["fp8"]["ms"]:8.2f} ms  '
              f'x{r["speedup"]:.3f}  top-1 agree {r["top1_agreement"]}')
    print(json.dumps({'card_after': card()}))
    if args.json:
        with open(args.json, 'w') as fh:
            json.dump(report, fh, indent=1)


if __name__ == '__main__':
    main()
