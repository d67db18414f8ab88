"""Time the packed-qkv attention core (vt_attn_fwd / vt_attn_bwd) at head widths 32, 64, 96 and 128 on the GPU.

    python tools/attn_head_dims.py [--reps 30] [--warmup 5] [--rounds 3] [--json OUT]

The shapes are the passes of TimeSformer-B / ViViT-B at D = 768 (batch 8, 8 frames of 196 patches) with the head count
that gives each width (24, 12, 8 and 6 heads): the spatial pass (64 frames x 197 tokens, whole-problem kernels at width
64, tiled ones otherwise), the temporal pass (1568 x 8, warp-per-problem kernel), ViViT's factorised temporal pass
(8 x 9, generic kernels, with 196-fold more rows as in a 16-frame clip) and the joint pass (2 clips x 1569 tokens, tiled
kernels).  Each row gives the median microseconds over `--rounds` timings of `--reps` launches (CUDA events) and that time
as a multiple of the larger of the two data-sheet floors: the algorithmic FLOPs (4 N^2 hd per problem forward, 2.5x that
backward) at 989 TFLOP/s dense BF16, and the bytes the call must move once (qkv, ctx and lse forward; qkv, ctx, dctx, lse
and dqkv backward) at 3.35 TB/s HBM3 (H100 SXM at 700 W).  The card's name, power limit and SM clocks are read with
read-only nvidia-smi queries and printed with the numbers.  Needs a CUDA device; there is no CPU path.
"""
import argparse
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from gemm_shapes import PEAK_TBS, PEAK_TFLOPS, card, events_ms  # noqa: E402

D = 768
PASSES = [('spatial', 64, 197), ('temporal', 1568, 8), ('vivit temporal', 1568, 9), ('joint', 2, 1569)]


def floors(Bp, N, H, hd):
    """(forward, backward) least time in microseconds: max(FLOPs / peak, bytes / bandwidth), and which bounds it"""
    probs = Bp * H
    fl = 4.0 * N * N * hd * probs
    row = N * H * hd * 2.0
    by_f = Bp * (3 * row + row) + 4.0 * probs * N
    by_b = Bp * (3 * row + row + row + 3 * row) + 4.0 * probs * N
    out = []
    for f, b in ((fl, by_f), (2.5 * fl, by_b)):
        tf, tb = f / (PEAK_TFLOPS * 1e12) * 1e6, b / (PEAK_TBS * 1e12) * 1e6
        out.append((max(tf, tb), 'FLOP' if tf >= tb else 'byte'))
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument('--reps', type=int, default=30)
    ap.add_argument('--warmup', type=int, default=5)
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--json', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit('attn_head_dims: needs a CUDA device')
    from videotransformer_pytorch_b200 import _lib
    _lib.load_library()
    K = _lib.K
    dev = torch.device('cuda:0')
    print('card:', card())
    rows = []
    g = torch.Generator(device=dev).manual_seed(0)
    for name, Bp, N in PASSES:
        for hd in (32, 64, 96, 128):
            H = D // hd
            scale = hd ** -0.5
            qkv = torch.randn(Bp * N, 3 * D, device=dev, generator=g).mul_(0.5).to(torch.bfloat16)
            ctx, lse, _ = K.attn_fwd(qkv, Bp, N, H, hd, scale)
            dctx = torch.randn(Bp * N, D, device=dev, generator=g).to(torch.bfloat16)
            fwd = lambda: K.attn_fwd(qkv, Bp, N, H, hd, scale)
            bwd = lambda: K.attn_bwd(qkv, ctx, dctx, lse, Bp, N, H, hd, scale)
            tf, tb = [], []
            for _ in range(args.rounds):
                tf.append(events_ms(fwd, args.reps, args.warmup) * 1e3)
                tb.append(events_ms(bwd, args.reps, args.warmup) * 1e3)
            (ff, fk), (fb, bk) = floors(Bp, N, H, hd)
            r = dict(name=name, Bp=Bp, N=N, H=H, hd=hd, fwd_us=statistics.median(tf), bwd_us=statistics.median(tb),
                     fwd_spread=max(tf) - min(tf), bwd_spread=max(tb) - min(tb), fwd_floor_us=ff, bwd_floor_us=fb,
                     fwd_bound=fk, bwd_bound=bk)
            rows.append(r)
            print(f"{name:15s} {Bp:5d} x {N:4d} x {H:2d}, hd {hd:3d}: fwd {r['fwd_us']:8.1f} us [{r['fwd_spread']:.1f}] "
                  f"= {r['fwd_us'] / ff:5.2f}x {fk} floor; bwd {r['bwd_us']:8.1f} us [{r['bwd_spread']:.1f}] "
                  f"= {r['bwd_us'] / fb:5.2f}x {bk} floor", flush=True)
    if args.json:
        with open(args.json, 'w') as fh:
            json.dump(dict(card=card(), rows=rows), fh, indent=1)


if __name__ == '__main__':
    main()
