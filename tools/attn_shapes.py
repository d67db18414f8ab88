"""Time every distinct attention-core call of the benched workloads stand-alone on the GPU.

    python tools/attn_shapes.py [--reps 30] [--warmup 5] [--rounds 3] [--workloads timesformer,vivit,mvit,maskfeat]
                                [--baseline-lib PATH] [--tiled] [--profile] [--json OUT]

The shapes are recorded, not listed: one eager fwd + bwd step of each workload (bench.py's models and batches) runs with
K.attn_fwd / attn_bwd / xattn_fwd / xattn_bwd wrapped, and the first call of each distinct shape keeps its real operands
(layout and strides included).  Each shape's forward and backward is then timed with CUDA events over `--reps` launches.
Per row: microseconds, the bytes the call must move at least once and its algorithmic FLOPs (attention backward counted
2.5x forward: S, dP, dV, dK, dQ), and the time over the larger of the two data-sheet floors (989 TFLOP/s dense BF16,
3.35 TB/s HBM3, H100 SXM at 700 W).

--baseline-lib PATH loads a second libvt_b200.so (another build of the same C ABI) and alternates the two libraries row by
row, `--rounds` times each, in this one process: the columns give the median of each and its spread (max - min).

--tiled adds this library once more with VT_ATTN_WHOLE=0 (the 64-row tiled tensor-core kernels instead of the
whole-problem ones on the packed-qkv path), alternated with the others in the same way.

--profile instead runs every forward and backward shape a few times under torch.profiler and prints the time of each
kernel it launches (the whole-problem kernels, or with --tiled also the tiled forward, dQ and dK/dV kernels); run it on its
own, the profiler slows the host.

The card's name, power limit and SM clocks are read with read-only nvidia-smi queries and printed with the numbers.
Needs a CUDA device; there is no CPU path.
"""
import argparse
import ctypes
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from gemm_shapes import PEAK_TBS, PEAK_TFLOPS, card, events_ms  # noqa: E402

WRAPPED = ('attn_fwd', 'attn_bwd', 'xattn_fwd', 'xattn_bwd')


def packed_kernel(N):
    """which vt_attn_* kernel the automatic choice takes (vt_attention.cu pick_impl, use_whole)"""
    return 'warp8' if N == 8 else 'generic' if N <= 32 else 'whole' if N <= 256 else 'tiled'


def set_whole(env):
    """VT_ATTN_WHOLE for the following calls (read by the library at every call); None: the library's default"""
    if env is None:
        os.environ.pop('VT_ATTN_WHOLE', None)
    else:
        os.environ['VT_ATTN_WHOLE'] = env


def record(workloads, dev):
    """{key: row} of the distinct attention calls of one eager step per workload; a row keeps the forward and backward
    operands of its shape's first call"""
    import bench
    from videotransformer_pytorch_b200 import _lib
    K = _lib.K
    rows = {}
    orig = {n: getattr(K, n) for n in WRAPPED}
    cur = {}

    def key_of(name, a):
        if name == 'attn_fwd':          # (qkv, Bp, N, H, hd, ...)
            return ('attn',) + tuple(a[1:5])
        if name == 'attn_bwd':          # (qkv, ctx, dctx, lse, Bp, N, H, hd, ...)
            return ('attn',) + tuple(a[4:8])
        q, k = a[0], a[1]
        return ('xattn',) + tuple(q.shape) + (k.shape[2],) + tuple(q.stride()) + tuple(k.stride())

    def wrap(name):
        def f(*a, **kw):
            key = key_of(name, a)
            row = rows.setdefault(key, {'key': key, 'workloads': []})
            if cur['w'] not in row['workloads']:
                row['workloads'].append(cur['w'])
            side = 'fwd' if name.endswith('fwd') else 'bwd'
            if side not in row:
                row[side] = (name, a, dict(kw))
            return orig[name](*a, **kw)
        return f

    for n in WRAPPED:
        setattr(K, n, wrap(n))
    try:
        for w in workloads:
            cur['w'] = w
            run = bench.WorkloadRun(w, dev, bench.WORKLOADS[w]['batch'], 0)
            inputs = run.prepare([t.to(dev) for t in run.host], run.meta)
            run.net(*inputs).backward()
            torch.cuda.synchronize()
            del run, inputs
    finally:
        for n in WRAPPED:
            setattr(K, n, orig[n])
    return [r for r in rows.values() if 'fwd' in r and 'bwd' in r]


def describe(row):
    """label, kernel, (fwd bytes, fwd flop), (bwd bytes, bwd flop)"""
    key = row['key']
    if key[0] == 'attn':
        _, Bp, N, H, hd = key
        e = Bp * N * H * hd * 2                  # one bf16 [Bp, N, H, hd] operand
        lse = Bp * H * N * 4
        f = 4.0 * Bp * H * N * N * hd
        return (f'{Bp}x{N}x{H} hd{hd}', packed_kernel(N), (4 * e + lse, f), (8 * e + lse, 2.5 * f))
    _, B, H, Nq, hd, Nk = key[:6]
    # q, o, dout, dq: bf16 [B, H, Nq, hd]; k, v: bf16 [B, H, Nk, hd]; dk, dv fp32; lse, delta fp32
    eq, ek, stat = B * H * Nq * hd * 2, B * H * Nk * hd * 2, B * H * Nq * 4
    f = 4.0 * B * H * Nq * Nk * hd
    return (f'{B}x{H} q{Nq} k{Nk} hd{hd}', 'xattn', (2 * eq + 2 * ek + stat, f),
            (4 * eq + 2 * ek + 4 * ek + 2 * stat, 2.5 * f))


def call(row, side):
    from videotransformer_pytorch_b200 import _lib
    name, a, kw = row[side]
    return getattr(_lib.K, name)(*a, **kw)


def open_lib(path):
    from videotransformer_pytorch_b200 import _lib
    lib = ctypes.CDLL(os.path.abspath(path))
    for n in _lib.EXPORTS:
        getattr(lib, n).restype = ctypes.c_int
    if lib.vt_version() != 1:
        sys.exit(f'attn_shapes: {path}: ABI version mismatch')
    return lib


def timings(rows, args, libs):
    """{(row index, side, lib name): [us per round]}, libraries (and VT_ATTN_WHOLE settings) alternated inside each round"""
    from videotransformer_pytorch_b200 import _lib
    res = {}
    own = _lib._dll
    try:
        for i, row in enumerate(rows):
            for _ in range(args.rounds):
                for lname, lib, env in libs:
                    _lib._dll = lib
                    set_whole(env)
                    for side in ('fwd', 'bwd'):
                        us = 1e3 * events_ms(lambda: call(row, side), args.reps, args.warmup)
                        res.setdefault((i, side, lname), []).append(us)
    finally:
        _lib._dll = own
        set_whole(None)
    return res


def report(rows, res, libs, out):
    names = [n for n, _, _ in libs]
    hdr = f'{"shape":28s} {"kernel":7s} {"pass":4s} {"MB":>7s} {"GFLOP":>7s} {"floor us":>8s}'
    for n in names:
        hdr += f' {"us " + n:>10s} {"+-":>6s} {"x floor":>7s}'
    for n in names[1:]:
        hdr += f' {n + "/" + names[0]:>10s}'
    print(hdr)
    for i, row in enumerate(rows):
        label, kern, fwd, bwd = describe(row)
        for side, (byts, flop) in (('fwd', fwd), ('bwd', bwd)):
            floor = max(flop / (PEAK_TFLOPS * 1e12), byts / (PEAK_TBS * 1e12)) * 1e6
            r = dict(shape=label, kernel=kern, workloads=row['workloads'], side=side, bytes=byts, flop=flop, floor_us=floor,
                     bound='hbm' if byts / PEAK_TBS > flop / PEAK_TFLOPS * 1e-3 else 'tensor')
            line = f'{label:28s} {kern:7s} {side:4s} {byts / 1e6:7.1f} {flop / 1e9:7.2f} {floor:8.1f}'
            for n in names:
                ts = res[(i, side, n)]
                med = statistics.median(ts)
                r[n] = dict(us=med, spread=max(ts) - min(ts), over_floor=med / floor, rounds=ts)
                line += f' {med:10.1f} {max(ts) - min(ts):6.1f} {med / floor:7.2f}'
            for n in names[1:]:
                r['ratio_' + n] = r[n]['us'] / r[names[0]]['us']
                line += f' {r["ratio_" + n]:10.3f}'
            out.append(r)
            print(line + f'   [{",".join(row["workloads"])}]')


def profile(rows, args, envs):
    """per-kernel split of every forward and backward shape, from torch.profiler (CUDA activity), for each
    VT_ATTN_WHOLE setting in `envs`"""
    from torch.profiler import ProfilerActivity
    from torch.profiler import profile as prof
    out = []
    try:
        for row in rows:
            label = describe(row)[0]
            for env in envs:
                set_whole(env)
                for side in ('fwd', 'bwd'):
                    for _ in range(args.warmup):
                        call(row, side)
                    torch.cuda.synchronize()
                    with prof(activities=[ProfilerActivity.CUDA]) as p:
                        for _ in range(args.reps):
                            call(row, side)
                        torch.cuda.synchronize()
                    per = {}
                    for ev in p.events():
                        if ev.device_type == torch.autograd.DeviceType.CUDA:
                            per[ev.name] = per.get(ev.name, 0.0) + ev.device_time / args.reps
                    for name, us in sorted(per.items(), key=lambda kv: -kv[1]):
                        out.append(dict(shape=label, side=side, whole=env, kernel=name, us=us))
                        print(f'{label:28s} {side} {us:9.1f} us  {name[:110]}')
    finally:
        set_whole(None)
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument('--reps', type=int, default=30)
    ap.add_argument('--warmup', type=int, default=5)
    ap.add_argument('--rounds', type=int, default=3, help='timings per row and library, alternating')
    ap.add_argument('--workloads', default='timesformer,vivit,mvit,maskfeat')
    ap.add_argument('--baseline-lib', default=None, help='a second libvt_b200.so, timed against this tree\'s')
    ap.add_argument('--tiled', action='store_true', help='also time / profile this library with VT_ATTN_WHOLE=0')
    ap.add_argument('--profile', action='store_true', help='only the torch.profiler split of the attention kernels')
    ap.add_argument('--json', default=None, help='also write the rows as JSON to this file')
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit('attn_shapes: no CUDA device; these are GPU timings and there is no CPU fallback')
    from videotransformer_pytorch_b200 import _lib
    dev = torch.device('cuda:0')
    info = card()
    print(json.dumps({'card': info}))
    lib = _lib.load_library()
    libs = [('this', lib, '1' if args.tiled else None)]
    if args.tiled:
        libs.append(('tiled', lib, '0'))
    if args.baseline_lib:
        libs.append(('base', open_lib(args.baseline_lib), None))
    rows = record([w for w in args.workloads.split(',') if w], dev)
    print(f'{len(rows)} distinct attention shapes')
    if args.profile:
        out = profile(rows, args, ['1', '0'] if args.tiled else [None])
    else:
        out = []
        report(rows, timings(rows, args, libs), libs, out)
    print(json.dumps({'card_after': card()}))
    if args.json:
        with open(args.json, 'w') as fh:
            json.dump({'card': info, 'rows': out}, fh, indent=1)


if __name__ == '__main__':
    main()
