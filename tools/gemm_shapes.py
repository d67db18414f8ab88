"""Time every distinct GEMM of the TimeSformer-B step (8 frames of 224^2, batch 8) stand-alone on the GPU.

    python tools/gemm_shapes.py [--reps 50] [--warmup 10] [--rounds 3] [--k-sweep] [--json OUT]

For each GEMM it runs vt_gemm with the layouts and epilogue the model uses, under the planner's choice and with each
tile width forced, and prints TFLOP/s, HBM GB/s (bytes the epilogue and operands must move at least once) and the time
over the larger of the two data-sheet floors (989 TFLOP/s dense BF16, 3.35 TB/s HBM3, H100 SXM at 700 W).  Every row is
timed with the register epilogue (VT_GEMM_STAGED_EPI=0) and the staged one (=1), alternating, `--rounds` times each in
this one process: the columns give the median of each, its spread (max - min over the rounds) and the ratio register /
staged.  The rate columns are the staged path's.  For the plain shapes it times torch.matmul (cuBLAS, bf16) as well: the
rate this card reaches at its power limit.

The evaluation forward's FC1 is timed both ways: 'gelu_h' (h alone from the epilogue) against the split form it replaces,
the 'bf16' GEMM that writes z plus the stand-alone GELU kernel (its own row, "gelu kernel").

--k-sweep times the wide-output GEMMs (qkv forward, the forward-only FC1 with gelu_h, FC2 data gradient) at their M x N
with K = 768, 1536, 3072 and 6144 and BN = 128, and fits the time per wave of tiles, t_tile = a * k-blocks + e: e is the
per-tile cost that does not scale with K (epilogue, pipeline fill), printed for both epilogues.

The card's name, power limit and SM clocks are read with read-only nvidia-smi queries and printed with the numbers.
Needs a CUDA device; there is no CPU path.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

PEAK_TFLOPS, PEAK_TBS = 989.0, 3.35
B, T, P, D, HID = 8, 8, 196, 768, 3072
S = 1 + P * T
M_TOK, M_TEMP, M_SPAT = B * S, B * P * T, B * T * (P + 1)     # 12552, 12544, 12608
SWITCH = 'VT_GEMM_STAGED_EPI'
SWEEP = ('qkv fwd temporal', 'fc1 fwd eval (gelu_h)', 'fc2 dgrad')
SWEEP_K = (768, 1536, 3072, 6144)


def card():
    q = 'name,power.limit,clocks.sm,clocks.max.sm'
    try:
        out = subprocess.run(['nvidia-smi', '-i', '0', f'--query-gpu={q}', '--format=csv,noheader'], capture_output=True,
                             text=True, timeout=30).stdout.strip()
    except Exception as exc:
        out = f'nvidia-smi unavailable ({exc})'
    return dict(zip(q.split(','), [v.strip() for v in out.split(',')])) if out.count(',') == 3 else {'nvidia-smi': out}


def events_ms(fn, reps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(reps):
        fn()
    t1.record()
    torch.cuda.synchronize()
    return t0.elapsed_time(t1) / reps


def ab_us(fn, args):
    """fn timed with the register (0) and the staged (1) epilogue, alternating: {mode: [us per round]}.  vt_gemm reads
    the switch on every call, so setting the environment between calls is enough."""
    prev = os.environ.get(SWITCH)
    res = {'0': [], '1': []}
    try:
        for _ in range(args.rounds):
            for mode in ('0', '1'):
                os.environ[SWITCH] = mode
                res[mode].append(1e3 * events_ms(fn, args.reps, args.warmup))
    finally:
        if prev is None:
            os.environ.pop(SWITCH, None)
        else:
            os.environ[SWITCH] = prev
    return res


def cases(dev):
    """(name, M, N, K, layouts, kwargs for K.gemm, epilogue bytes per output element, plain)"""
    from videotransformer_pytorch_b200 import ops
    maps = ops.token_maps(B, T, P, dev)
    aff = ops.affine_row_maps(B, T, P, D)
    bias_d, bias_3d, bias_h = (torch.randn(n, device=dev) for n in (D, 3 * D, HID))
    stream = torch.randn(B * S + B * T, D, device=dev)
    out = [
        ('qkv fwd temporal', M_TEMP, 3 * D, D, (0, 0), dict(epi='bf16', bias=bias_3d), 2, True),
        ('qkv fwd spatial', M_SPAT, 3 * D, D, (0, 0), dict(epi='bf16', bias=bias_3d), 2, True),
        ('proj fwd temporal (affine)', M_TEMP, D, D, (0, 0),
         dict(epi='f32', bias=bias_d, bias2=bias_d, aux=stream, out=stream, aux_row=maps['temporal'], out_row=maps['temporal'],
              row_map=aff['temporal']), 8, False),
        ('proj fwd spatial (affine, cls rows)', M_SPAT, D, D, (0, 0),
         dict(epi='f32', bias=bias_d, aux=stream, out=stream, aux_row=maps['sp_aux'], out_row=maps['sp_out'],
              row_map=aff['spatial']), 8, False),
        ('fc1 fwd eval (gelu_h)', M_TOK, HID, D, (0, 0), dict(epi='gelu_h', bias=bias_h), 2, False),
        ('fc1 fwd split (bf16; + gelu kernel)', M_TOK, HID, D, (0, 0), dict(epi='bf16', bias=bias_h), 2, False),
        ('fc2 fwd (f32 residual)', M_TOK, D, HID, (0, 0), dict(epi='f32', bias=bias_d, aux=stream[:M_TOK]), 8, False),
        ('fc2 dgrad', M_TOK, HID, D, (0, 1), dict(epi='bf16'), 2, False),
        ('fc1 dgrad', M_TOK, D, HID, (0, 1), dict(epi='bf16'), 2, True),
        ('proj dgrad', M_TEMP, D, D, (0, 1), dict(epi='bf16'), 2, True),
        ('qkv dgrad', M_TEMP, D, 3 * D, (0, 1), dict(epi='bf16'), 2, True),
        ('qkv wgrad', 3 * D, D, M_TEMP, (1, 1), dict(epi='f32', split_ok=True), 4, True),
        ('proj wgrad', D, D, M_TEMP, (1, 1), dict(epi='f32', split_ok=True), 4, True),
        ('fc1 wgrad', HID, D, M_TOK, (1, 1), dict(epi='f32', split_ok=True), 4, True),
        ('fc2 wgrad', D, HID, M_TOK, (1, 1), dict(epi='f32', split_ok=True), 4, True),
    ]
    return out


def operands(M, N, Kd, a_mn, b_mn, dev):
    a = (torch.randn(Kd, M, device=dev) if a_mn else torch.randn(M, Kd, device=dev)).mul_(0.1).bfloat16()
    b = (torch.randn(Kd, N, device=dev) if b_mn else torch.randn(N, Kd, device=dev)).mul_(0.1).bfloat16()
    return a, b


def fmt_ab(res):
    """median and spread of each epilogue, and the ratio register / staged"""
    reg, stg = statistics.median(res['0']), statistics.median(res['1'])
    return dict(us_reg=reg, us_staged=stg, spread_reg=max(res['0']) - min(res['0']),
                spread_staged=max(res['1']) - min(res['1']), ratio=reg / stg)


def shapes(K, dev, args, rows):
    hdr = (f'{"gemm":38s} {"M":>6s} {"N":>5s} {"K":>6s} {"tile":>6s} {"us reg":>8s} {"+-":>5s} {"us stg":>8s} {"+-":>5s} '
           f'{"reg/stg":>7s} {"TFLOP/s":>8s} {"GB/s":>7s} {"x floor":>7s}')
    print(hdr)
    for name, M, N, Kd, (a_mn, b_mn), kw, epi_b, plain in cases(dev):
        a, b = operands(M, N, Kd, a_mn, b_mn, dev)
        flop = 2.0 * M * N * Kd
        byts = 2.0 * (M * Kd + N * Kd) + epi_b * M * N
        floor_us = max(flop / (PEAK_TFLOPS * 1e12), byts / (PEAK_TBS * 1e12)) * 1e6
        for bn in (0, 128, 192, 256):
            res = ab_us(lambda: K.gemm(a, b, M, N, Kd, a_mn=bool(a_mn), b_mn=bool(b_mn), force_bn=bn, **kw), args)
            r = dict(gemm=name, M=M, N=N, K=Kd, tile=bn or 'auto', **fmt_ab(res))
            us = r['us_staged']
            r.update(tflops=flop / us * 1e-6, gbs=byts / us * 1e-3, over_floor=us / floor_us)
            rows.append(r)
            print(f'{name:38s} {M:6d} {N:5d} {Kd:6d} {str(r["tile"]):>6s} {r["us_reg"]:8.1f} {r["spread_reg"]:5.1f} '
                  f'{us:8.1f} {r["spread_staged"]:5.1f} {r["ratio"]:7.3f} {r["tflops"]:8.1f} {r["gbs"]:7.0f} '
                  f'{r["over_floor"]:7.2f}')
        if plain:
            A = a.t() if a_mn else a
            Bm = b if b_mn else b.t()
            us = 1e3 * events_ms(lambda: torch.matmul(A, Bm), args.reps, args.warmup)
            r = dict(gemm=name, M=M, N=N, K=Kd, tile='cublas', us=us, tflops=flop / us * 1e-6, over_floor=us / floor_us)
            rows.append(r)
            print(f'{name:38s} {M:6d} {N:5d} {Kd:6d} {"cublas":>6s} {"":>8s} {"":>5s} {us:8.1f} {"":>5s} {"":>7s} '
                  f'{r["tflops"]:8.1f} {"":>7s} {r["over_floor"]:7.2f}')
        if name.startswith('fc1 fwd split'):
            # the rest of the split form: vt_gelu_fwd_bf16 reads z and writes h (2 x M x N bf16)
            z = torch.randn(M, N, device=dev).bfloat16()
            us = 1e3 * events_ms(lambda: K.gelu(z), args.reps, args.warmup)
            r = dict(gemm='gelu kernel (after fc1 split)', M=M, N=N, K=0, tile='-', us=us, gbs=4.0 * M * N / us * 1e-3)
            rows.append(r)
            print(f'{r["gemm"]:38s} {M:6d} {N:5d} {0:6d} {"-":>6s} {"":>8s} {"":>5s} {us:8.1f} {"":>5s} {"":>7s} '
                  f'{"":>8s} {r["gbs"]:7.0f}')


def k_sweep(K, dev, args, sms, rows):
    import numpy as np
    print(f'k-sweep (BN = 128): t_tile = time / waves, waves = ceil(tiles / {sms} SMs); fit t_tile = a * kblocks + e')
    print(f'{"gemm":24s} {"K":>5s} {"kblk":>4s} {"waves":>5s} {"us reg":>8s} {"us stg":>8s} {"tile reg":>8s} {"tile stg":>8s}')
    for name, M, N, _, (a_mn, b_mn), kw, _, _ in cases(dev):
        if name not in SWEEP:
            continue
        waves = -(-(-(-M // 128) * -(-N // 128)) // sms)
        pts = {'0': [], '1': []}
        for Kd in SWEEP_K:
            a, b = operands(M, N, Kd, a_mn, b_mn, dev)
            kb = Kd // 64
            res = ab_us(lambda: K.gemm(a, b, M, N, Kd, a_mn=bool(a_mn), b_mn=bool(b_mn), force_bn=128, **kw), args)
            r = dict(gemm=name, sweep=True, M=M, N=N, K=Kd, tile=128, waves=waves, **fmt_ab(res))
            rows.append(r)
            for mode, key in (('0', 'us_reg'), ('1', 'us_staged')):
                pts[mode].append((kb, r[key] / waves))
            print(f'{name:24s} {Kd:5d} {kb:4d} {waves:5d} {r["us_reg"]:8.1f} {r["us_staged"]:8.1f} '
                  f'{r["us_reg"] / waves:8.2f} {r["us_staged"] / waves:8.2f}')
        fit = {}
        for mode, label in (('0', 'reg'), ('1', 'staged')):
            x, y = np.array(pts[mode]).T
            a_fit, e_fit = np.polyfit(x, y, 1)
            fit[label] = dict(a_us_per_kblock=float(a_fit), e_us_per_tile=float(e_fit))
        rows.append(dict(gemm=name, sweep_fit=fit))
        print(f'{name:24s} fit: register a = {fit["reg"]["a_us_per_kblock"]:.3f} us/k-block, e = '
              f'{fit["reg"]["e_us_per_tile"]:.2f} us/tile; staged a = {fit["staged"]["a_us_per_kblock"]:.3f}, '
              f'e = {fit["staged"]["e_us_per_tile"]:.2f}')


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument('--reps', type=int, default=50)
    ap.add_argument('--warmup', type=int, default=10)
    ap.add_argument('--rounds', type=int, default=3, help='alternating register / staged timings per row')
    ap.add_argument('--k-sweep', action='store_true', help='only the K sweep of the wide-output GEMMs')
    ap.add_argument('--json', default=None, help='also write the rows as JSON to this file')
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit('gemm_shapes: no CUDA device; these are GPU timings and there is no CPU fallback')
    from videotransformer_pytorch_b200 import _lib
    K = _lib.K
    dev = 'cuda:0'
    torch.manual_seed(0)
    info = card()
    sms = _lib.load_library().vt_sm_count()
    print(json.dumps({'card': info, 'sms': sms}))
    rows = []
    if args.k_sweep:
        k_sweep(K, dev, args, sms, rows)
    else:
        shapes(K, dev, args, rows)
    print(json.dumps({'card_after': card()}))
    if args.json:
        with open(args.json, 'w') as fh:
            json.dump({'card': info, 'rows': rows}, fh, indent=1)


if __name__ == '__main__':
    main()
