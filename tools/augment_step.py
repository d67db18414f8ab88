#!/usr/bin/env python
"""GPU clip transforms (augment.py): device time per batch of each pipeline, the CPU transform they replace, and the
graphed TimeSformer-B train step with the transform inside it against the same step fed an already cropped uint8 clip.

    python tools/augment_step.py [--iters 50] [--steps 20] [--cpu-clips 10]

Prints one JSON line per measurement, after a line with the card's name and power limit read in the same run.
  * transform: CUDA events around `iters` back-to-back runs of the kernels on prepared arenas (batch 8, T = 8 and 16,
    all clips 256x340 or all 320x427), three windows: median and range.  train_ra / mim_ra are the training forms with
    auto_augment='rand_aug' (RandAugment in place of ColorJitter); their draws differ per prepare, the timed runs replay
    the last one.
  * cpu_reference: torchvision's composition of the reference's pipelines (data_transform.py:495-615 and the test
    transform of data_trainer.py:110-115, ToTensor + Normalize included) on one thread, per 8-frame clip, three windows.
  * train_step: ms per step of GraphedTrainStep over TimeSformer-B + a 400-class head at batch 8, 8 x 224^2, host work
    included (the transform's draws and its two uploads), with the train transform (ColorJitter), with the RandAugment
    train transform, and fed an already cropped clip; the three arms alternate over three windows each.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))

from resolution_step import Net, card  # noqa: E402

MEAN, STD = (0.45,) * 3, (0.225,) * 3


def forms(S=224):
    from videotransformer_pytorch_b200 import augment as A
    return {'train': lambda: A.create_video_transform(S, is_training=True, interpolation='bicubic', mean=MEAN, std=STD),
            'mim': lambda: A.create_video_transform(S, is_training=True, scale=(0.5, 1.0), color_jitter=None,
                                                    interpolation='bicubic', objective='mim', mean=MEAN, std=STD),
            'train_ra': lambda: A.create_video_transform(S, is_training=True, auto_augment='rand_aug', interpolation='bicubic',
                                                         mean=MEAN, std=STD),
            'mim_ra': lambda: A.create_video_transform(S, is_training=True, scale=(0.5, 1.0), auto_augment='rand_aug',
                                                       interpolation='bicubic', objective='mim', mean=MEAN, std=STD),
            'val': lambda: A.create_video_transform(S, is_training=False, interpolation='bicubic', mean=MEAN, std=STD),
            'test': lambda: A.ThreeCropTest(256, S, mean=MEAN, std=STD)}


def windows(fn, iters, n=3):
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    out = []
    for _ in range(n):
        t0.record()
        for _ in range(iters):
            fn()
        t1.record()
        torch.cuda.synchronize()
        out.append(t0.elapsed_time(t1) / iters)
    out.sort()
    return out


def transform_times(iters):
    from videotransformer_pytorch_b200 import augment as A
    g = torch.Generator().manual_seed(0)
    for T in (8, 16):
        for h, w in ((256, 340), (320, 427)):
            clips = A.pack_clips([torch.randint(0, 256, (T, h, w, 3), dtype=torch.uint8, generator=g) for _ in range(8)],
                                 pin=True)
            for name, mk in forms().items():
                tf = mk()
                tf.prepare(clips)
                tf.run()
                t = windows(tf.run, iters)
                torch.manual_seed(0)
                host = time.perf_counter()
                for _ in range(iters):
                    tf.prepare(clips)
                torch.cuda.synchronize()
                host = (time.perf_counter() - host) / iters
                yield dict(what='transform', form=name, batch=8, frames=T, decode=f'{h}x{w}', ms_per_batch=round(t[1], 4),
                           ms_range=[round(t[0], 4), round(t[2], 4)], prepare_ms=round(host * 1e3, 3),
                           kernel_launches=1 + int(tf.jitter is not None or tf.rand_augment is not None))


def cpu_reference(n_clips):
    try:
        from torchvision import transforms as TV
    except ImportError:
        return [dict(what='cpu_reference', note='torchvision not installed: not measured')]
    torch.set_num_threads(1)
    norm = TV.Normalize(torch.tensor(MEAN), torch.tensor(STD))
    to_tensor = lambda x: x.float().div(255)
    I = TV.InterpolationMode
    pipes = {'train': TV.Compose([TV.RandomResizedCrop(224, interpolation=I.BICUBIC), TV.RandomHorizontalFlip(0.5),
                                  TV.ColorJitter(0.4, 0.4, 0.4), to_tensor, norm]),
             'mim': TV.Compose([TV.RandomResizedCrop(224, scale=(0.5, 1.0), interpolation=I.BICUBIC),
                                TV.RandomHorizontalFlip(0.5), to_tensor, norm]),
             'train_ra': TV.Compose([TV.RandomResizedCrop(224, interpolation=I.BICUBIC), TV.RandomHorizontalFlip(0.5),
                                     TV.RandAugment(), to_tensor, norm]),
             'mim_ra': TV.Compose([TV.RandomResizedCrop(224, scale=(0.5, 1.0), interpolation=I.BICUBIC),
                                   TV.RandomHorizontalFlip(0.5), TV.RandAugment(), to_tensor, norm]),
             'val': TV.Compose([TV.Resize(256, interpolation=I.BICUBIC), TV.CenterCrop(224), to_tensor, norm]),
             'test': TV.Compose([TV.Resize(256), lambda x: torch.stack([x[..., 16:240, :224], x[..., 16:240, -224:],
                                                                         x[..., 16:240, 58:282]]), to_tensor, norm])}
    res = []
    for h, w in ((256, 340), (320, 427)):
        clip = torch.randint(0, 256, (8, 3, h, w), dtype=torch.uint8)
        for name, f in pipes.items():
            f(clip)
            ts = []
            for _ in range(3):
                t = time.perf_counter()
                for _ in range(n_clips):
                    f(clip)
                ts.append((time.perf_counter() - t) / n_clips * 1e3)
            ts.sort()
            res.append(dict(what='cpu_reference', form=name, frames=8, decode=f'{h}x{w}', threads=1,
                            ms_per_clip=round(ts[1], 2), ms_range=[round(ts[0], 2), round(ts[2], 2)]))
    torch.set_num_threads(os.cpu_count() or 1)
    return res


def train_steps(steps, warmup):
    from videotransformer_pytorch_b200 import augment as A
    from videotransformer_pytorch_b200.graph import GraphedTrainStep
    dev = torch.device('cuda')
    torch.manual_seed(0)
    net = Net(8).to(dev).train()
    net.model.set_input_normalization(MEAN, STD)
    y = torch.randint(0, 400, (8,), device=dev)
    g = torch.Generator().manual_seed(1)
    packed = [A.pack_clips([torch.randint(0, 256, (8, h, w, 3), dtype=torch.uint8, generator=g) for _ in range(8)], pin=True)
              for h, w in ((256, 340), (320, 427))]
    x = torch.randint(0, 256, (8, 8, 224, 224, 3), dtype=torch.uint8, generator=g).to(dev)
    plain = GraphedTrainStep(net, (x, y))
    graphed = {}
    for form in ('train', 'train_ra'):
        tf = forms()[form]()
        tf.reserve(8 * 8 * 320 * 427 * 3, 8)
        tf.prepare(packed[0])
        graphed[form] = (tf, GraphedTrainStep(lambda lab, tf=tf: net(tf.run(), lab), [y], params=list(net.parameters())))
    k = [0]

    def with_tf(form):
        tf, step = graphed[form]
        k[0] ^= 1
        tf.prepare(packed[k[0]])
        step(y)
    arms = {'cropped_uint8_input': lambda: plain(x, y), 'gpu_transform_inside': lambda: with_tf('train'),
            'gpu_transform_ra_inside': lambda: with_tf('train_ra')}
    steps_of = {'cropped_uint8_input': plain, 'gpu_transform_inside': graphed['train'][1],
                'gpu_transform_ra_inside': graphed['train_ra'][1]}
    times = {a: [] for a in arms}
    for fn in arms.values():
        for _ in range(warmup):
            fn()
    for _ in range(3):
        for a, fn in arms.items():
            torch.cuda.synchronize()
            t = time.perf_counter()
            for _ in range(steps):
                fn()
            torch.cuda.synchronize()
            times[a].append((time.perf_counter() - t) / steps * 1e3)
    for a, ts in times.items():
        ts.sort()
        yield dict(what='train_step', arm=a, batch=8, frames=8, ms_per_step=round(ts[1], 3),
                   ms_range=[round(ts[0], 3), round(ts[2], 3)],
                   kernels_per_replay=steps_of[a].kernels_per_replay)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=50)
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=5)
    ap.add_argument('--cpu-clips', type=int, default=10)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('augment_step.py measures on a CUDA device; none found')
    print(json.dumps(dict(card=card(), torch=torch.__version__)), flush=True)
    for r in transform_times(args.iters):
        print(json.dumps(r), flush=True)
    for r in train_steps(args.steps, args.warmup):
        print(json.dumps(r), flush=True)
    for r in cpu_reference(args.cpu_clips):
        print(json.dumps(r), flush=True)


if __name__ == '__main__':
    main()
