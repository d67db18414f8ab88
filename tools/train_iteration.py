#!/usr/bin/env python
"""Whole training iteration (forward, backward, per-parameter clip, optimizer update) with the optimizer step eager after
the captured forward + backward, and with the optimizer step captured in the same graph.

    python tools/train_iteration.py [--reps 20] [--rounds 3] [--clip 1.0] [--configs all|name,name] [--json OUT]

Configurations: TimeSformer-B + 400-class head at batch 8 and 1 with AdamW and SGD-nesterov; ViViT-B + head at batch 1
with AdamW; MViT-B (MaskFeat.forward_features, cls row) + head at batch 8 with AdamW over the reference's layer-decay
groups (optimizer.py:57-158, layer_decay 0.75).  The optimizers use the decay / no-decay groups of the reference, and the
LR and weight decay of the groups change before every iteration, as a scheduler would.  Arms:
  eager    : GraphedTrainStep replay, then opt.step(clip_grad=...)
  captured : GraphedTrainStep(optimizer=opt, clip_grad=...), one replay
Per arm and round, two numbers per iteration:
  device ms : CUDA events around `--reps` back-to-back iterations, synchronised, divided by reps
  host us   : wall time of each call until it returns, with the GPU idle when the call starts (a synchronise before
              each call, outside the window; none inside it), averaged over reps
The arms alternate in one process, `--rounds` times; each cell is the median over the rounds, with the range beside it.
The card's name and power limit are read with a read-only nvidia-smi query in the same run.  Needs a CUDA device.
"""
from __future__ import annotations

import argparse
import json
import math
import os
import statistics
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

NUM_CLASSES, IMG = 400, 224
CONFIGS = {      # name: (backbone, batch, optimizer)
    'timesformer-b8-adamw': ('timesformer', 8, 'adamw'),
    'timesformer-b8-sgd': ('timesformer', 8, 'sgd'),
    'timesformer-b1-adamw': ('timesformer', 1, 'adamw'),
    'timesformer-b1-sgd': ('timesformer', 1, 'sgd'),
    'vivit-b1-adamw': ('vivit', 1, 'adamw'),
    'mvit-b8-adamw-layer-decay': ('mvit', 8, 'adamw'),
}


def card():
    q = subprocess.run(['nvidia-smi', '-i', str(torch.cuda.current_device()),
                        '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True)
    return q.stdout.strip() if q.returncode == 0 else torch.cuda.get_device_name()


class Trainee(torch.nn.Module):
    """backbone + ClassificationHead + cross-entropy (model_trainer.py:189-216 without mixup)"""

    def __init__(self, backbone):
        super().__init__()
        from videotransformer_pytorch_b200 import ClassificationHead, MaskFeat, TimeSformer, ViViT
        self.backbone = backbone
        if backbone == 'timesformer':
            self.model = TimeSformer(num_frames=8, img_size=IMG, patch_size=16, embed_dims=768, num_heads=12,
                                     num_transformer_layers=12, attention_type='divided_space_time')
        elif backbone == 'vivit':
            self.model = ViViT(num_frames=16, img_size=IMG, patch_size=16, embed_dims=768, num_heads=12,
                               num_transformer_layers=12, attention_type='fact_encoder')
        else:
            self.model = MaskFeat(pool_q_stride_size=[[1, 1, 2, 2], [3, 1, 2, 2]], feature_dim=2 * 2 * 2 * 3 * 9)
            # fine-tuning freezes the decoder (model_trainer.py:78-79); forward_features does not use the mask token
            for p in self.model.decoder_pred.parameters():
                p.requires_grad = False
            self.model.mask_token.requires_grad = False
        self.cls_head = ClassificationHead(NUM_CLASSES, self.model.embed_dims)
        with torch.no_grad():
            for n, p in self.model.named_parameters():
                if 'temporal_fc' in n:
                    p.normal_(std=0.02)

    def forward(self, x, y):
        f = self.model.forward_features(x)[:, 0] if self.backbone == 'mvit' else self.model(x)
        return torch.nn.functional.cross_entropy(self.cls_head(f), y)


def decay_groups(net, lr, wd):
    """get_pretrain_param_groups (optimizer.py:44-63): 1-D tensors and biases without weight decay"""
    no, yes = [], []
    for n, p in net.named_parameters():
        if p.requires_grad:
            (no if p.ndim == 1 or n.endswith('.bias') else yes).append(p)
    return [{'params': no, 'weight_decay': 0., 'lr': lr}, {'params': yes, 'weight_decay': wd, 'lr': lr}]


def layer_decay_groups(net, lr, wd, layer_decay=0.75, num_layers=16):
    """build_finetune_optimizer for arch='mvit': a group per (layer, decay / no-decay) with lr_scale =
    layer_decay ** (num_layers + 1 - layer); patch embedding and positions are layer 0, block i is layer i + 1, the
    rest (final norm, head) the last layer"""
    L = num_layers + 2
    skip = net.model.no_weight_decay_keywords()
    groups = {}
    for name, p in net.named_parameters():
        if not p.requires_grad:
            continue
        short = name.replace('model.', '', 1).replace('mvit.', '', 1)
        nd = p.ndim == 1 or name.endswith('.bias') or any(s in name for s in skip)
        if short.startswith('patch_embed') or short.startswith('cls_positional_encoding'):
            layer = 0
        elif short.startswith('blocks'):
            layer = int(short.split('.')[1]) + 1
        else:
            layer = L - 1
        scale = layer_decay ** (L - 1 - layer)
        g = groups.setdefault((layer, nd), {'params': [], 'weight_decay': 0. if nd else wd, 'lr': lr * scale,
                                            'lr_scale': scale})
        g['params'].append(p)
    return list(groups.values())


def make_optimizer(net, backbone, kind):
    from videotransformer_pytorch_b200.optim import FusedAdamW, FusedSGD
    if kind == 'sgd':
        return FusedSGD(decay_groups(net, 5e-3, 1e-4), lr=5e-3, momentum=0.9, nesterov=True, weight_decay=1e-4)
    groups = layer_decay_groups(net, 5e-4, 0.05) if backbone == 'mvit' else decay_groups(net, 5e-4, 0.05)
    return FusedAdamW(groups, lr=5e-4, betas=(0.9, 0.999), weight_decay=0.05)


def schedule(opt, it):
    """what a scheduler does between steps: rewrite every group's lr and the decay group's weight decay"""
    f = 0.5 * (1 + math.cos(math.pi * (it % 100) / 100))
    for g in opt.param_groups:
        g.setdefault('base_lr', g['lr'])
        g['lr'] = g['base_lr'] * f
        if g['weight_decay']:
            g['weight_decay'] = 0.05 + 0.01 * f


def measure(name, args):
    from videotransformer_pytorch_b200.graph import GraphedTrainStep
    backbone, B, kind = CONFIGS[name]
    frames = 8 if backbone == 'timesformer' else 16
    torch.manual_seed(0)
    net = Trainee(backbone).cuda().train()
    g = torch.Generator().manual_seed(1)
    x = torch.randn(B, frames, 3, IMG, IMG, generator=g).cuda()
    y = torch.randint(0, NUM_CLASSES, (B,), generator=g).cuda()
    opt_e, opt_c = make_optimizer(net, backbone, kind), make_optimizer(net, backbone, kind)
    plain = GraphedTrainStep(net, (x, y))
    captured = GraphedTrainStep(net, (x, y), optimizer=opt_c, clip_grad=args.clip)
    it = [0]

    def eager_arm():
        schedule(opt_e, it[0])
        plain(x, y)
        opt_e.step(clip_grad=args.clip)
        it[0] += 1

    def captured_arm():
        schedule(opt_c, it[0])
        captured(x, y)
        it[0] += 1

    arms = {'eager': eager_arm, 'captured': captured_arm}
    for fn in arms.values():        # warm both arms (first eager step binds the tables)
        for _ in range(3):
            fn()
    torch.cuda.synchronize()
    res = {a: {'device_ms': [], 'host_us': []} for a in arms}
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for r in range(args.rounds):
        order = list(arms) if r % 2 == 0 else list(reversed(arms))
        for a in order:
            fn = arms[a]
            torch.cuda.synchronize()
            t0.record()
            for _ in range(args.reps):
                fn()
            t1.record()
            torch.cuda.synchronize()
            res[a]['device_ms'].append(t0.elapsed_time(t1) / args.reps)
            host = 0.0
            for _ in range(args.reps):
                torch.cuda.synchronize()
                h0 = time.perf_counter()
                fn()
                host += time.perf_counter() - h0
            torch.cuda.synchronize()
            res[a]['host_us'].append(1e6 * host / args.reps)
    out = {'config': name, 'batch': B, 'optimizer': kind, 'params_in_table': len(opt_c._tab.params),
           'kernels_per_replay': {'eager': plain.kernels_per_replay, 'captured': captured.kernels_per_replay}}
    for a in arms:
        for k, v in res[a].items():
            out[f'{a}_{k}'] = dict(median=statistics.median(v), min=min(v), max=max(v), runs=v)
    del plain, captured, opt_e, opt_c, net
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument('--reps', type=int, default=20)
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--clip', type=float, default=1.0)
    ap.add_argument('--configs', default='all')
    ap.add_argument('--json', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('train_iteration.py needs a CUDA device')
    names = list(CONFIGS) if args.configs == 'all' else args.configs.split(',')
    gpu = card()
    print(f'# {gpu}; {args.rounds} rounds x {args.reps} iterations per arm, clip_grad {args.clip}')
    print('| config | eager device ms | captured device ms | eager host us | captured host us |')
    print('|---|---|---|---|---|')
    rows = []
    for n in names:
        r = measure(n, args)
        rows.append(r)
        cell = lambda d, f: f"{d['median']:{f}} ({d['min']:{f}}-{d['max']:{f}})"
        print(f"| {n} | {cell(r['eager_device_ms'], '.2f')} | {cell(r['captured_device_ms'], '.2f')} | "
              f"{cell(r['eager_host_us'], '.0f')} | {cell(r['captured_host_us'], '.0f')} |", flush=True)
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, 'w') as fh:
            json.dump({'card': gpu, 'clip': args.clip, 'reps': args.reps, 'rounds': args.rounds, 'results': rows},
                      fh, indent=1)


if __name__ == '__main__':
    main()
