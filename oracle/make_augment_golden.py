"""Goldens of the GPU clip transforms (videotransformer_pytorch_b200/augment.py): the reference's own transforms
(data_transform.py, on torchvision) run on seeded synthetic uint8 clips.

    python oracle/make_augment_golden.py /path/to/VideoTransformer-pytorch

Writes tests/golden/augment_inputs.npz (+ continuation files) with the decode-resolution clips, and
tests/golden/augment_<pipeline>.npz for train (supervised), mim, val and test.  Each batch case holds the torch seed, the
clip indices, the parameters the reference drew (recorded by calling the same get_params in the same order under the
same seed) and the reference's uint8 output (before ToTensor + Normalize).  torchvision's version is recorded: the
reference does not pin it, so its semantics are those of the installed version."""
import math
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, 'tests', 'golden')

# (T, H, W): 256x340 and 320x427 decode sizes, a portrait frame, a frame small enough that the crop upscales,
# and an aspect ratio beyond 4/3 : 3/4 enough to make RandomResizedCrop fall back to its central crop
CLIPS = [(2, 256, 340), (2, 320, 427), (2, 340, 256), (2, 40, 56), (2, 16, 200)]
CASES = {'big': dict(S=224, clips=[0, 1, 2], seeds=[1]), 'small': dict(S=32, clips=[3, 4, 3, 4], seeds=[3, 4, 5, 6])}


def make_clip(k, T, H, W):
    """smooth content plus a little noise (compresses well), uint8 T C H W"""
    rng = np.random.default_rng(100 + k)
    y, x = np.mgrid[0:H, 0:W].astype(np.float64)
    frames = []
    for t in range(T):
        ph = rng.uniform(0, 2 * np.pi, 3)
        chans = [127.5 + 100 * np.sin(x / (9 + 5 * c) + y / (13 + 3 * c) + ph[c] + 0.3 * t) for c in range(3)]
        img = np.stack(chans) + rng.integers(-2, 3, (3, H, W))
        frames.append(np.clip(np.rint(img), 0, 255).astype(np.uint8))
    return np.stack(frames)


def pipelines(T, S):
    import data_transform as DT
    kw = dict(mean=(0.45,) * 3, std=(0.225,) * 3)
    train = DT.create_video_transform(input_size=S, is_training=True, hflip=0.5, color_jitter=0.4,
                                      interpolation='bicubic', **kw)
    mim, _ = DT.create_video_transform(input_size=S, is_training=True, scale=(0.5, 1.0), hflip=0.5, color_jitter=None,
                                       interpolation='bicubic', objective='mim', **kw)
    val = DT.create_video_transform(input_size=S, is_training=False, interpolation='bicubic', **kw)
    test = DT.Compose([DT.Resize(scale_range=(-1, 256)), DT.ThreeCrop(size=S)])
    return {'train': DT.Compose(train.transforms[:-2]), 'mim': mim, 'val': DT.Compose(val.transforms[:2]), 'test': test}


def draw_params(name, tf, clip):
    """The parameters the transform is about to draw, by the same get_params calls in Compose order (the generator is
    left where the transform leaves it)."""
    from torchvision import transforms as TV
    rows = []
    if name in ('train', 'mim'):
        rrc = tf.transforms[0]
        i, j, h, w = TV.RandomResizedCrop.get_params(clip, rrc.scale, rrc.ratio)
        flip = bool(torch.rand(1) < tf.transforms[1].p)
        rows += [i, j, h, w, int(flip)]
        if name == 'train':
            cj = tf.transforms[2]
            fn_idx, b, c, s, _ = cj.get_params(cj.brightness, cj.contrast, cj.saturation, cj.hue)
            rows += fn_idx.tolist() + [b, c, s]
    return np.array(rows, dtype=np.float64)


def main(ref_dir):
    sys.path.insert(0, ref_dir)
    import torchvision
    clips = [make_clip(k, *c) for k, c in enumerate(CLIPS)]
    # inputs: one clip per file (each under 1 MB)
    for k, c in enumerate(clips):
        path = os.path.join(GOLD, 'augment_inputs.npz' if k == 0 else f'augment_inputs.{k}.npz')
        np.savez_compressed(path, **{f'clip{k}': c})
    for name in ('train', 'mim', 'val', 'test'):
        out = {'torchvision_version': np.array(torchvision.__version__)}
        for case, spec in CASES.items():
            S = spec['S']
            clip_ids = [1] if (name, case) == ('test', 'big') else spec['clips']     # three views each: keep it small
            for seed in spec['seeds']:
                tf = pipelines(2, S)[name]
                if name == 'test':
                    tf.randomize_parameters()        # the reference's Resize builds its torchvision Resize here
                torch.manual_seed(seed)
                params = [draw_params(name, tf, torch.from_numpy(clips[k])) for k in clip_ids]
                torch.manual_seed(seed)
                ys = [tf(torch.from_numpy(clips[k])).numpy() for k in clip_ids]
                key = f'{case}/{seed}'
                out[f'{key}/S'] = np.array(S)
                out[f'{key}/clips'] = np.array(clip_ids)
                for b, (p, y) in enumerate(zip(params, ys)):
                    out[f'{key}/params{b}'] = p
                    out[f'{key}/y{b}'] = y               # T C S S, or views T C S S for test
        np.savez_compressed(os.path.join(GOLD, f'augment_{name}.npz'), **out)
        print(name, os.path.getsize(os.path.join(GOLD, f'augment_{name}.npz')))


if __name__ == '__main__':
    main(sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, '..', 'reference'))
