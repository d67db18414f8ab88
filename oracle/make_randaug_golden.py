"""Goldens of the GPU RandAugment training transform (augment.create_video_transform(..., auto_augment='rand_aug')): the
reference's own transforms (data_transform.py, on torchvision) with auto_augment='rand_aug', for the supervised and mim
objectives, run on the clips of tests/golden/augment_inputs*.npz (oracle/make_augment_golden.py).

    python oracle/make_randaug_golden.py /path/to/VideoTransformer-pytorch

Writes tests/golden/augment_randaug_<objective>.npz (+ continuation files, each under 1 MB).  Each batch case holds the
torch seed, the clip indices, the crop and flip the reference drew, the RandAugment ops it applied (op index in
torchvision's order and the magnitude handed to _apply_op, recorded by wrapping _apply_op), the RandomResizedCrop + flip
output before RandAugment and the final uint8 output (before ToTensor + Normalize).  Seeds of the S = 32 case are taken
in order until every op has appeared and every signed op with both signs."""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, 'tests', 'golden')
sys.path.insert(0, ROOT)

OPS = ('Identity', 'ShearX', 'ShearY', 'TranslateX', 'TranslateY', 'Rotate', 'Brightness', 'Color', 'Contrast',
       'Sharpness', 'Posterize', 'Solarize', 'AutoContrast', 'Equalize')
SIGNED = set(range(1, 10))
BIG = dict(S=224, clips=[0, 1, 2], seeds=[1])
SMALL = dict(S=32, clips=[3, 4, 3, 4])
MAX_BYTES = 900_000


def pipeline(S, objective):
    import data_transform as DT
    kw = dict(mean=(0.45,) * 3, std=(0.225,) * 3)
    if objective == 'mim':
        tf, _ = DT.create_video_transform(input_size=S, is_training=True, scale=(0.5, 1.0), hflip=0.5, auto_augment='rand_aug',
                                          interpolation='bicubic', objective='mim', **kw)
        return tf
    tf = DT.create_video_transform(input_size=S, is_training=True, hflip=0.5, auto_augment='rand_aug',
                                   interpolation='bicubic', **kw)
    return DT.Compose(tf.transforms[:-2])


def run_case(S, objective, seed, clips, clip_ids):
    """-> per clip (params, pre, y): the reference's transform under `seed`, with its draws recorded as it runs"""
    from torchvision import transforms as TV
    from torchvision.transforms import autoaugment as AA
    tf = pipeline(S, objective)
    rrc, flip, ra = tf.transforms
    assert isinstance(ra, AA.RandAugment) and len(tf.transforms) == 3
    applied, orig = [], AA._apply_op

    def record(img, op_name, magnitude, interpolation, fill):
        applied.append((OPS.index(op_name), magnitude))
        return orig(img, op_name, magnitude, interpolation, fill)
    torch.manual_seed(seed)
    out = []
    AA._apply_op = record
    try:
        for k in clip_ids:
            x = torch.from_numpy(clips[k])
            state = torch.get_rng_state()
            box = TV.RandomResizedCrop.get_params(x, rrc.scale, rrc.ratio)
            flipped = bool(torch.rand(1) < flip.p)
            torch.set_rng_state(state)
            pre = flip(rrc(x))
            del applied[:]
            y = ra(pre)
            ops = [v for a in applied for v in a]
            params = np.array(list(box) + [int(flipped), len(applied)] + ops, dtype=np.float64)
            out.append((params, pre.numpy(), y.numpy()))
    finally:
        AA._apply_op = orig
    return out


def write(name, arrays):
    """split the arrays over name.npz, name.1.npz, ... so that each file stays under MAX_BYTES"""
    import io
    parts, cur, size = [], {}, 0
    for k, v in arrays.items():
        buf = io.BytesIO()
        np.savez_compressed(buf, v)
        n = buf.tell()
        if cur and size + n > MAX_BYTES:
            parts.append(cur)
            cur, size = {}, 0
        cur[k], size = v, size + n
    parts.append(cur)
    for i, p in enumerate(parts):
        path = os.path.join(GOLD, f'{name}.npz' if i == 0 else f'{name}.{i}.npz')
        np.savez_compressed(path, **p)
        print(path, os.path.getsize(path))


def main(ref_dir):
    sys.path.insert(0, ref_dir)
    import torchvision
    from tests.conftest import load_golden
    z = load_golden('augment_inputs')
    clips = {int(k[4:]): z[k] for k in z.files}
    for objective in ('supervised', 'mim'):
        out = {'torchvision_version': np.array(torchvision.__version__)}
        seen = set()
        cases = [('big', BIG['S'], BIG['clips'], s) for s in BIG['seeds']]
        seed = 0
        todo = list(cases)
        while todo:
            case, S, ids, sd = todo.pop(0)
            key = f'{case}/{sd}'
            out[f'{key}/S'], out[f'{key}/clips'] = np.array(S), np.array(ids)
            for b, (p, pre, y) in enumerate(run_case(S, objective, sd, clips, ids)):
                out[f'{key}/params{b}'], out[f'{key}/pre{b}'], out[f'{key}/y{b}'] = p, pre, y
                for op, m in zip(p[6::2], p[7::2]):
                    seen.add((int(op), m < 0 if int(op) in SIGNED else False))
            need = {(op, neg) for op in range(14) for neg in ((False, True) if op in SIGNED else (False,))}
            if not todo and not need <= seen:
                todo.append(('small', SMALL['S'], SMALL['clips'], seed))
                seed += 1
        print(objective, 'small seeds', list(range(seed)))
        write(f'augment_randaug_{objective}', out)


if __name__ == '__main__':
    main(sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, '..', 'reference'))
