"""GPU RandAugment, host side, on the CPU: the restated draws against torchvision's RandAugment, the kernel's fp32 twin
(tests/emu_randaug.py) against torchvision's _apply_op over every op, sign, magnitude, size and several kinds of content
(bit for bit, except warped pixels whose fp64 source coordinate lies within the derived bound of a half-integer), the twin
and the whole host path under emulation against the reference goldens (oracle/make_randaug_golden.py), errors
and descriptor packing."""
import ctypes
import math

import numpy as np
import pytest
import torch

from tests.conftest import load_golden
from tests.emu_augment import parse
from tests.emu_kernels import EmuKernels
from tests.emu_randaug import GEOMETRIC, near_tie_mask, randaug_frames

OBJECTIVES = ('supervised', 'mim')
SIZES = (224, 256, 32, 17, 3, 2)
MAGNITUDES = (0, 9, 15, 30)
CONTENTS = ('random', 'smooth', 'constant_frame', 'constant_channel', 'two_valued', 'one_bin')


@pytest.fixture
def emu_ra():
    from videotransformer_pytorch_b200 import _lib
    old = _lib.K
    _lib.K = EmuKernels(exact=True, inference_forms=True)
    yield _lib.K
    _lib.K = old


def content(kind, S, seed=0, T=2):
    """uint8 [T, S, S, 3]"""
    g = np.random.default_rng(seed + S)
    if kind == 'random':
        x = g.integers(0, 256, (T, S, S, 3))
    elif kind == 'smooth':
        y, xx = np.mgrid[0:S, 0:S]
        x = np.stack([np.stack([127.5 + 100 * np.sin(xx / (5 + c) + y / (7 + 2 * c) + t) for c in range(3)], -1)
                      for t in range(T)])
    elif kind == 'constant_frame':
        x = np.full((T, S, S, 3), 77)
    elif kind == 'constant_channel':
        x = g.integers(0, 256, (T, S, S, 3))
        x[..., 1] = 200
    elif kind == 'two_valued':
        x = np.where(g.random((T, S, S, 3)) < 0.3, 40, 200)
    else:                                                    # every pixel in one bin but one
        x = np.full((T, S, S, 3), 128)
        x[:, S // 2, S // 3] = (3, 250, 129)
    return torch.from_numpy(np.rint(x).clip(0, 255).astype(np.uint8))


def slot(op, m, S):
    """the (op, arg, one_minus, theta) the kernel reads for one drawn op, via the host's descriptor packing"""
    from videotransformer_pytorch_b200 import _lib
    from videotransformer_pytorch_b200 import augment as A
    d = _lib.RandAugDesc()
    A._pack_randaug(d, [(op, m)], S)
    return d.op[0], d.arg[0], d.one_minus[0], list(d.theta[0])


def compare(mine, ref, op, theta, S):
    """-> (differing bytes that are not exempt, exempt pixels); mine / ref uint8 [T, S, S, 3]"""
    diff = (mine != ref).any(dim=-1)
    if op in GEOMETRIC:
        near, _ = near_tie_mask(theta, S)
        return int((diff & ~torch.from_numpy(near)[None]).sum()), int(near.sum())
    return int(diff.sum()), 0


@pytest.mark.parametrize('num_ops,magnitude,bins', [(2, 9, 31), (4, 15, 31), (1, 30, 31), (3, 0, 11), (0, 9, 31)])
def test_draws_match_randaugment(monkeypatch, num_ops, magnitude, bins):
    AA = pytest.importorskip('torchvision.transforms.autoaugment')
    from videotransformer_pytorch_b200 import augment as A
    rec = []
    monkeypatch.setattr(AA, '_apply_op', lambda img, name, m, interpolation, fill: rec.append((name, m)) or img)
    for S in (224, 32):
        for seed in range(40):
            torch.manual_seed(seed)
            del rec[:]
            AA.RandAugment(num_ops, magnitude, bins)(torch.zeros(2, 3, S, S, dtype=torch.uint8))
            after = torch.rand(1)
            torch.manual_seed(seed)
            mine = A.rand_augment_params(S, num_ops, magnitude, bins)
            assert [(A.RANDAUG_OPS[op], m) for op, m in mine] == rec, (S, seed)
            assert torch.equal(torch.rand(1), after)                 # the generator is left where torchvision leaves it


def test_magnitude_table_values():
    from videotransformer_pytorch_b200 import augment as A
    mags = {A.RANDAUG_OPS[k]: float(m[9]) for k, (m, _) in enumerate(A._randaug_space(31, 224)) if m.ndim}
    assert mags['ShearX'] == 0.09000000357627869 and mags['Rotate'] == 9.0 and mags['Posterize'] == 7.0
    assert int(mags['TranslateX']) == 30 and int(float(A._randaug_space(31, 32)[3][0][9])) == 4
    assert mags['Solarize'] == 178.5 and mags['Brightness'] == 0.26999998092651367


@pytest.mark.parametrize('S', SIZES)
@pytest.mark.parametrize('op', range(14))
def test_twin_against_apply_op(op, S):
    """every sign, magnitude and content: bit for bit except the exempt (near-tie) warped pixels, whose count is printed"""
    AA = pytest.importorskip('torchvision.transforms.autoaugment')
    from torchvision.transforms import InterpolationMode
    from videotransformer_pytorch_b200 import augment as A
    name = A.RANDAUG_OPS[op]
    mags, signed = A._randaug_space(31, S)[op]
    exempt, px = 0, 0
    for mi in MAGNITUDES if mags.ndim else (0,):
        m0 = float(mags[mi].item()) if mags.ndim else 0.0
        for m in ((m0, -m0) if signed else (m0,)):
            for kind in CONTENTS:
                x = content(kind, S, seed=op + mi)
                ref = AA._apply_op(x.permute(0, 3, 1, 2), name, m, InterpolationMode.NEAREST, None).permute(0, 2, 3, 1)
                s = slot(op, m, S)
                bad, near = compare(randaug_frames(x, [s]), ref, op, s[3], S)
                assert bad == 0, (name, m, kind)
                exempt, px = exempt + near, px + S * S
    print(f'{name} S={S}: {exempt} of {px} pixels exempt (fp64 source within the bound of a half-integer)')


def test_warp_bound_at_224():
    from videotransformer_pytorch_b200 import augment as A
    for op, m in ((5, 9.0), (5, -9.0), (1, 0.09000000357627869), (2, -0.09000000357627869), (3, 30.45)):
        near, b = near_tie_mask(A.randaug_theta(op, m, 224), 224)
        print(f'op {op} m {m}: bound {b:.2e}, {int(near.sum())} of {224 * 224} pixels within it')
        assert b < 3e-4 and near.sum() < 100


def _golden(objective):
    z = load_golden(f'augment_randaug_{objective}')
    keys = sorted({k.rsplit('/', 1)[0] for k in z.files if '/' in k})
    return z, keys


def _golden_ops(p):
    n = int(p[5])
    return [(int(p[6 + 2 * s]), float(p[7 + 2 * s])) for s in range(n)]


def test_goldens_cover_every_op_and_sign():
    for objective in OBJECTIVES:
        z, keys = _golden(objective)
        assert str(z['torchvision_version']).startswith('0.26')
        seen = {(op, m < 0) for key in keys for b in range(len(z[f'{key}/clips'])) for op, m in _golden_ops(z[f'{key}/params{b}'])}
        assert {op for op, _ in seen} == set(range(14)) and all((op, True) in seen for op in range(1, 10)), objective


def _near_any(slots, S):
    near = np.zeros((S, S), bool)
    for s in slots:
        if s[0] in GEOMETRIC:
            near |= near_tie_mask(s[3], S)[0]
    return near


def _check_against_golden(mine, ref, slots, S):
    """-> pixels that differ; each must be behind a near-tie warp (a warped pixel whose fp64 source is within the bound
    of a half-integer can move every later op's input, so any differing pixel needs such a warp among the ops)"""
    diff = (mine != ref).any(dim=-1)
    if diff.any():
        assert _near_any(slots, S).any()
    return int(diff.sum())


@pytest.mark.parametrize('objective', OBJECTIVES)
def test_twin_on_golden_crops(objective):
    """the twin fed each golden's RandomResizedCrop + flip output and its recorded ops gives the golden's output"""
    z, keys = _golden(objective)
    n_diff, n_clips = 0, 0
    for key in keys:
        S = int(z[f'{key}/S'])
        for b in range(len(z[f'{key}/clips'])):
            pre = torch.from_numpy(z[f'{key}/pre{b}']).permute(0, 2, 3, 1).contiguous()
            ref = torch.from_numpy(z[f'{key}/y{b}']).permute(0, 2, 3, 1)
            slots = [slot(op, m, S) for op, m in _golden_ops(z[f'{key}/params{b}'])]
            n_diff += _check_against_golden(randaug_frames(pre, slots), ref, slots, S)
            n_clips += 1
    print(f'{objective}: {n_diff} pixels differ over {n_clips} clips, each behind a near-tie warp')


@pytest.mark.parametrize('objective', OBJECTIVES)
def test_host_path_reproduces_goldens(emu_ra, objective):
    """create_video_transform(auto_augment='rand_aug') under the kernel twin, fed the golden's clips under its seed: crop,
    flip and RandAugment ops identical; the crop within 1 of the reference's (the resize's near-half-integer bytes); the
    output is the twin's RandAugment of that crop, and equals the reference's wherever the crop does (near-tie warps
    aside)."""
    from videotransformer_pytorch_b200 import augment as A
    from tests.emu_augment import resize_window
    from tests.test_augment_host import _golden_clips
    clips = _golden_clips()
    z, keys = _golden(objective)
    same_crop, n_all = 0, 0
    for key in keys:
        S, ids = int(z[f'{key}/S']), [int(i) for i in z[f'{key}/clips']]
        kw = dict(scale=(0.5, 1.0), objective='mim') if objective == 'mim' else {}
        tf = A.create_video_transform(S, is_training=True, auto_augment='rand_aug', interpolation='bicubic',
                                      device='cpu', **kw)
        assert tf.rand_augment == (2, 9, 31) and tf.jitter is None
        torch.manual_seed(int(key.split('/')[1]))
        out = tf([torch.from_numpy(clips[i]).permute(0, 2, 3, 1) for i in ids])
        for b, i in enumerate(ids):
            p, v = z[f'{key}/params{b}'], tf.params[b][0]
            assert v['crop'] == tuple(int(q) for q in p[:4]) and v['flip'] == bool(p[4]), key
            assert v['ra'] == _golden_ops(p), key
            pre = torch.from_numpy(z[f'{key}/pre{b}']).permute(0, 2, 3, 1)
            ref = torch.from_numpy(z[f'{key}/y{b}']).permute(0, 2, 3, 1)
            mine_pre = resize_window(clips[i].transpose(0, 2, 3, 1), v['crop'], (S, S), (0, 0), S, 0, v['flip'])
            assert int((mine_pre.int() - pre.int()).abs().max()) <= 1, key
            slots = [slot(op, m, S) for op, m in v['ra']]
            assert torch.equal(out[b, :], randaug_frames(mine_pre, slots)), key
            if torch.equal(mine_pre, pre):
                same_crop += 1
                _check_against_golden(out[b], ref, slots, S)
            n_all += 1
    print(f'{objective}: {same_crop} of {n_all} crops equal the reference bit for bit; their outputs match it')
    assert same_crop >= n_all // 2


def test_packing_and_launch_sequence(emu_ra):
    from videotransformer_pytorch_b200 import _lib
    from videotransformer_pytorch_b200 import augment as A
    g = torch.Generator().manual_seed(0)
    clips = [torch.randint(0, 256, (2, h, w, 3), dtype=torch.uint8, generator=g) for h, w in ((40, 56), (64, 48), (36, 36))]
    plain = A.create_video_transform(32, is_training=True, device='cpu')
    tf = A.create_video_transform(32, is_training=True, auto_augment=True, device='cpu')
    torch.manual_seed(3)
    a = plain(clips)
    torch.manual_seed(3)
    b = tf(clips)
    assert [c[0] for c in emu_ra.calls] == ['resized_crop_u8', 'color_jitter_u8', 'resized_crop_u8', 'rand_augment_u8']
    ncrop = 3 * ctypes.sizeof(_lib.CropDesc)
    assert plain.desc.numel() == ncrop + 3 * ctypes.sizeof(_lib.JitterDesc)        # the layout without RandAugment
    assert tf.desc.numel() == ncrop + 3 * ctypes.sizeof(_lib.RandAugDesc)
    k = ctypes.sizeof(_lib.CropDesc)                    # the first clip's crop and flip come before any op draw
    assert bytes(tf.desc[:k].numpy()) == bytes(plain.desc[:k].numpy())
    for d, v in zip(parse(tf.desc[ncrop:], _lib.RandAugDesc, 3), tf.params):
        ops = v[0]['ra']
        assert d.n_ops == 2 and [d.op[s] for s in range(2)] == [op for op, _ in ops]
        for s, (op, m) in enumerate(ops):
            if op in GEOMETRIC:
                assert list(d.theta[s]) == [float(t) for t in A.randaug_theta(op, m, 32)]
            elif 6 <= op <= 9:
                assert d.arg[s] == np.float32(1.0 + m) and d.one_minus[s] == np.float32(1.0 - (1.0 + m))
            elif op == 10:
                assert d.arg[s] == 256 - 2 ** (8 - int(m))
            elif op == 11:
                assert d.arg[s] == np.float32(m)
    tf.reserve(1 << 20, 5, device='cpu')
    assert tf.desc.numel() >= 5 * (ctypes.sizeof(_lib.CropDesc) + ctypes.sizeof(_lib.RandAugDesc))
    assert a.shape == b.shape == (3, 2, 32, 32, 3)


def test_bad_descriptor_zeroes_the_clip_and_sets_err(emu_ra):
    from videotransformer_pytorch_b200 import _lib
    x = content('random', 16).unsqueeze(0).repeat(3, 1, 1, 1, 1)
    descs = (_lib.RandAugDesc * 3)()
    descs[0].n_ops, descs[0].op[0] = 1, 14
    descs[1].n_ops = 5
    descs[2].n_ops, descs[2].op[0], descs[2].arg[0] = 1, 10, 240.0
    err = torch.zeros(1, dtype=torch.int32)
    y = emu_ra.rand_augment_u8(x.clone(), torch.frombuffer(bytearray(bytes(descs)), dtype=torch.uint8), err)
    assert int(err) == 1 and int(y[:2].max()) == 0 and torch.equal(y[2], x[2] & 240)


def test_errors(emu_ra):
    from videotransformer_pytorch_b200 import augment as A
    with pytest.raises(NotImplementedError, match="rand_aug"):
        A.create_video_transform(224, is_training=True, auto_augment='rand-m9-mstd0.5-inc1')
    with pytest.raises(ValueError):
        A.create_video_transform(320, is_training=True, auto_augment='rand_aug')              # S <= 256
    with pytest.raises(ValueError):
        A.ClipTransform(224, 'train', color_jitter=0.4, rand_augment=(2, 9, 31))             # not with ColorJitter
    with pytest.raises(ValueError):
        A.ClipTransform(224, 'center', resize_to=256, rand_augment=(2, 9, 31))               # training only
    for bad in ((5, 9, 31), (2, 31, 31), (2, -1, 31), (2, 0, 1)):
        with pytest.raises(ValueError):
            A.ClipTransform(224, 'train', rand_augment=bad)
    val = A.create_video_transform(224, is_training=False, auto_augment='rand_aug', device='cpu')  # eval: not applied
    assert val.rand_augment is None
    assert emu_ra.calls == []
