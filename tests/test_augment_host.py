"""GPU clip transforms, host side, on the CPU: the restated parameter draws against torchvision's get_params, the kernels'
fp32 twin (tests/emu_augment.py) against torchvision's jitter (bit for bit) and F.interpolate's resize (within the stated
pre-rounding bound), the whole host path under emulation against the reference goldens (oracle/make_augment_golden.py),
and descriptor packing of mixed sizes."""
import numpy as np
import pytest
import torch

from tests.conftest import load_golden
from tests.emu_augment import axis_weights, jitter_frames, parse, resize_window
from tests.emu_kernels import EmuKernels

PIPELINES = ('train', 'mim', 'val', 'test')
SIZE_CLASSES = [(256, 340), (320, 427), (340, 256), (40, 56), (16, 200), (480, 640)]


def resize_bound(n_in_h, n_in_w, RH, RW, filter_id):
    """|twin - F.interpolate| before rounding.  Per pass of n taps, torch's weights may differ from the twin's by a few
    fp32 ulps of O(1) (FMA contraction in its filter, <= 2.4e-7 each on values <= 255) and each of its n accumulation steps
    by half an ulp of a partial sum <= 255 * sum|w| < 332 (1.5e-5); the width pass's error is carried through the height
    pass's weights (sum|w| <= 1.3).  So  2.3 * n * (1.5e-5 + 255 * 2.4e-7) <= 1.75e-4 * n  per axis, summed over axes."""
    from videotransformer_pytorch_b200.augment import max_taps
    return 1.75e-4 * (max_taps(n_in_h, RH, filter_id) + max_taps(n_in_w, RW, filter_id))


@pytest.fixture
def emu_aug():
    from videotransformer_pytorch_b200 import _lib
    old = _lib.K
    _lib.K = EmuKernels(exact=True, inference_forms=True)
    yield _lib.K
    _lib.K = old


def test_draws_match_torchvision_get_params():
    TV = pytest.importorskip('torchvision.transforms')
    from videotransformer_pytorch_b200 import augment as A
    fallbacks = 0
    for H, W in SIZE_CLASSES:
        for scale in ((0.08, 1.0), (0.5, 1.0)):
            for seed in range(40):
                img = torch.empty(3, H, W, dtype=torch.uint8)
                torch.manual_seed(seed)
                ref = TV.RandomResizedCrop.get_params(img, list(scale), [3. / 4., 4. / 3.])
                ref_flip = bool(torch.rand(1) < 0.5)
                cj = TV.ColorJitter(0.4, 0.4, 0.4)
                fn_idx, b, c, s, h = cj.get_params(cj.brightness, cj.contrast, cj.saturation, cj.hue)
                after = torch.rand(1)
                torch.manual_seed(seed)
                mine = A.random_resized_crop_params(H, W, scale, (3. / 4., 4. / 3.))
                flip = bool(torch.rand(1) < 0.5)
                ops = A.color_jitter_params((0.6, 1.4), (0.6, 1.4), (0.6, 1.4))
                assert mine == ref and flip == ref_flip, (H, W, seed)
                f = {0: b, 1: c, 2: s}
                assert ops == [(int(i), f[int(i)]) for i in fn_idx.tolist() if int(i) < 3] and h is None
                assert torch.equal(torch.rand(1), after)                   # the generator is left where torchvision leaves it
                fallbacks += (H, W) == (16, 200)
    assert fallbacks                                                       # 16 x 200 only ever takes the central crop


def test_fallback_branch_is_the_central_crop():
    from videotransformer_pytorch_b200 import augment as A
    torch.manual_seed(0)
    assert A.random_resized_crop_params(16, 200, (0.08, 1.0), (3. / 4., 4. / 3.)) == (0, 89, 16, 21)


@pytest.mark.parametrize('seed', range(12))
def test_jitter_twin_is_torchvision_bit_for_bit(seed):
    TV = pytest.importorskip('torchvision.transforms')
    g = np.random.default_rng(seed)
    S = [32, 224, 256, 17][seed % 4]
    clip = torch.from_numpy(g.integers(0, 256, (2, 3, S, S)).astype(np.uint8))
    if seed % 3 == 0:
        clip = (clip // 4 + 100).to(torch.uint8)           # low contrast: the mean sits mid-range
    cj = TV.ColorJitter(0.4, 0.4, 0.4)
    torch.manual_seed(seed)
    fn_idx, b, c, s, _ = cj.get_params(cj.brightness, cj.contrast, cj.saturation, cj.hue)
    torch.manual_seed(seed)
    ref = cj(clip)
    f = {0: b, 1: c, 2: s}
    ops = [(int(i), f[int(i)], float(np.float32(1.0 - f[int(i)]))) for i in fn_idx.tolist() if int(i) < 3]
    mine = jitter_frames(clip.permute(0, 2, 3, 1).contiguous(), ops)
    assert torch.equal(mine.permute(0, 3, 1, 2), ref)


def _preround(frames, crop, size, mode):
    import torch.nn.functional as F
    cy, cx, ch, cw = crop
    x = torch.from_numpy(frames).permute(0, 3, 1, 2)[:, :, cy:cy + ch, cx:cx + cw].float()
    return F.interpolate(x, size=size, mode=mode, align_corners=False, antialias=True).permute(0, 2, 3, 1)


def _twin_preround(frames, crop, size, filter_id):
    cy, cx, ch, cw = crop
    RH, RW = size
    x = torch.from_numpy(np.ascontiguousarray(frames[:, cy:cy + ch, cx:cx + cw])).float()
    lo_x, n_x, w_x = axis_weights(np.arange(RW), cw, RW, filter_id)
    lo_y, n_y, w_y = axis_weights(np.arange(RH), ch, RH, filter_id)
    h = torch.zeros((x.shape[0], ch, RW, 3))
    for j in range(int(n_x.max())):
        h = h + x[:, :, torch.from_numpy(np.minimum(lo_x + j, cw - 1))] * torch.from_numpy(w_x[:, j])[None, None, :, None]
    acc = torch.zeros((x.shape[0], RH, RW, 3))
    for i in range(int(n_y.max())):
        acc = acc + h[:, torch.from_numpy(np.minimum(lo_y + i, ch - 1))] * torch.from_numpy(w_y[:, i])[None, :, None, None]
    return acc


RESIZE_CASES = [((256, 340), (0, 0, 256, 340), (224, 224), 'bicubic'), ((256, 340), (10, 20, 200, 300), (224, 224), 'bicubic'),
                ((90, 70), (0, 0, 90, 70), (224, 224), 'bicubic'), ((320, 427), (0, 0, 320, 427), (256, 341), 'bilinear'),
                ((320, 427), (5, 9, 311, 400), (224, 224), 'bilinear'), ((480, 640), (0, 0, 480, 640), (96, 96), 'bicubic'),
                ((40, 52), (3, 1, 30, 44), (97, 61), 'bicubic'), ((448, 448), (0, 0, 448, 448), (64, 64), 'bicubic')]


@pytest.mark.parametrize('size,crop,out,mode', RESIZE_CASES)
def test_twin_resize_within_stated_bound_of_interpolate(size, crop, out, mode):
    g = np.random.default_rng(sum(size))
    fr = g.integers(0, 256, (2, *size, 3)).astype(np.uint8)
    fid = 0 if mode == 'bicubic' else 1
    err = (_preround(fr, crop, out, mode) - _twin_preround(fr, crop, out, fid)).abs().max().item()
    bound = resize_bound(crop[2], crop[3], out[0], out[1], fid)
    print(f'{size} crop {crop} -> {out} {mode}: max |twin - interpolate| = {err:.2e} (bound {bound:.2e})')
    assert err <= bound


def test_twin_resize_equals_torchvision_away_from_half_integers():
    TF = pytest.importorskip('torchvision.transforms.functional')
    g = np.random.default_rng(7)
    fr = g.integers(0, 256, (2, 256, 340, 3)).astype(np.uint8)
    crop = (12, 30, 210, 280)
    ref = TF.resized_crop(torch.from_numpy(fr).permute(0, 3, 1, 2), *crop, [224, 224],
                          interpolation=TF.InterpolationMode.BICUBIC, antialias=True).permute(0, 2, 3, 1)
    mine = resize_window(fr, crop, (224, 224), (0, 0), 224, 0, False)
    pre = _preround(fr, crop, (224, 224), 'bicubic')
    diff = (mine.int() - ref.int()).abs()
    bound = resize_bound(210, 280, 224, 224, 0)
    near_half = ((pre.clamp(0, 255) - pre.clamp(0, 255).floor() - 0.5).abs() <= bound)
    assert diff.max() <= 1 and bool((near_half | (diff == 0)).all())


def _golden_clips():
    z = load_golden('augment_inputs')
    return {int(k[4:]): z[k] for k in z.files}


def _golden_cases(name):
    z = load_golden(f'augment_{name}')
    keys = sorted({k.rsplit('/', 1)[0] for k in z.files if '/' in k})
    return z, keys


@pytest.mark.parametrize('name', PIPELINES)
def test_host_path_reproduces_goldens(emu_aug, name):
    """The transform under the kernel twin, fed the golden's clips under its seed: drawn parameters identical, outputs
    within 1 (a resize pixel one off where its pre-rounding value is near a half-integer); with jitter within 3, since up
    to three factors of at most 1.4 each can carry that one off to 1.4^3 < 3 before the last truncation."""
    from videotransformer_pytorch_b200 import augment as A
    clips = _golden_clips()
    z, keys = _golden_cases(name)
    assert str(z['torchvision_version']).startswith('0.26')
    worst, n_off, n_all = 0, 0, 0
    for key in keys:
        S, ids = int(z[f'{key}/S']), [int(i) for i in z[f'{key}/clips']]
        if name == 'test':
            tf = A.ThreeCropTest(256, S, device='cpu')
        else:
            kw = dict(scale=(0.5, 1.0), color_jitter=None, objective='mim') if name == 'mim' else {}
            tf = A.create_video_transform(S, is_training=name != 'val', interpolation='bicubic', device='cpu', **kw)
        seed = int(key.split('/')[1])
        torch.manual_seed(seed)
        out = tf([torch.from_numpy(clips[i]).permute(0, 2, 3, 1) for i in ids])
        assert out.shape == (len(ids) * tf.views, 2, S, S, 3)
        for b in range(len(ids)):
            p = z[f'{key}/params{b}']
            if name in ('train', 'mim'):
                v = tf.params[b][0]
                assert v['crop'] == tuple(int(q) for q in p[:4]) and v['flip'] == bool(p[4]), key
                if name == 'train':
                    f = {0: p[9], 1: p[10], 2: p[11]}
                    assert [(op, fac) for op, fac in v['ops']] == [(int(i), f[int(i)]) for i in p[5:9] if int(i) < 3]
            y = torch.from_numpy(z[f'{key}/y{b}'])
            ref = y.permute(0, 1, 3, 4, 2) if name == 'test' else y.permute(0, 2, 3, 1)[None]
            got = out[b * tf.views:(b + 1) * tf.views]
            d = (got.int() - ref.int()).abs()
            worst = max(worst, int(d.max()))
            n_off += int((d > 0).sum())
            n_all += d.numel()
    print(f'{name}: max |diff| {worst}, {n_off / n_all:.2e} of {n_all} bytes differ')
    assert worst <= (3 if name == "train" else 1) and n_off / n_all < 1e-2


def test_three_crop_views_and_offsets(emu_aug):
    """left, right, centre of the resized frame, clip-major, at y = (H - S) // 2 and x = 0, W - S, (W - S) // 2"""
    from videotransformer_pytorch_b200 import augment as A
    tf = A.ThreeCropTest(40, 32, device='cpu')
    views = tf.draw([(40, 100), (100, 40)])
    assert [v['window'] for v in views[0]] == [(4, 0), (4, 68), (4, 34)]
    assert [v['window'] for v in views[1]] == [(34, 0), (34, 8), (34, 4)]
    assert views[0][0]['resized'] == (40, 100) and views[1][0]['resized'] == (100, 40)
    val = A.create_video_transform(32, is_training=False, device='cpu')          # Resize(36) then CenterCrop(32)
    (v,), = val.draw([(320, 427)])
    assert v['resized'] == (36, 48) and v['window'] == (2, 8)


def test_packing_of_mixed_sizes(emu_aug):
    from videotransformer_pytorch_b200 import _lib
    from videotransformer_pytorch_b200 import augment as A
    g = torch.Generator().manual_seed(0)
    clips = [torch.randint(0, 256, (3, h, w, 3), dtype=torch.uint8, generator=g) for h, w in ((40, 56), (64, 48), (36, 36))]
    tchw = [clips[0].permute(0, 3, 1, 2), clips[1], clips[2]]            # the dataset's permuted view is accepted too
    packed, labels = A.collate_uint8([(c, k) for k, c in enumerate(tchw)])
    assert isinstance(packed, A.PackedClips) and labels.tolist() == [0, 1, 2]
    assert packed.sizes.tolist() == [[3, 40, 56, 0], [3, 64, 48, 3 * 40 * 56 * 3], [3, 36, 36, 3 * (40 * 56 + 64 * 48) * 3]]
    for c, (T, H, W, off) in zip(clips, packed.sizes.tolist()):
        assert torch.equal(packed.data[off:off + T * H * W * 3].view(T, H, W, 3), c)
    tf = A.create_video_transform(32, is_training=True, device='cpu')
    torch.manual_seed(3)
    a = tf(packed)
    torch.manual_seed(3)
    b = tf(clips)                                                        # list form: same draws, same bytes
    assert torch.equal(a, b)
    crops = parse(tf.desc, _lib.CropDesc, 3)
    assert [(d.src_offset, d.H, d.W, d.pitch) for d in crops] == [(o, h, w, 3 * w) for _, h, w, o in packed.sizes.tolist()]
    assert [c[0] for c in emu_aug.calls if 'crop' in c[0] or 'jitter' in c[0]] == ['resized_crop_u8', 'color_jitter_u8'] * 2


def test_errors(emu_aug):
    from videotransformer_pytorch_b200 import augment as A
    with pytest.raises(NotImplementedError):
        A.create_video_transform(224, is_training=True, auto_augment='rand-m9-mstd0.5-inc1')
    with pytest.raises(ValueError):
        A.create_video_transform(320, is_training=True, color_jitter=0.4)                      # jitter needs S <= 256
    with pytest.raises(ValueError):
        A.create_video_transform(224, is_training=True, interpolation='random')
    tf = A.create_video_transform(32, is_training=False, device='cpu')
    with pytest.raises(ValueError):
        tf([torch.zeros(2, 40, 40, 3, dtype=torch.uint8), torch.zeros(3, 40, 40, 3, dtype=torch.uint8)])   # mixed T
    with pytest.raises(ValueError):                 # 600 -> 36 (val short side): a 16.7x bicubic downscale, > 32 taps
        A.create_video_transform(32, is_training=False, interpolation='bicubic', device='cpu')(
            [torch.zeros(1, 600, 600, 3, dtype=torch.uint8)])
    assert emu_aug.calls == []
