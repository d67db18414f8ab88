"""GPU clip transforms (csrc/vt_augment.cu through augment.py) on the H100: the kernels bit for bit against their CPU twin
(tests/emu_augment.py), the resize against torch within the stated pre-rounding bound, the jitter against torchvision
exactly, every pipeline against the reference goldens, views / flip / mixed sizes, guard bytes, graph replay and the models
and HOG targets fed the transformed clip."""
import ctypes as C

import numpy as np
import pytest
import torch

from tests.emu_augment import resize_window
from tests.emu_kernels import EmuKernels
from tests.test_augment_host import PIPELINES, _golden_cases, _golden_clips, _preround, resize_bound

pytestmark = pytest.mark.gpu
dev = torch.device('cuda')


def _crop_desc(H, W, crop, resized, window=(0, 0), flip=0, filter_id=0, offset=0):
    from videotransformer_pytorch_b200 import _lib
    d = _lib.CropDesc()
    d.src_offset, d.H, d.W, d.pitch = offset, H, W, 3 * W
    d.crop_y, d.crop_x, d.crop_h, d.crop_w = crop
    d.RH, d.RW = resized
    d.oy, d.ox = window
    d.flip, d.filter = flip, filter_id
    return bytes(d)


def _dev_bytes(b):
    return torch.frombuffer(bytearray(b), dtype=torch.uint8).to(dev)


RESIZE = [((256, 340), (0, 0, 256, 340), (224, 224), 'bicubic'), ((256, 340), (17, 41, 199, 263), (224, 224), 'bicubic'),
          ((320, 427), (0, 0, 320, 427), (224, 224), 'bicubic'), ((90, 70), (0, 0, 90, 70), (224, 224), 'bicubic'),
          ((320, 427), (5, 9, 311, 400), (224, 224), 'bilinear'), ((480, 640), (0, 0, 480, 640), (96, 96), 'bicubic'),
          ((40, 52), (3, 1, 30, 44), (64, 64), 'bicubic')]


@pytest.mark.parametrize('size,crop,out,mode', RESIZE)
def test_resize_kernel_against_twin_and_torch(size, crop, out, mode):
    from videotransformer_pytorch_b200 import _lib
    g = np.random.default_rng(sum(size) + crop[0])
    fr = g.integers(0, 256, (2, *size, 3)).astype(np.uint8)
    fid = 0 if mode == 'bicubic' else 1
    S = out[0]
    src = torch.from_numpy(fr).reshape(-1).to(dev)
    err = torch.zeros(1, dtype=torch.int32, device=dev)
    y = torch.empty((1, 2, S, S, 3), dtype=torch.uint8, device=dev)
    _lib.K.resized_crop_u8(src, _dev_bytes(_crop_desc(*size, crop, out, filter_id=fid)), y, err)
    y = y[0].cpu()
    assert int(err) == 0
    assert torch.equal(y, resize_window(fr, crop, out, (0, 0), S, fid, False))          # the twin, bit for bit
    pre = _preround(fr, crop, out, mode).clamp(0, 255)
    ref = torch.round(pre).to(torch.uint8)
    d = (y.int() - ref.int()).abs()
    bound = resize_bound(crop[2], crop[3], out[0], out[1], fid)
    near_half = (pre - pre.floor() - 0.5).abs() <= bound
    print(f'{size} {crop} -> {out} {mode}: {float((d > 0).float().mean()):.2e} of pixels +-1')
    assert int(d.max()) <= 1 and bool((near_half | (d == 0)).all())


def test_jitter_kernel_on_its_resize_output_is_torchvision():
    TV = pytest.importorskip('torchvision.transforms')
    from videotransformer_pytorch_b200 import augment as A
    g = torch.Generator().manual_seed(1)
    clips = [torch.randint(0, 256, (4, 256, 340, 3), dtype=torch.uint8, generator=g) for _ in range(6)]
    tf = A.create_video_transform(224, is_training=True, interpolation='bicubic')
    torch.manual_seed(5)
    tf.prepare([c.to(dev) for c in clips])
    n = len(clips)
    y = torch.empty((n, 4, 224, 224, 3), dtype=torch.uint8, device=dev)
    from videotransformer_pytorch_b200 import _lib
    _lib.K.resized_crop_u8(tf.src, tf.desc[:n * C.sizeof(_lib.CropDesc)], y, tf.err)
    resized = y.cpu()
    _lib.K.color_jitter_u8(y, tf.desc[n * C.sizeof(_lib.CropDesc):])
    for b in range(n):
        ops = tf.params[b][0]['ops']
        ref = resized[b].permute(0, 3, 1, 2)
        for op, f in ops:
            fn = {0: TV.functional.adjust_brightness, 1: TV.functional.adjust_contrast, 2: TV.functional.adjust_saturation}[op]
            ref = fn(ref, f)
        assert torch.equal(y[b].cpu(), ref.permute(0, 2, 3, 1)), (b, ops)


@pytest.mark.parametrize('name', PIPELINES)
def test_pipelines_against_goldens_and_twin(name):
    from videotransformer_pytorch_b200 import _lib
    from videotransformer_pytorch_b200 import augment as A
    clips = _golden_clips()
    z, keys = _golden_cases(name)
    worst, n_off, n_all = 0, 0, 0
    for key in keys:
        S, ids = int(z[f'{key}/S']), [int(i) for i in z[f'{key}/clips']]
        if name == 'test':
            mk = lambda d: A.ThreeCropTest(256, S, device=d)
        else:
            kw = dict(scale=(0.5, 1.0), color_jitter=None, objective='mim') if name == 'mim' else {}
            mk = lambda d: A.create_video_transform(S, is_training=name != 'val', interpolation='bicubic', device=d, **kw)
        seed = int(key.split('/')[1])
        torch.manual_seed(seed)
        tf = mk(None)
        out = tf([torch.from_numpy(clips[i]).permute(0, 2, 3, 1).to(dev) for i in ids]).cpu()
        assert int(tf.err) == 0
        old = _lib.K
        _lib.K = EmuKernels(exact=True, inference_forms=True)
        try:
            torch.manual_seed(seed)
            twin = mk('cpu')([torch.from_numpy(clips[i]).permute(0, 2, 3, 1) for i in ids])
        finally:
            _lib.K = old
        assert torch.equal(out, twin), key
        for b in range(len(ids)):
            y = torch.from_numpy(z[f'{key}/y{b}'])
            ref = y.permute(0, 1, 3, 4, 2) if name == 'test' else y.permute(0, 2, 3, 1)[None]
            d = (out[b * tf.views:(b + 1) * tf.views].int() - ref.int()).abs()
            worst, n_off, n_all = max(worst, int(d.max())), n_off + int((d > 0).sum()), n_all + d.numel()
    print(f'{name}: max |diff| {worst} against the reference, {n_off / n_all:.2e} of {n_all} bytes differ')
    assert worst <= (3 if name == 'train' else 1) and n_off / n_all < 1e-2


def test_flip_views_and_mixed_sizes_in_one_launch():
    from videotransformer_pytorch_b200 import _lib
    from videotransformer_pytorch_b200 import augment as A
    g = torch.Generator().manual_seed(2)
    clips = [torch.randint(0, 256, (3, h, w, 3), dtype=torch.uint8, generator=g).to(dev)
             for h, w in ((256, 340), (320, 427), (340, 256), (48, 64))]
    n0 = _lib.launch_count()
    tf = A.ThreeCropTest(256, 224)
    out = tf(clips)
    assert _lib.launch_count() - n0 == 1 and out.shape == (12, 3, 224, 224, 3)
    for b, c in enumerate(clips):
        RH, RW = A.resize_short_side(c.shape[1], c.shape[2], 256)
        for v, (oy, ox) in enumerate([((RH - 224) // 2, 0), ((RH - 224) // 2, RW - 224), ((RH - 224) // 2, (RW - 224) // 2)]):
            ref = resize_window(c.cpu().numpy(), (0, 0, c.shape[1], c.shape[2]), (RH, RW), (oy, ox), 224, 1, False)
            assert torch.equal(out[3 * b + v].cpu(), ref), (b, v)
    # flip: the mirrored window of the same resize
    src = clips[1].reshape(-1)
    y = torch.empty((2, 3, 224, 224, 3), dtype=torch.uint8, device=dev)
    desc = _crop_desc(320, 427, (10, 20, 300, 380), (224, 224)) + _crop_desc(320, 427, (10, 20, 300, 380), (224, 224), flip=1)
    _lib.K.resized_crop_u8(src, _dev_bytes(desc), y)
    assert torch.equal(y[1], y[0].flip(2))


def test_guard_bytes_and_bad_descriptors():
    from videotransformer_pytorch_b200 import _lib
    G, S, T = 4096, 224, 2
    n = 2
    buf = torch.full((n * T * S * S * 3 + 2 * G,), 0xA5, dtype=torch.uint8, device=dev)
    y = buf[G:G + n * T * S * S * 3].view(n, T, S, S, 3)
    fr = torch.randint(0, 256, (T, 256, 340, 3), dtype=torch.uint8, device=dev)
    src = fr.reshape(-1)
    err = torch.zeros(1, dtype=torch.int32, device=dev)
    good = _crop_desc(256, 340, (0, 0, 256, 340), (224, 224))
    _lib.K.resized_crop_u8(src, _dev_bytes(good + good), y, err)
    jd = _lib.JitterDesc()
    jd.n_ops, jd.op[0], jd.op[1], jd.op[2] = 3, 1, 2, 0
    for s, f in enumerate((1.4, 0.6, 1.2)):
        jd.factor[s], jd.one_minus[s] = f, np.float32(1.0 - np.float32(f))
    _lib.K.color_jitter_u8(y, _dev_bytes(bytes(jd) * n))
    torch.cuda.synchronize()
    assert int(err) == 0
    assert bool((buf[:G] == 0xA5).all()) and bool((buf[-G:] == 0xA5).all())
    # a source past the buffer, and a 20x downscale (more taps than the kernel holds): zeros and the error flag
    far = _crop_desc(256, 340, (0, 0, 256, 340), (224, 224), offset=1)
    steep = _crop_desc(256, 340, (0, 0, 256, 340), (16, 16))
    for bad, S2 in ((far, 224), (steep, 16)):
        err.zero_()
        y2 = torch.full((1, T, S2, S2, 3), 7, dtype=torch.uint8, device=dev)
        _lib.K.resized_crop_u8(src, _dev_bytes(bad), y2, err)
        assert int(err) == 1 and int(y2.max()) == 0


def test_graph_replay_with_other_clips_sizes_and_draws():
    from videotransformer_pytorch_b200 import augment as A
    tf = A.create_video_transform(224, is_training=True, interpolation='bicubic')
    ref_tf = A.create_video_transform(224, is_training=True, interpolation='bicubic')
    g = torch.Generator().manual_seed(3)

    def batch(sizes):
        return [torch.randint(0, 256, (4, h, w, 3), dtype=torch.uint8, generator=g) for h, w in sizes]
    first = A.pack_clips(batch([(256, 340)] * 4), pin=True)
    tf.reserve(4 * 4 * 320 * 454 * 3, 4)
    torch.manual_seed(0)
    tf.prepare(first)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        tf.run()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        static_out = tf.run()
    for k, sizes in enumerate([[(320, 427), (256, 340), (340, 256), (256, 454)], [(256, 340)] * 4, [(64, 80)] * 4]):
        clips = batch(sizes)
        torch.manual_seed(10 + k)
        tf.prepare(A.pack_clips(clips, pin=True))
        graph.replay()
        torch.manual_seed(10 + k)
        eager = ref_tf([c.to(dev) for c in clips])
        assert torch.equal(static_out, eager), k
    with pytest.raises(RuntimeError):
        tf.prepare(batch([(256, 340)] * 3))                  # 3 clips: the graph was captured for 4


def test_models_and_hog_fed_the_transformed_clip():
    """TimeSformer-B in eval and the MaskFeat HOG targets from the GPU transform's clip equal the same model / kernel fed the
    identical uint8 clip built on the host (the twin, from the kernel's own parameters)."""
    from videotransformer_pytorch_b200 import _lib, hog
    from videotransformer_pytorch_b200 import augment as A
    from videotransformer_pytorch_b200 import TimeSformer
    g = torch.Generator().manual_seed(4)
    clips = [torch.randint(0, 256, (8, h, w, 3), dtype=torch.uint8, generator=g) for h, w in ((256, 340), (320, 427))]
    for kind in ('val', 'mim'):
        if kind == 'val':
            mk = lambda d: A.create_video_transform(224, is_training=False, interpolation='bicubic', device=d)
        else:
            mk = lambda d: A.create_video_transform(224, is_training=True, scale=(0.5, 1.0), color_jitter=None,
                                                    interpolation='bicubic', objective='mim', device=d)
        torch.manual_seed(21)
        x = mk(None)([c.to(dev) for c in clips])
        old = _lib.K
        _lib.K = EmuKernels(exact=True, inference_forms=True)
        try:
            torch.manual_seed(21)
            host = mk('cpu')(clips)
        finally:
            _lib.K = old
        assert torch.equal(x.cpu(), host)
        if kind == 'val':
            torch.manual_seed(0)
            m = TimeSformer(num_frames=8, img_size=224).to(dev).eval()
            m.set_input_normalization((0.45,) * 3, (0.225,) * 3)
            with torch.no_grad():
                a, b = m(x), m(host.to(dev))
            assert torch.equal(a, b)
        else:
            markers = [[[0, 2], [2, 1]], [[1, 3]]]
            assert torch.equal(hog.hog_targets_batch(x, markers), hog.hog_targets_batch(host.to(dev), markers))
