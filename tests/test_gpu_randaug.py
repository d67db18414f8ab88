"""GPU RandAugment (vt_rand_augment_u8 through augment.py) on the H100: the kernel bit for bit against its CPU twin
(tests/emu_randaug.py) over every op, sign, magnitude, size and content with several op lists in one launch, against
torchvision (near-tie warped pixels exempt), the pipelines against the reference goldens and the twin, guard bytes, bad
descriptors, graph replay, and the HOG targets and TimeSformer fed the transformed clip."""
import pytest
import torch

from tests.emu_augment import resize_window
from tests.emu_kernels import EmuKernels
from tests.emu_randaug import GEOMETRIC, desc_ops, near_tie_mask, randaug_frames
from tests.test_randaug_host import (CONTENTS, MAGNITUDES, OBJECTIVES, SIZES, _check_against_golden, _golden,
                                     _golden_ops, content, slot)

pytestmark = pytest.mark.gpu
dev = torch.device('cuda')


def _dev_bytes(b):
    return torch.frombuffer(bytearray(b), dtype=torch.uint8).to(dev)


def _op_lists(S, seed):
    """every op alone at every magnitude and sign, then random lists of 1-4 ops -> [[(op, m), ...], ...]"""
    from videotransformer_pytorch_b200 import augment as A
    lists = []
    for op in range(14):
        mags, signed = A._randaug_space(31, S)[op]
        for mi in MAGNITUDES if mags.ndim else (0,):
            m = float(mags[mi].item()) if mags.ndim else 0.0
            lists += [[(op, m)], [(op, -m)]] if signed else [[(op, m)]]
    g = torch.Generator().manual_seed(seed)
    for _ in range(12):
        k = int(torch.randint(1, 5, (1,), generator=g))
        lists.append(A.rand_augment_params(S, k, int(torch.randint(0, 31, (1,), generator=g)), 31))
    return lists


def _descs(lists, S):
    from videotransformer_pytorch_b200 import _lib
    from videotransformer_pytorch_b200 import augment as A
    d = (_lib.RandAugDesc * len(lists))()
    for k, ops in enumerate(lists):
        A._pack_randaug(d[k], ops, S)
    return d


@pytest.mark.parametrize('S', SIZES)
def test_kernel_is_the_twin_bit_for_bit(S):
    from videotransformer_pytorch_b200 import _lib
    lists = _op_lists(S, S)
    x = torch.stack([content(CONTENTS[k % len(CONTENTS)], S, seed=k) for k in range(len(lists))])
    descs = _descs(lists, S)
    err = torch.zeros(1, dtype=torch.int32, device=dev)
    y = _lib.K.rand_augment_u8(x.to(dev), _dev_bytes(bytes(descs)), err).cpu()
    assert int(err) == 0
    for k in range(len(lists)):
        assert torch.equal(y[k], randaug_frames(x[k], desc_ops(descs[k]))), (S, lists[k])


@pytest.mark.parametrize('S', (224, 32, 17))
def test_kernel_against_torchvision(S):
    AA = pytest.importorskip('torchvision.transforms.autoaugment')
    from torchvision.transforms import InterpolationMode
    from videotransformer_pytorch_b200 import _lib
    from videotransformer_pytorch_b200 import augment as A
    lists = _op_lists(S, 100 + S)
    x = torch.stack([content(CONTENTS[k % len(CONTENTS)], S, seed=k) for k in range(len(lists))])
    descs = _descs(lists, S)
    y = _lib.K.rand_augment_u8(x.to(dev), _dev_bytes(bytes(descs))).cpu()
    exempt = 0
    for k, ops in enumerate(lists):
        ref = x[k].permute(0, 3, 1, 2)
        for op, m in ops:
            ref = AA._apply_op(ref, A.RANDAUG_OPS[op], m, InterpolationMode.NEAREST, None)
        diff = (y[k] != ref.permute(0, 2, 3, 1)).any(dim=-1)
        if diff.any():                       # only behind a warp with pixels near a tie
            assert any(op in GEOMETRIC and near_tie_mask(A.randaug_theta(op, m, S), S)[0].any() for op, m in ops), ops
            exempt += int(diff.sum())
    print(f'S={S}: {exempt} pixels differ from torchvision, each behind a near-tie warp')


@pytest.mark.parametrize('objective', OBJECTIVES)
def test_pipelines_against_goldens_and_twin(objective):
    from videotransformer_pytorch_b200 import _lib
    from videotransformer_pytorch_b200 import augment as A
    from tests.test_augment_host import _golden_clips
    clips = _golden_clips()
    z, keys = _golden(objective)
    for key in keys:
        S, ids = int(z[f'{key}/S']), [int(i) for i in z[f'{key}/clips']]
        kw = dict(scale=(0.5, 1.0), objective='mim') if objective == 'mim' else {}
        mk = lambda d: A.create_video_transform(S, is_training=True, auto_augment='rand_aug', interpolation='bicubic',
                                                device=d, **kw)
        seed = int(key.split('/')[1])
        torch.manual_seed(seed)
        tf = mk(None)
        out = tf([torch.from_numpy(clips[i]).permute(0, 2, 3, 1).to(dev) for i in ids]).cpu()
        assert int(tf.err) == 0
        old = _lib.K
        _lib.K = EmuKernels(exact=True, inference_forms=True)
        try:
            torch.manual_seed(seed)
            twin_tf = mk('cpu')
            twin = twin_tf([torch.from_numpy(clips[i]).permute(0, 2, 3, 1) for i in ids])
        finally:
            _lib.K = old
        assert torch.equal(out, twin), key
        for b in range(len(ids)):
            p = z[f'{key}/params{b}']
            assert tf.params[b][0]['ra'] == _golden_ops(p)
            ref = torch.from_numpy(z[f'{key}/y{b}']).permute(0, 2, 3, 1)
            pre = torch.from_numpy(z[f'{key}/pre{b}']).permute(0, 2, 3, 1)
            v = tf.params[b][0]
            mine_pre = resize_window(clips[ids[b]].transpose(0, 2, 3, 1), v['crop'], (S, S), (0, 0), S, 0, v['flip'])
            if torch.equal(mine_pre, pre):    # the reference's crop: its output too, near-tie warps aside
                _check_against_golden(out[b], ref, [slot(op, m, S) for op, m in v['ra']], S)


def test_guard_bytes_and_bad_descriptors():
    from videotransformer_pytorch_b200 import _lib
    G, S, T, n = 4096, 224, 2, 3
    buf = torch.full((n * T * S * S * 3 + 2 * G,), 0xA5, dtype=torch.uint8, device=dev)
    y = buf[G:G + n * T * S * S * 3].view(n, T, S, S, 3)
    y.copy_(torch.randint(0, 256, (n, T, S, S, 3), dtype=torch.uint8, device=dev))
    lists = [[(5, 9.0), (13, 0.0)], [(9, -0.27), (1, 0.3), (3, 30.45), (12, 0.0)], [(11, 178.5), (2, -0.09)]]
    err = torch.zeros(1, dtype=torch.int32, device=dev)
    _lib.K.rand_augment_u8(y, _dev_bytes(bytes(_descs(lists, S))), err)
    torch.cuda.synchronize()
    assert int(err) == 0
    assert bool((buf[:G] == 0xA5).all()) and bool((buf[-G:] == 0xA5).all())
    bad = _descs([[(5, 9.0)], [(5, 9.0)], [(7, 0.5)]], S)
    bad[0].op[0] = 14
    bad[1].n_ops = 5
    x = torch.randint(0, 256, (n, T, S, S, 3), dtype=torch.uint8, device=dev)
    y2 = x.clone()
    _lib.K.rand_augment_u8(y2, _dev_bytes(bytes(bad)), err)
    assert int(err) == 1 and int(y2[:2].max()) == 0
    assert torch.equal(y2[2].cpu(), randaug_frames(x[2].cpu(), desc_ops(bad[2])))


def test_graph_replay_with_other_clips_sizes_and_draws():
    from videotransformer_pytorch_b200 import augment as A
    tf = A.create_video_transform(224, is_training=True, auto_augment='rand_aug', interpolation='bicubic')
    ref_tf = A.create_video_transform(224, is_training=True, auto_augment='rand_aug', interpolation='bicubic')
    g = torch.Generator().manual_seed(3)

    def batch(sizes):
        return [torch.randint(0, 256, (4, h, w, 3), dtype=torch.uint8, generator=g) for h, w in sizes]
    tf.reserve(4 * 4 * 320 * 454 * 3, 4)
    torch.manual_seed(0)
    tf.prepare(A.pack_clips(batch([(256, 340)] * 4), pin=True))
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
        assert [v[0]['ra'] for v in tf.params] == [v[0]['ra'] for v in ref_tf.params]
    assert int(tf.err) == 0


def test_models_and_hog_fed_the_transformed_clip():
    """the MaskFeat HOG targets and TimeSformer-B's forward from the device clip equal the same fed the twin's clip"""
    from videotransformer_pytorch_b200 import _lib, hog
    from videotransformer_pytorch_b200 import augment as A
    from videotransformer_pytorch_b200 import TimeSformer
    g = torch.Generator().manual_seed(4)
    clips = [torch.randint(0, 256, (8, h, w, 3), dtype=torch.uint8, generator=g) for h, w in ((256, 340), (320, 427))]
    for objective in OBJECTIVES:
        kw = dict(scale=(0.5, 1.0), objective='mim') if objective == 'mim' else {}
        mk = lambda d: A.create_video_transform(224, is_training=True, auto_augment='rand_aug', interpolation='bicubic',
                                                device=d, **kw)
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
        if objective == 'supervised':
            torch.manual_seed(0)
            m = TimeSformer(num_frames=8, img_size=224).to(dev).eval()
            m.set_input_normalization((0.45,) * 3, (0.225,) * 3)
            with torch.no_grad():
                a, b = m(x), m(host.to(dev))
            assert torch.equal(a, b)
        else:
            markers = [[[0, 2], [2, 1]], [[1, 3]]]
            assert torch.equal(hog.hog_targets_batch(x, markers), hog.hog_targets_batch(host.to(dev), markers))
