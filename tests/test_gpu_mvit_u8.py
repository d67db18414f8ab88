"""MaskFeat / MViT fed the decoder's uint8 clip: vt_im2col3d_u8_bf16 against its CPU twin and against the float route, the
MaskFeat pre-training step and the supervised MViT Mixup step, forward-only form and graph capture.  -m gpu"""
import random

import numpy as np
import pytest
import torch

from tests.conftest import rel_err
from tests.emu_kernels import EmuKernels
from tests.test_mvit_u8_host import IMAGENET_NORM, REF_NORM, build, reference_float_clip

pytestmark = pytest.mark.gpu
FILTER = ((3, 7, 7), (2, 4, 4), (1, 3, 3))                   # create_conv_patch_embed, video_transformer.py:585-618
KPAD = 448


def K():
    from videotransformer_pytorch_b200 import _lib
    return _lib.K


def _u8(shape, seed):
    return torch.randint(0, 256, shape, dtype=torch.uint8, generator=torch.Generator().manual_seed(seed))


def _kernel_cols(u8, mean, std, plan):
    """vt_im2col3d_u8_bf16 writing into memory that held NaN: the caching allocator hands the freed block back."""
    B, T, H, W, _ = u8.shape
    To, Ho, Wo = ((n + 2 * p - k) // s + 1 for n, p, k, s in zip((T, H, W), FILTER[2], FILTER[0], FILTER[1]))
    x, m, s = u8.cuda(), torch.tensor(mean).cuda(), torch.tensor(std).cuda()
    p = None if plan is None else plan.cuda()
    nan = torch.full((B * To * Ho * Wo, KPAD), float('nan'), dtype=torch.bfloat16, device='cuda')
    ptr = nan.data_ptr()
    del nan
    cols, out = K().im2col3d_u8(x, m, s, p, *FILTER, KPAD)
    assert cols.data_ptr() == ptr and out == (To, Ho, Wo)
    return cols


GEOMS = [(2, 16, 224, 224), (2, 8, 32, 32), (4, 8, 32, 48), (4, 4, 64, 40)]


def _plans(H, W):
    return {'noplan': None, 'mode0': (0, 1.0, (0, 0, 0, 0)), 'mixup': (1, 0.3137, (0, 0, 0, 0)),
            'cutmix_edges': (2, 0.7, (0, 9, W - 7, W)), 'cutmix_full': (2, 0.0, (0, H, 0, W)),
            'cutmix_empty': (2, 1.0, (5, 5, 0, W))}


@pytest.mark.parametrize('geom', GEOMS, ids=lambda g: 'x'.join(map(str, g)))
@pytest.mark.parametrize('plan', list(_plans(1, 1)))
def test_kernel_equals_twin(geom, plan):
    B, T, H, W = geom
    u8 = _u8((B, T, H, W, 3), sum(geom))
    spec = _plans(H, W)[plan]
    pl = None if spec is None else torch.tensor([spec[0], spec[1], *spec[2]], dtype=torch.float32)
    mean, std = IMAGENET_NORM if B == 4 else REF_NORM
    cols = _kernel_cols(u8, mean, std, pl).cpu()
    twin, _ = EmuKernels(exact=False).im2col3d_u8(u8, torch.tensor(mean), torch.tensor(std), pl, *FILTER, KPAD)
    assert not cols.isnan().any()
    assert torch.equal(cols, twin)


def _within_one_bf16_ulp(a, b):
    a, b = a.float(), b.float()
    mag = torch.maximum(a.abs(), b.abs())
    ulp = torch.where(mag > 0, torch.exp2(torch.floor(torch.log2(mag)) - 7), torch.zeros_like(mag))
    return (a - b).abs() <= ulp


@pytest.mark.parametrize('geom', [(2, 16, 224, 224), (4, 8, 32, 32)], ids=['maskfeat', 's32'])
def test_kernel_against_float_route(geom):
    """No plan: bit for bit vt_im2col3d_bf16 of the reference's CPU-normalised clip.  Mixup / CutMix: the package's float
    Mixup (the reference's tensor ops) under the same numpy seed draws the same lam and box, and every element is within one
    bf16 ulp (the reference rounds 1 - lam from fp64, the kernel takes it in fp32)."""
    from videotransformer_pytorch_b200 import Mixup
    B, T, H, W = geom
    u8 = _u8((B, T, H, W, 3), 7)
    xf = reference_float_clip(u8, *REF_NORM).cuda()
    mean, std = (torch.tensor(v).cuda() for v in REF_NORM)
    ref, _ = K().im2col3d(xf, *FILTER, KPAD)
    got, _ = K().im2col3d_u8(u8.cuda(), mean, std, None, *FILTER, KPAD)
    assert torch.equal(got, ref)
    labels = torch.arange(B, device='cuda') % 3
    seen = set()
    for seed in range(12):
        mix = Mixup(num_classes=3)
        np.random.seed(seed)
        mixed, y8 = mix(u8.cuda(), labels)
        np.random.seed(seed)
        xm, yf = mix(xf.clone(), labels)
        np.random.seed(seed)
        assert (mixed.mode, mixed.lam, mixed.box) == mix.draw((H, W))
        assert torch.equal(y8, yf)
        ref, _ = K().im2col3d(xm, *FILTER, KPAD)
        got, _ = K().im2col3d_u8(mixed.clip, mean, std, mixed.plan, *FILTER, KPAD)
        close = _within_one_bf16_ulp(got, ref)
        n_diff = int((got != ref).sum())
        print(f'seed {seed} mode {mixed.mode} lam {mixed.lam:.4f} box {mixed.box}: {n_diff} of {ref.numel()} differ')
        assert bool(close.all())
        if mixed.mode == 2:
            assert n_diff == 0
        seen.add(mixed.mode)
    assert seen == {1, 2}


# ---- MaskFeat pre-training ----------------------------------------------------------------------------------
def _model(maskfeat_golden):
    g = maskfeat_golden('maskfeat_s32')
    return g, build(g).cuda().train()


def _masks(g, B, seed):
    from videotransformer_pytorch_b200.mask_generator import CubeMaskGenerator
    c = g.cfg
    dr = c['downsample_rate']
    gen = CubeMaskGenerator(input_size=(c['thw'][0], c['thw'][1] // dr, c['thw'][2] // dr), min_num_patches=1)
    random.seed(seed)
    masks, markers = zip(*(gen() for _ in range(B)))
    return torch.from_numpy(np.stack(masks)).cuda(), list(markers)


def _grads(m):
    return {n: p.grad.clone() for n, p in m.named_parameters() if p.grad is not None}


def _assert_grads(got, ref, ref2, what):
    """Bit for bit where the float step itself is reproducible; elsewhere (fp32 atomics in the pooling-attention dK/dV)
    within the spread of two float runs."""
    exact = 0
    for n, r in ref.items():
        if torch.equal(r, ref2[n]):
            assert torch.equal(got[n], r), (what, n)
            exact += 1
        else:
            assert rel_err(got[n].cpu(), r.cpu()) < 2e-3, (what, n)
    print(f'{what}: {exact} of {len(ref)} gradients reproducible and bit-identical')


def test_maskfeat_pretrain_step_uint8_equals_float(maskfeat_golden):
    from videotransformer_pytorch_b200 import hog
    g, m = _model(maskfeat_golden)
    B = 2
    u8 = _u8((B, g.cfg['num_frames'], g.cfg['img_size'], g.cfg['img_size'], 3), 21).cuda()
    mask, markers = _masks(g, B, 3)
    target = hog.hog_targets_batch(u8, markers)
    xf = reference_float_clip(u8.cpu(), *REF_NORM).cuda()

    def step(x):
        m.zero_grad(set_to_none=True)
        pred, loss = m(x, target, mask, markers)
        loss.backward()
        return pred.detach(), loss.detach(), _grads(m)

    p8, l8, g8 = step(u8)
    pf, lf, gf = step(xf)
    _, _, gf2 = step(xf)
    assert float(lf) > 0
    assert torch.equal(p8, pf) and torch.equal(l8, lf)
    _assert_grads(g8, gf, gf2, 'pre-training step')


def test_integration_mim_recipe_runs(maskfeat_golden):
    """INTEGRATION.md §4: the `mim` transform's uint8 clip feeds MaskFeat and the HOG targets."""
    from videotransformer_pytorch_b200 import augment, hog
    g, model = _model(maskfeat_golden)
    S = g.cfg['img_size']
    gen = torch.Generator().manual_seed(8)
    clips = [torch.randint(0, 256, (g.cfg['num_frames'], h, w, 3), dtype=torch.uint8, generator=gen)
             for h, w in ((48, 64), (40, 52))]
    mean, std = IMAGENET_NORM
    tf = augment.create_video_transform(input_size=S, is_training=True, scale=(0.5, 1.0), hflip=0.5, color_jitter=None,
                                        interpolation='bicubic', objective='mim', mean=mean, std=std)
    model.set_input_normalization(tf.mean, tf.std)
    mask, cube_marker = _masks(g, 2, 11)
    torch.manual_seed(0)
    x = tf(augment.pack_clips(clips, pin=True))
    assert x.dtype == torch.uint8 and tuple(x.shape) == (2, g.cfg['num_frames'], S, S, 3)
    target = hog.hog_targets_batch(x, cube_marker)
    pred, loss = model(x, target, mask.cuda(), cube_marker)
    loss.backward()
    assert torch.isfinite(loss) and all(p.grad is not None for p in model.parameters())
    _, loss_f = model(reference_float_clip(x.cpu(), mean, std).cuda(), target, mask, cube_marker)
    assert torch.equal(loss.detach(), loss_f.detach())


# ---- supervised MViT with Mixup --------------------------------------------------------------------------------
def test_mvit_mixup_step_against_fp64_oracle(maskfeat_golden):
    """model_trainer.py -arch mvit: Mixup on the batch -> forward_features(x)[:, 0] -> head -> soft-target CE, fed the uint8
    batch, against mvit_oracle in fp64 fed the fp64-mixed clip (tolerances of test_gpu_mvit's MaskFeat gradients)."""
    from oracle import mvit_oracle as MO
    from videotransformer_pytorch_b200 import ClassificationHead, Mixup
    g, m = _model(maskfeat_golden)
    torch.manual_seed(1)
    head = ClassificationHead(5, m.mvit.norm_embed.normalized_shape[0], init_std=0.2).cuda()
    B = 4
    u8 = _u8((B, g.cfg['num_frames'], g.cfg['img_size'], g.cfg['img_size'], 3), 31)
    labels = torch.tensor([0, 3, 1, 4])
    for seed, want in ((0, 1), (2, 2)):
        mix = Mixup(num_classes=5)
        np.random.seed(seed)
        mixed, y = mix(u8.cuda(), labels.cuda())
        assert mixed.mode == want
        m.zero_grad(set_to_none=True)
        head.zero_grad(set_to_none=True)
        logits_g = head(m.forward_features(mixed)[:, 0])
        loss = head.loss(m.forward_features(mixed)[:, 0], y)
        loss.backward()
        # oracle: the reference's float clip in fp64, mixed in fp64 with the same draw
        x = (u8.double() / 255 - torch.tensor(REF_NORM[0], dtype=torch.float64)) / torch.tensor(REF_NORM[1], dtype=torch.float64)
        x = x.permute(0, 1, 4, 2, 3)
        if mixed.mode == 1:
            x = x * mixed.lam + x.flip(0) * (1 - mixed.lam)
        else:
            yl, yh, xl, xh = mixed.box
            x = x.clone()
            x[..., yl:yh, xl:xh] = x.flip(0)[..., yl:yh, xl:xh]
        sd = {n: p.detach().cpu().double().requires_grad_(True) for n, p in m.named_parameters()}
        hw, hb = (head.cls_head.weight.detach().cpu().double().requires_grad_(True),
                  head.cls_head.bias.detach().cpu().double().requires_grad_(True))
        logits = MO.maskfeat_forward_features(sd, x.contiguous(), None, g.cfg)[:, 0] @ hw.t() + hb
        loss_o = (-y.cpu().double() * logits.log_softmax(-1)).sum(-1).mean()
        loss_o.backward()
        assert rel_err(logits_g.detach().cpu(), logits.detach()) < 4e-2          # feature tolerance of test_gpu_mvit
        assert abs(loss.item() - loss_o.item()) < 4e-2 * abs(loss_o.item())
        # mask_token and decoder_pred take no part in forward_features; norm_k.bias is zero in theory
        errs = sorted((rel_err(p.grad.cpu(), sd[n].grad), n) for n, p in m.named_parameters()
                      if sd[n].grad is not None and not n.endswith('attn.norm_k.bias'))
        assert len(errs) > 50
        errs.append((rel_err(head.cls_head.weight.grad.cpu(), hw.grad), 'head.weight'))
        errs.sort()
        median, worst = errs[len(errs) // 2][0], errs[-1]
        print(f'mode {mixed.mode}: loss {loss.item():.6f} vs {loss_o.item():.6f}, grad rel-L2 median {median:.2e} worst {worst}')
        assert median < 5e-2 and worst[0] < 0.3, errs[-5:]


# ---- forward-only form and graph capture -----------------------------------------------------------------------
def test_uint8_forward_only_equals_grad_forward(maskfeat_golden):
    from videotransformer_pytorch_b200 import Mixup
    g, m = _model(maskfeat_golden)
    m.eval()
    u8 = _u8((2, g.cfg['num_frames'], g.cfg['img_size'], g.cfg['img_size'], 3), 41).cuda()
    np.random.seed(0)
    mixed, _ = Mixup(num_classes=3)(u8, torch.tensor([0, 1], device='cuda'))
    for x in (u8, mixed):
        f_grad = m.forward_features(x)
        with torch.no_grad():
            f_ng = m.forward_features(x)
        assert f_grad.requires_grad and torch.equal(f_ng, f_grad.detach())


class _PlanClip:
    """The clip + plan pair a captured step reads (mixup.MixedClip without the host-side draw)."""

    def __new__(cls, clip, plan):
        from videotransformer_pytorch_b200 import MixedClip
        mc = MixedClip.__new__(MixedClip)
        mc.clip, mc.plan = clip, plan
        return mc


class PretrainStep(torch.nn.Module):
    def __init__(self, net):
        super().__init__()
        self.net = net

    def forward(self, x, target, mask, cmask):
        return self.net.forward_with_center_mask(x, target, mask, cmask)[1]


class MixStep(torch.nn.Module):
    def __init__(self, net, head):
        super().__init__()
        self.net, self.head = net, head

    def forward(self, x, plan, y):
        return self.head.loss(self.net.forward_features(_PlanClip(x, plan))[:, 0], y)


def _batches(g, n):
    c = g.cfg
    return [_u8((2, c['num_frames'], c['img_size'], c['img_size'], 3), 50 + i).cuda() for i in range(n)]


def test_graphed_pretrain_step_replays_uint8_batches(maskfeat_golden):
    from videotransformer_pytorch_b200 import hog
    from videotransformer_pytorch_b200.graph import GraphedTrainStep
    g, m = _model(maskfeat_golden)
    batches = _batches(g, 3)

    def inputs(x, seed):
        mask, markers = _masks(g, 2, seed)
        return x, hog.hog_targets_batch(x, markers), mask, m.center_frame_mask(mask, markers)

    step = GraphedTrainStep(PretrainStep(m), inputs(batches[0], 0))     # before any eager backward
    for i, x in enumerate(batches[1:]):
        inp = inputs(x, i + 1)
        loss_g = step(*inp).clone()
        grads_g = _grads(m)
        eager = []
        for _ in range(2):
            m.zero_grad(set_to_none=True)
            loss_e = m.forward_with_center_mask(*inp)[1]
            loss_e.backward()
            eager.append((loss_e.detach(), _grads(m)))
        assert torch.equal(loss_g, eager[0][0]), (i, float(loss_g), float(eager[0][0]))
        _assert_grads(grads_g, eager[0][1], eager[1][1], f'graphed pre-training replay {i}')


def test_graphed_mixup_step_replays_uint8_batches(maskfeat_golden):
    """The Mixup draw reaches the captured step through plan_out: Mixup writes it into the graph's static plan buffer."""
    from videotransformer_pytorch_b200 import ClassificationHead, Mixup
    from videotransformer_pytorch_b200.graph import GraphedTrainStep
    g, m = _model(maskfeat_golden)
    batches = _batches(g, 3)
    torch.manual_seed(2)
    head = ClassificationHead(3, m.mvit.norm_embed.normalized_shape[0], init_std=0.2).cuda()
    mix = Mixup(num_classes=3)
    labels = torch.tensor([0, 2], device='cuda')
    plan = torch.zeros(6, dtype=torch.float32, device='cuda')
    np.random.seed(0)
    _, y0 = mix(batches[0], labels, plan_out=plan)
    mstep = MixStep(m, head)
    used = [p for n, p in mstep.named_parameters() if not n.startswith('net.decoder_pred')]   # not in forward_features
    gstep = GraphedTrainStep(mstep, (batches[0], plan, y0), params=used)                      # before any eager backward
    static_plan = gstep.static_inputs[1]
    modes = set()
    for i, x in enumerate(batches[1:] + batches[:1]):
        np.random.seed(10 + i)
        mixed, y = mix(x, labels, plan_out=static_plan)
        modes.add(mixed.mode)
        loss_g = gstep(x, static_plan, y).clone()
        grads_g = _grads(mstep)
        eager = []
        for _ in range(2):
            mstep.zero_grad(set_to_none=True)
            np.random.seed(10 + i)
            mixed_e, y_e = mix(x, labels)
            loss_e = head.loss(m.forward_features(mixed_e)[:, 0], y_e)
            loss_e.backward()
            eager.append((loss_e.detach(), _grads(mstep)))
        assert torch.equal(loss_g, eager[0][0]), (i, float(loss_g), float(eager[0][0]))
        _assert_grads(grads_g, eager[0][1], eager[1][1], f'graphed Mixup replay {i} (mode {mixed.mode})')
    assert len(modes) >= 2
