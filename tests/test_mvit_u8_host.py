"""MaskFeat's uint8 input path without a GPU: the CPU twin of vt_im2col3d_u8_bf16 (EmuKernels.im2col3d_u8) against the
reference's float pipeline, a loop-for-loop walk-through of the kernel's CTA -> staged window -> 16-byte store
mapping, and MaskFeat on the CPU emulation fed uint8 clips."""
import numpy as np
import pytest
import torch

from tests.emu_kernels import EmuKernels

REF_NORM = ((0.45, 0.45, 0.45), (0.225, 0.225, 0.225))                 # data_trainer.py defaults
IMAGENET_NORM = ((0.485, 0.456, 0.406), (0.229, 0.224, 0.225))


def reference_float_clip(u8, mean, std):
    """The reference's ToTensor + Normalize on the CPU (data_transform.py:62-64, :534-539): pic.float().div(255), then
    torchvision's in-place sub_(mean).div_(std) with fp32 mean / std, on [B, T, C, H, W]."""
    x = u8.permute(0, 1, 4, 2, 3).float().div(255)
    m = torch.as_tensor(mean, dtype=torch.float32).view(1, 1, -1, 1, 1)
    s = torch.as_tensor(std, dtype=torch.float32).view(1, 1, -1, 1, 1)
    return x.sub_(m).div_(s).contiguous()


@pytest.mark.parametrize('norm', [REF_NORM, IMAGENET_NORM], ids=['reference', 'imagenet'])
def test_twin_is_the_reference_float_clip_for_every_byte(norm):
    """A 1x1x1 conv makes cols the normalised clip itself: the twin equals the reference's fp32 clip bit for bit for all
    256 byte values in every channel, and so does the kernel's arithmetic restated in numpy fp32."""
    mean, std = norm
    u = torch.arange(256, dtype=torch.uint8)
    u8 = torch.stack([u, u.flip(0), u.roll(97)], dim=-1).view(1, 1, 16, 16, 3)
    em = EmuKernels(exact=True)
    cols, out = em.im2col3d_u8(u8, torch.tensor(mean), torch.tensor(std), None, (1, 1, 1), (1, 1, 1), (0, 0, 0), 8)
    assert out == (1, 16, 16) and cols.dtype == torch.float32
    ref = reference_float_clip(u8, mean, std).permute(0, 1, 3, 4, 2).reshape(256, 3)
    assert torch.equal(cols[:, :3], ref)
    assert torch.equal(cols[:, 3:], torch.zeros(256, 5))
    f = np.float32
    kern = (u8.numpy().reshape(256, 3).astype(f) / f(255) - np.array(mean, f)) / np.array(std, f)
    assert np.array_equal(kern, ref.numpy())


# ---- CPU walk-through of im2col3d_u8_kernel ---------------------------------------------------------------
SMEM_DEFAULT, SMEM_MAX = 48 * 1024, 200 * 1024


def _rows_per_cta(C, kt, kh, sh, Wp, Kpad):
    """The launcher's choice (vt_im2col3d_u8_bf16): most rows in {4, 2, 1} whose window fits 48 KB."""
    smem = lambda ohb: Kpad * 4 + C * kt * ((ohb - 1) * sh + kh) * Wp * 2
    ohb = 4
    while ohb > 1 and smem(ohb) > SMEM_DEFAULT:
        ohb //= 2
    assert smem(ohb) <= SMEM_MAX
    return ohb


def walk_kernel(u8, mean, std, plan, kernel, stride, padding, kpad, threads=256):
    """im2col3d_u8_kernel restated loop for loop: blockIdx -> (b, ot, row block); the window and the offset table filled
    by a thread-strided loop; cols written in 16-byte chunks.  Returns (cols as bf16, times each element was written)."""
    B, T, H, W, C = u8.shape
    (kt, kh, kw), (st, sh, sw), (pt, ph, pw) = kernel, stride, padding
    To, Ho, Wo = ((n + 2 * p - k) // s + 1 for n, p, k, s in zip((T, H, W), padding, kernel, stride))
    Kreal = C * kt * kh * kw
    Wp = W + 2 * pw
    ohb = _rows_per_cta(C, kt, kh, sh, Wp, kpad)
    R = (ohb - 1) * sh + kh
    f = np.float32
    xs = u8.numpy()
    mode, lam, yl, yh, xl, xh = (0, f(1), 0, 0, 0, 0) if plan is None else (
        int(plan[0]), f(plan[1]), int(plan[2]), int(plan[3]), int(plan[4]), int(plan[5]))
    lam_o = f(f(1) - lam)
    norm = lambda v, c: (f(v) / f(255) - f(mean[c])) / f(std[c])
    cols = np.full((B * To * Ho * Wo, kpad), np.nan, dtype=f)
    hits = np.zeros(cols.shape, dtype=np.int32)
    hblocks = (Ho + ohb - 1) // ohb
    for blk in range(B * To * hblocks):
        hb, ot, b = blk % hblocks, (blk // hblocks) % To, blk // (hblocks * To)
        oh0 = hb * ohb
        noh = min(ohb, Ho - oh0)
        tab = np.empty(kpad, dtype=np.int64)
        for tid in range(threads):
            for k in range(tid, kpad, threads):
                off = -1
                if k < Kreal:
                    dw, dh, dt, c = k % kw, (k // kw) % kh, (k // (kw * kh)) % kt, k // (kw * kh * kt)
                    off = ((c * kt + dt) * R + dh) * Wp + dw
                tab[k] = off
        win = np.empty(C * kt * R * Wp, dtype=f)
        for tid in range(threads):
            for e in range(tid, win.size, threads):
                xw, line = e % Wp, e // Wp
                r, dt, c = line % R, (line // R) % kt, line // (R * kt)
                ti, hi, wi = ot * st - pt + dt, oh0 * sh - ph + r, xw - pw
                v = f(0)
                if 0 <= ti < T and 0 <= hi < H and 0 <= wi < W:
                    v = norm(xs[b, ti, hi, wi, c], c)
                    o = norm(xs[B - 1 - b, ti, hi, wi, c], c)
                    if mode == 1:
                        v = f(v * lam) + f(o * lam_o)
                    elif mode == 2 and yl <= hi < yh and xl <= wi < xh:
                        v = o
                win[e] = v
        win = torch.from_numpy(win).to(torch.bfloat16).float().numpy()      # __float2bfloat16_rn
        cpr = kpad // 8
        row0 = ((b * To + ot) * Ho + oh0) * Wo
        for tid in range(threads):
            for q in range(tid, noh * Wo * cpr, threads):
                rl, k0 = q // cpr, (q % cpr) * 8
                ohl, ow = rl // Wo, rl % Wo
                base = ohl * sh * Wp + ow * sw
                for j in range(8):
                    off = tab[k0 + j]
                    cols[row0 + rl, k0 + j] = win[base + off] if off >= 0 else 0.0
                    hits[row0 + rl, k0 + j] += 1
    return torch.from_numpy(cols), hits


def _plan(mode, lam, box):
    return torch.tensor([mode, lam, *box], dtype=torch.float32)


WALK_CASES = [
    # (B, T, H, W, C), kernel, stride, padding, kpad
    ((2, 4, 12, 12, 3), (3, 7, 7), (2, 4, 4), (1, 3, 3), 448),        # MaskFeat's filter
    ((2, 3, 9, 13, 3), (3, 3, 3), (1, 2, 2), (1, 1, 1), 88),          # odd sides, H != W
    ((4, 5, 7, 5, 2), (2, 3, 3), (2, 1, 2), (0, 1, 0), 24),           # no temporal padding, stride 1 rows
    ((2, 2, 6, 10, 3), (1, 5, 3), (1, 3, 1), (0, 2, 1), 64),          # wide pad columns (45 real of 64)
]
WALK_PLANS = [None, (0, 1.0, (0, 0, 0, 0)), (1, 0.3137, (0, 0, 0, 0)), (2, 0.6, (0, 4, 3, 100)), (2, 0.0, (2, 2, 0, 5))]


@pytest.mark.parametrize('case', range(len(WALK_CASES)))
@pytest.mark.parametrize('plan', range(len(WALK_PLANS)), ids=['noplan', 'mode0', 'mixup', 'cutmix_edge', 'cutmix_empty'])
def test_kernel_walk_covers_cols_once_and_matches_twin(case, plan):
    shape, kernel, stride, padding, kpad = WALK_CASES[case]
    u8 = torch.randint(0, 256, shape, dtype=torch.uint8, generator=torch.Generator().manual_seed(case))
    mean, std = IMAGENET_NORM if shape[-1] == 3 else ((0.4, 0.6), (0.2, 0.3))
    pl = None if WALK_PLANS[plan] is None else _plan(*WALK_PLANS[plan])
    cols, hits = walk_kernel(u8, mean, std, pl, kernel, stride, padding, kpad)
    assert (hits == 1).all()
    twin, _ = EmuKernels(exact=False).im2col3d_u8(u8, torch.tensor(mean), torch.tensor(std), pl, kernel, stride, padding, kpad)
    assert torch.equal(cols, twin.float())


def test_rows_per_cta_at_maskfeat_sizes():
    """At 224 the window of two output rows (3 x 3 x 11 lines of 230) and the table fit 48 KB; at 32 four rows do."""
    assert _rows_per_cta(3, 3, 7, 4, 230, 448) == 2
    assert _rows_per_cta(3, 3, 7, 4, 38, 448) == 4


# ---- MaskFeat on the CPU emulation ------------------------------------------------------------------------
def build(g):
    from videotransformer_pytorch_b200 import MaskFeat
    kw = dict(g.kwargs)
    for k in ('pool_q_stride_size', 'embed_dim_mul', 'atten_head_mul'):
        if k in kw:
            kw[k] = [list(r) for r in kw[k]]
    m = MaskFeat(**kw)
    m.load_state_dict(g.state(torch.float32), strict=True)
    return m


def _clip(g, B, seed):
    c = g.cfg
    return torch.randint(0, 256, (B, c['num_frames'], c['img_size'], c['img_size'], 3), dtype=torch.uint8,
                         generator=torch.Generator().manual_seed(seed))


@pytest.mark.parametrize('norm', [None, IMAGENET_NORM], ids=['default', 'imagenet'])
def test_maskfeat_uint8_equals_reference_normalised_clip(maskfeat_golden, emu, norm):
    g = maskfeat_golden('maskfeat_s32')
    m = build(g).train()
    if norm is not None:
        m.set_input_normalization(*norm)
    mean, std = norm or REF_NORM
    assert m.input_normalization() == (tuple(mean), tuple(std))
    u8 = _clip(g, g.B, 3)
    xf = reference_float_clip(u8, mean, std)
    with torch.no_grad():
        assert torch.equal(m.forward_features(u8, g.mask), m.forward_features(xf, g.mask))
    pred8, loss8 = m(u8, g.target.double(), g.mask, g.cube_marker)
    loss8.backward()
    grads8 = {n: p.grad.clone() for n, p in m.named_parameters()}
    m.zero_grad(set_to_none=True)
    predf, lossf = m(xf, g.target.double(), g.mask, g.cube_marker)
    lossf.backward()
    assert torch.equal(pred8, predf) and torch.equal(loss8, lossf)
    for n, p in m.named_parameters():
        assert torch.equal(grads8[n], p.grad), n


@pytest.mark.parametrize('seed', [0, 1, 2, 5])
def test_maskfeat_mixed_uint8_equals_float_mixup(maskfeat_golden, emu, seed):
    """Mixup on the uint8 batch (a MixedClip) against the package's float Mixup on the reference-normalised clip, same
    numpy seed: CutMix copies are exact; the Mixup blend differs from the reference's by how 1 - lam is rounded (fp64
    scalar vs fp32), at most an ulp per element."""
    from videotransformer_pytorch_b200 import MixedClip, Mixup
    g = maskfeat_golden('maskfeat_s32')
    m = build(g).eval()
    u8 = _clip(g, 2, 10 + seed)
    target = torch.tensor([1, 3])
    mix = Mixup(num_classes=5)
    np.random.seed(seed)
    mixed, y8 = mix(u8, target)
    np.random.seed(seed)
    xf, yf = mix(reference_float_clip(u8, *REF_NORM), target)
    assert isinstance(mixed, MixedClip) and torch.equal(y8, yf)
    with torch.no_grad():
        f8, ff = m.forward_features(mixed)[:, 0], m.forward_features(xf)[:, 0]
    if mixed.mode == 2:
        assert torch.equal(f8, ff)
    else:
        assert float((f8 - ff).norm() / ff.norm()) < 1e-5


def test_maskfeat_rejects_bad_uint8_inputs(maskfeat_golden, emu):
    from videotransformer_pytorch_b200 import MixedClip
    g = maskfeat_golden('maskfeat_s32')
    m = build(g)
    u8 = _clip(g, 2, 0)
    with pytest.raises(RuntimeError, match='uint8 clip'):
        m.forward_features(u8.permute(0, 1, 4, 2, 3).contiguous())          # channels first
    with pytest.raises(RuntimeError, match='uint8 clip'):
        m.forward_features(u8[:, :-2])                                     # wrong frame count
    with pytest.raises(RuntimeError, match='MixedClip must wrap a uint8 clip'):
        m.forward_features(MixedClip(reference_float_clip(u8, *REF_NORM), 1, 0.5, (0, 0, 0, 0)))
