"""Clip transforms on the GPU, from decode-resolution uint8 frames to the [B, T, S, S, 3] uint8 clip the models, Mixup and
hog.hog_targets_batch accept.

The reference builds its transforms with torchvision (data_transform.py:495-615, data_trainer.py:60-121) and runs them in
the DataLoader workers on each uint8 T C H W clip.  Here the workers only decode (collate_uint8 packs a batch of clips of
any sizes into one flat buffer) and the per-pixel work runs in two kernels (csrc/vt_augment.cu):

  train       RandomResizedCrop(S, scale, ratio) -> RandomHorizontalFlip(hflip) -> ColorJitter(cj, cj, cj)
              or, with auto_augment, -> RandAugment() instead of ColorJitter (supervised and mim)
  train mim   RandomResizedCrop(S, scale=(0.5, 1)) -> RandomHorizontalFlip, no jitter
  val         Resize(floor(S / crop_pct)) (short side) -> CenterCrop(S)
  test        Resize(256) (short side, bilinear) -> ThreeCrop(S): views left, right, centre, clip-major

ToTensor + Normalize are not applied to the bytes: hand `mean` / `std` to the model with set_input_normalization, whose
patch-operand kernel applies them.

The random parameters are drawn on the host from torch's default CPU generator with the calls torchvision 0.26 makes, in
the order Compose applies the transforms, once per clip (all frames of a clip share them): RandomResizedCrop.get_params,
then torch.rand(1) < hflip, then ColorJitter.get_params (torch.randperm(4) and one uniform_ per factor; hue is never drawn)
or RandAugment's draws (per op torch.randint(14), then torch.randint(2) for the sign of a signed op).  Under the same
seed the crops, flips, jitter factors and RandAugment ops are the reference's.  The resize matches torchvision's uint8
output up to the last bits of its fp32 pre-rounding value (a byte can differ by 1 where that value lies within
1.75e-4 per filter tap, 2.8e-3 at 256x340 -> 224^2, of a half-integer); the jitter is bit for bit torchvision's on the
same input, and so is RandAugment except where a warped pixel's source coordinate lies within about 2e-4 of a
half-integer (see rand_augment_params).

The kernels read only two fixed device arenas (source bytes and descriptors), each refilled by one copy in `prepare`, and
their launch configuration depends only on (clips, T, S).  So `run` can be captured in a CUDA graph (graph.GraphedTrainStep,
graph.GraphedForward) and replayed with other clips, sizes and draws:

    tf = create_video_transform(224, is_training=True, interpolation='bicubic')
    tf.prepare(first_batch)                                    # sizes the arenas
    step = GraphedTrainStep(lambda y: loss_fn(model(tf.run()), y), [labels])
    for clips, labels in loader:
        tf.prepare(clips)                                      # draws + one H2D copy of sources, one of descriptors
        step(labels)
"""
from __future__ import annotations

import ctypes as C
import math
from typing import NamedTuple, Optional, Sequence, Union

import numpy as np
import torch

from . import _lib

IMAGENET_DEFAULT_MEAN, IMAGENET_DEFAULT_STD = (0.485, 0.456, 0.406), (0.229, 0.224, 0.225)
DEFAULT_CROP_PCT = 0.875
FILTERS = {'bicubic': 0, 'bilinear': 1}
MAX_TAPS = 32                     # VT_CROP_MAX_TAPS
BRIGHTNESS, CONTRAST, SATURATION = 0, 1, 2
MAX_JITTER_SIDE = 256             # vt_color_jitter_u8: the frame in shared memory, its grayscale sum exact in fp32
RANDAUG_OPS = ('Identity', 'ShearX', 'ShearY', 'TranslateX', 'TranslateY', 'Rotate', 'Brightness', 'Color', 'Contrast',
               'Sharpness', 'Posterize', 'Solarize', 'AutoContrast', 'Equalize')      # torchvision's order = kernel op code
RANDAUG_DEFAULTS = (2, 9, 31)     # RandAugment(): num_ops, magnitude, num_magnitude_bins
MAX_RANDAUG_SIDE = 256            # vt_rand_augment_u8: the frame in shared memory


# ---- parameter draws: torchvision 0.26's get_params, same torch calls in the same order --------------------------------
def random_resized_crop_params(height: int, width: int, scale, ratio):
    """RandomResizedCrop.get_params -> (i, j, h, w)"""
    area = height * width
    log_ratio = torch.log(torch.tensor(ratio))
    for _ in range(10):
        target_area = area * torch.empty(1).uniform_(scale[0], scale[1]).item()
        aspect_ratio = torch.exp(torch.empty(1).uniform_(log_ratio[0], log_ratio[1])).item()
        w = int(round(math.sqrt(target_area * aspect_ratio)))
        h = int(round(math.sqrt(target_area / aspect_ratio)))
        if 0 < w <= width and 0 < h <= height:
            i = torch.randint(0, height - h + 1, size=(1,)).item()
            j = torch.randint(0, width - w + 1, size=(1,)).item()
            return i, j, h, w
    in_ratio = float(width) / float(height)          # fallback: central crop
    if in_ratio < min(ratio):
        w = width
        h = int(round(w / min(ratio)))
    elif in_ratio > max(ratio):
        h = height
        w = int(round(h * max(ratio)))
    else:
        w, h = width, height
    return (height - h) // 2, (width - w) // 2, h, w


def color_jitter_params(brightness, contrast, saturation):
    """ColorJitter.get_params without hue -> [(op, factor), ...] in application order (ops with a None range skipped)"""
    fn_idx = torch.randperm(4)
    f = {}
    for op, rng in ((BRIGHTNESS, brightness), (CONTRAST, contrast), (SATURATION, saturation)):
        f[op] = None if rng is None else float(torch.empty(1).uniform_(rng[0], rng[1]))
    return [(int(i), f[int(i)]) for i in fn_idx.tolist() if int(i) in f and f[int(i)] is not None]


def _randaug_space(num_bins: int, S: int):
    """RandAugment._augmentation_space(num_bins, (S, S)) as a list in op order: (magnitudes, signed)"""
    return [(torch.tensor(0.0), False),
            (torch.linspace(0.0, 0.3, num_bins), True),
            (torch.linspace(0.0, 0.3, num_bins), True),
            (torch.linspace(0.0, 150.0 / 331.0 * S, num_bins), True),
            (torch.linspace(0.0, 150.0 / 331.0 * S, num_bins), True),
            (torch.linspace(0.0, 30.0, num_bins), True),
            (torch.linspace(0.0, 0.9, num_bins), True),
            (torch.linspace(0.0, 0.9, num_bins), True),
            (torch.linspace(0.0, 0.9, num_bins), True),
            (torch.linspace(0.0, 0.9, num_bins), True),
            (8 - (torch.arange(num_bins) / ((num_bins - 1) / 4)).round().int(), False),
            (torch.linspace(255.0, 0.0, num_bins), False),
            (torch.tensor(0.0), False),
            (torch.tensor(0.0), False)]


def rand_augment_params(S: int, num_ops: int = 2, magnitude: int = 9, num_magnitude_bins: int = 31):
    """RandAugment.forward's draws on an S x S image -> [(op, signed magnitude), ...] with op the index in RANDAUG_OPS
    and the magnitude torchvision hands to _apply_op: per op torch.randint(14), then torch.randint(2) for the sign of a
    signed op (not drawn for the others)."""
    space = _randaug_space(num_magnitude_bins, S)
    out = []
    for _ in range(num_ops):
        op = int(torch.randint(len(space), (1,)).item())
        mags, signed = space[op]
        m = float(mags[magnitude].item()) if mags.ndim > 0 else 0.0
        if signed and torch.randint(2, (1,)):
            m *= -1.0
        out.append((op, m))
    return out


def _inverse_affine(center, angle, translate, shear):
    """torchvision's _get_inverse_affine_matrix at scale 1 (the same double operations in the same order)"""
    rot, sx, sy = math.radians(angle), math.radians(shear[0]), math.radians(shear[1])
    (cx, cy), (tx, ty) = center, translate
    a = math.cos(rot - sy) / math.cos(sy)
    b = -math.cos(rot - sy) * math.tan(sx) / math.cos(sy) - math.sin(rot)
    c = math.sin(rot - sy) / math.cos(sy)
    d = -math.sin(rot - sy) * math.tan(sx) / math.cos(sy) + math.cos(rot)
    m = [d, -b, 0.0, -c, a, 0.0]
    m[2] += m[0] * (-cx - tx) + m[1] * (-cy - ty)
    m[5] += m[3] * (-cx - tx) + m[4] * (-cy - ty)
    m[2] += cx
    m[5] += cy
    return m


def randaug_theta(op: int, m: float, S: int):
    """The grid matrix of a warp op as _gen_affine_grid uses it: the inverse affine matrix F.affine / F.rotate build
    (shears about the top-left corner, translations by int(m), rotation by -m), rounded to fp32, divided in fp32 by S / 2."""
    corner = [-S * 0.5, -S * 0.5]                     # center=[0, 0] in F.affine's centred coordinates
    if op in (1, 2):
        sh = math.degrees(math.atan(m))
        mat = _inverse_affine(corner, 0.0, [0.0, 0.0], [sh, 0.0] if op == 1 else [0.0, sh])
    elif op in (3, 4):
        t = [1.0 * int(m), 0.0] if op == 3 else [0.0, 1.0 * int(m)]
        mat = _inverse_affine([0.0, 0.0], 0.0, t, [0.0, 0.0])
    else:
        mat = _inverse_affine([0.0, 0.0], -m, [0.0, 0.0], [0.0, 0.0])
    return np.float32(mat) / np.float32(0.5 * S)


def _jitter_range(value):
    """ColorJitter._check_input for brightness / contrast / saturation: v -> (max(0, 1 - v), 1 + v); 0 -> None"""
    if value is None:
        return None
    if isinstance(value, (tuple, list)):
        lo, hi = float(value[0]), float(value[1])
    else:
        lo, hi = max(0.0, 1.0 - float(value)), 1.0 + float(value)
    return None if lo == hi == 1.0 else (lo, hi)


def resize_short_side(height: int, width: int, size: int):
    """torchvision Resize(size) output (h, w): the short side becomes size, the long side int(size * long / short)"""
    short, long = (width, height) if width <= height else (height, width)
    new_short, new_long = size, int(size * long / short)
    return (new_long, new_short) if width <= height else (new_short, new_long)


def max_taps(n_in: int, n_out: int, filter_id: int) -> int:
    """Taps per output of the antialiased filter along an axis of n_in cells resized to n_out (fp32, like the kernel)"""
    scale = np.float32(n_in) / np.float32(n_out)
    half = np.float32(2.0 if filter_id == FILTERS['bicubic'] else 1.0)
    support = half * scale if scale >= 1 else half
    return 2 * int(math.ceil(support)) + 1


# ---- batches of decode-resolution clips -----------------------------------------------------------------------------
class PackedClips(NamedTuple):
    """A batch of uint8 clips packed back to back: data is flat uint8, sizes int64 [B, 4] = (T, H, W, byte offset) with
    clip b at data[offset:offset + T*H*W*3] as [T, H, W, 3].  DataLoader(pin_memory=True) pins `data`."""
    data: torch.Tensor
    sizes: torch.Tensor


def pack_clips(clips: Sequence[torch.Tensor], pin: bool = False) -> PackedClips:
    """uint8 [T, H, W, 3] clips (or the decoder's T C H W permuted view) -> PackedClips (one flat buffer)"""
    hwc = [_as_thwc(c) for c in clips]
    sizes = torch.zeros((len(hwc), 4), dtype=torch.int64)
    off = 0
    for b, c in enumerate(hwc):
        sizes[b, :3] = torch.tensor(c.shape[:3])
        sizes[b, 3] = off
        off += c.numel()
    data = torch.empty(off, dtype=torch.uint8, pin_memory=pin)
    for b, c in enumerate(hwc):
        o = int(sizes[b, 3])
        data[o:o + c.numel()].view(c.shape).copy_(c)
    return PackedClips(data, sizes)


def _as_thwc(v) -> torch.Tensor:
    v = torch.as_tensor(v)
    if v.dtype != torch.uint8 or v.dim() != 4:
        raise ValueError(f'expected a uint8 clip [T, H, W, 3] or [T, 3, H, W], got {tuple(v.shape)} {v.dtype}')
    if v.shape[-1] != 3 and v.shape[1] == 3:          # the dataset's torch.from_numpy(video).permute(0, 3, 1, 2)
        v = v.permute(0, 2, 3, 1)
    if v.shape[-1] != 3:
        raise ValueError(f'expected 3 channels, got clip shape {tuple(v.shape)}')
    return v


def collate_uint8(batch):
    """collate_fn for the reference's Kinetics dataset built with transform=None: the decode-resolution clips of the
    batch go into one flat uint8 buffer (PackedClips, so the batch costs one host-to-device copy; pinned here in the main
    process, by DataLoader(pin_memory=True) when collated in workers); the other fields are collated as torch's default
    collate does, or left as lists where their shapes differ (cube markers)."""
    from torch.utils.data import default_collate, get_worker_info
    items = [b if isinstance(b, (tuple, list)) else (b,) for b in batch]
    pin = get_worker_info() is None and torch.cuda.is_available()
    out = [pack_clips([it[0] for it in items], pin=pin)]
    for k in range(1, len(items[0])):
        col = [it[k] for it in items]
        try:
            out.append(default_collate(col))
        except (RuntimeError, TypeError):
            out.append(col)
    return tuple(out)


# ---- the device transform -----------------------------------------------------------------------------------------------
class ClipTransform:
    """One of the reference's clip pipelines on the GPU.  __call__(clips) = prepare(clips) then run().

    clips: a list of uint8 clips [T, H, W, 3] (CUDA or CPU; sizes may differ, T may not) or a PackedClips.  Returns uint8
    [B, T, S, S, 3], or [B * 3, T, S, S, 3] clip-major for the three-crop test pipeline (TopKAccuracy(views=3))."""

    def __init__(self, size: int, mode: str, *, scale=(0.08, 1.0), ratio=(3. / 4., 4. / 3.), hflip=0.5, color_jitter=None,
                 interpolation='bilinear', resize_to: Optional[int] = None, mean=IMAGENET_DEFAULT_MEAN,
                 std=IMAGENET_DEFAULT_STD, rand_augment=None, device=None):
        if mode not in ('train', 'center', 'three'):
            raise ValueError(f'unknown mode {mode!r}')
        if interpolation not in FILTERS:
            raise ValueError(f'interpolation {interpolation!r}: the GPU transforms support {sorted(FILTERS)}')
        self.size, self.mode = int(size), mode
        self.scale, self.ratio, self.hflip = tuple(scale), tuple(ratio), float(hflip)
        self.filter = FILTERS[interpolation]
        self.resize_to = resize_to
        self.jitter = None
        if color_jitter is not None:
            cj = (float(color_jitter),) * 3 if not isinstance(color_jitter, (tuple, list)) else tuple(color_jitter)
            if len(cj) not in (3, 4):
                raise ValueError('color_jitter: a scalar or 3 / 4 values')
            if len(cj) == 4 and cj[3]:
                raise NotImplementedError('hue jitter is not implemented on the GPU (the reference never draws it)')
            self.jitter = tuple(_jitter_range(v) for v in cj[:3])
            if all(r is None for r in self.jitter):
                self.jitter = None
        if self.jitter is not None and self.size > MAX_JITTER_SIDE:
            raise ValueError(f'ColorJitter on the GPU needs S <= {MAX_JITTER_SIDE} (got {self.size})')
        self.rand_augment = None
        if rand_augment is not None:
            num_ops, magnitude, bins = (int(v) for v in rand_augment)
            if mode != 'train' or self.jitter is not None:
                raise ValueError('rand_augment is a training transform and replaces color_jitter')
            if not (0 <= num_ops <= _lib.RANDAUG_MAX_OPS and bins >= 2 and 0 <= magnitude < bins):
                raise ValueError(f'rand_augment=(num_ops, magnitude, num_magnitude_bins) needs num_ops <= '
                                 f'{_lib.RANDAUG_MAX_OPS} and 0 <= magnitude < num_magnitude_bins, got {tuple(rand_augment)}')
            if self.size > MAX_RANDAUG_SIDE:
                raise ValueError(f'RandAugment on the GPU needs S <= {MAX_RANDAUG_SIDE} (got {self.size})')
            self.rand_augment = (num_ops, magnitude, bins)
        self.mean, self.std = tuple(mean), tuple(std)
        self.views = 3 if mode == 'three' else 1
        self.device = torch.device(device) if device is not None else None
        self.src = None               # source arena (uint8), desc = descriptor arena: crop table, then the jitter or
                                      # RandAugment table
        self.desc = None
        self.err = None
        self._shape = None            # (outputs, T) of the last prepare
        self._captured = False
        self._staging, self._events, self._slot, self._keep = [], [], 0, [None, None, None]

    # -- host ----------------------------------------------------------------------------------------------------------
    def draw(self, sizes):
        """sizes: [(H, W), ...] per clip -> descriptors, a list per clip of dicts (one per output view) with the crop box,
        resized size, window, flip, filter, jitter ops and RandAugment ops ('ra'), drawn in the reference's order."""
        S, out = self.size, []
        for H, W in sizes:
            if self.mode == 'train':
                i, j, h, w = random_resized_crop_params(H, W, self.scale, self.ratio)
                flip = bool(torch.rand(1) < self.hflip) if self.hflip > 0 else False
                ops = color_jitter_params(*self.jitter) if self.jitter is not None else []
                ra = rand_augment_params(S, *self.rand_augment) if self.rand_augment is not None else []
                out.append([dict(crop=(i, j, h, w), resized=(S, S), window=(0, 0), flip=flip, ops=ops, ra=ra)])
                continue
            RH, RW = resize_short_side(H, W, self.resize_to)
            if S > RH or S > RW:
                raise ValueError(f'crop size {S} is bigger than the resized frame {(RH, RW)}')
            if self.mode == 'center':
                wins = [(int(round((RH - S) / 2.0)), int(round((RW - S) / 2.0)))]
            else:
                y = (RH - S) // 2
                wins = [(y, 0), (y, RW - S), (y, (RW - S) // 2)]
            out.append([dict(crop=(0, 0, H, W), resized=(RH, RW), window=win, flip=False, ops=[]) for win in wins])
        return out

    def _pack(self, views, shapes, offsets):
        n = sum(len(v) for v in views)
        crops, jit = (_lib.CropDesc * n)(), (_lib.JitterDesc * n)()
        ra = (_lib.RandAugDesc * n)() if self.rand_augment is not None else None
        k = 0
        for b, per_clip in enumerate(views):
            T, H, W = shapes[b]
            for v in per_clip:
                (cy, cx, ch, cw), (RH, RW), (oy, ox) = v['crop'], v['resized'], v['window']
                for n_in, n_out in ((ch, RH), (cw, RW)):
                    if max_taps(n_in, n_out, self.filter) > MAX_TAPS:
                        raise ValueError(f'downscale {n_in} -> {n_out} needs more than {MAX_TAPS} filter taps')
                d = crops[k]
                d.src_offset, d.H, d.W, d.pitch = offsets[b], H, W, 3 * W
                d.crop_y, d.crop_x, d.crop_h, d.crop_w = cy, cx, ch, cw
                d.RH, d.RW, d.oy, d.ox = RH, RW, oy, ox
                d.flip, d.filter = int(v['flip']), self.filter
                jd = jit[k]
                jd.n_ops = len(v['ops'])
                for s, (op, f) in enumerate(v['ops']):
                    jd.op[s] = op
                    jd.factor[s] = f                                     # an fp32 value (from a float32 tensor)
                    jd.one_minus[s] = np.float32(1.0 - f)               # torchvision: (1.0 - ratio) in double, fp32 op
                if ra is not None:
                    _pack_randaug(ra[k], v['ra'], self.size)
                k += 1
        return bytes(crops) + (bytes(jit) if ra is None else bytes(ra)), n

    def _stage(self, payload: bytes, nbytes_cap: int, dev):
        cuda = dev.type == 'cuda'
        if not self._staging or self._staging[0].numel() < len(payload):
            self._staging = [torch.empty(max(len(payload), nbytes_cap), dtype=torch.uint8, pin_memory=cuda)
                             for _ in range(3 if cuda else 1)]
            self._events = [torch.cuda.Event() if cuda else None for _ in self._staging]
        slot = self._slot
        self._slot = (slot + 1) % len(self._staging)
        if self._events[slot] is not None:
            self._events[slot].synchronize()       # that buffer's upload (three batches ago) must have finished
        host = self._staging[slot]
        C.memmove(host.data_ptr(), payload, len(payload))
        return host, slot

    def _device(self, hint):
        dev = self.device or hint
        if dev.type == 'cuda' and dev.index is None:
            dev = torch.device('cuda', torch.cuda.current_device())
        return dev

    def _arena(self, name, nbytes, dev):
        buf = getattr(self, name)
        if buf is not None and buf.numel() >= nbytes and buf.device == dev:
            return buf
        if self._captured:
            raise RuntimeError(f'ClipTransform: the batch needs {nbytes} bytes of {name} arena, more than the '
                               f'{0 if buf is None else buf.numel()} a captured graph reads; call reserve() before capture')
        buf = torch.empty(max(nbytes, 0 if buf is None else buf.numel()), dtype=torch.uint8, device=dev)
        setattr(self, name, buf)
        return buf

    def reserve(self, src_bytes: int, clips: int, device=None):
        """Size the arenas for batches of up to `clips` clips and `src_bytes` source bytes (before a graph capture)."""
        dev = self._device(torch.device(device) if device is not None else torch.device('cuda'))
        self._arena('src', src_bytes, dev)
        self._arena('desc', clips * self.views * (C.sizeof(_lib.CropDesc) + C.sizeof(self._second_desc())), dev)

    def _second_desc(self):
        """the descriptor type of the table after the crop table"""
        return _lib.RandAugDesc if self.rand_augment is not None else _lib.JitterDesc

    def prepare(self, clips: Union[PackedClips, Sequence[torch.Tensor]]):
        """Draw this batch's parameters and upload sources and descriptors into the arenas."""
        if isinstance(clips, PackedClips):
            sizes = clips.sizes.tolist()
            shapes = [tuple(s[:3]) for s in sizes]
            offsets = [s[3] for s in sizes]
            total = clips.data.numel()
            dev = self._device(clips.data.device if clips.data.is_cuda else torch.device('cuda'))
        else:
            clips = [_as_thwc(c) for c in clips]
            shapes = [tuple(c.shape[:3]) for c in clips]
            offsets, total = [], 0
            for c in clips:
                offsets.append(total)
                total += c.numel()
            dev = self._device(clips[0].device if clips[0].is_cuda else torch.device('cuda'))
        if not shapes:
            raise ValueError('empty batch')
        if len({s[0] for s in shapes}) != 1:
            raise ValueError(f'clips of one batch must have the same number of frames, got {sorted({s[0] for s in shapes})}')
        views = self.draw([(H, W) for _, H, W in shapes])
        payload, n = self._pack(views, shapes, offsets)
        T = shapes[0][0]
        if self._captured and self._shape != (n, T):
            raise RuntimeError(f'ClipTransform: a captured graph runs {self._shape[0]} outputs of {self._shape[1]} frames, '
                               f'this batch needs {n} of {T}')
        src = self._arena('src', total, dev)
        desc = self._arena('desc', len(payload), dev)
        if self.err is None or self.err.device != dev:
            self.err = torch.zeros(1, dtype=torch.int32, device=dev)
        if isinstance(clips, PackedClips):
            src[:total].copy_(clips.data, non_blocking=True)
        else:
            for c, o in zip(clips, offsets):
                src[o:o + c.numel()].view(c.shape).copy_(c, non_blocking=True)
        host, slot = self._stage(payload, desc.numel(), dev)
        desc[:len(payload)].copy_(host[:len(payload)], non_blocking=True)
        if self._events[slot] is not None:
            self._events[slot].record(torch.cuda.current_stream(dev))
            self._keep[slot] = clips               # a pinned source buffer must outlive its copy
        self._shape = (n, T)
        self.params = views
        return views

    # -- device --------------------------------------------------------------------------------------------------------
    def run(self) -> torch.Tensor:
        """Launch the transform on the arenas (one resize launch, then one jitter or RandAugment launch in training with
        either)."""
        if self._shape is None:
            raise RuntimeError('ClipTransform.run: nothing prepared')
        n, T = self._shape
        S = self.size
        if self.src.is_cuda and torch.cuda.is_current_stream_capturing():
            self._captured = True
        out = torch.empty((n, T, S, S, 3), dtype=torch.uint8, device=self.src.device)
        ncrop = n * C.sizeof(_lib.CropDesc)
        _lib.K.resized_crop_u8(self.src, self.desc[:ncrop], out, self.err)
        if self.jitter is not None:
            _lib.K.color_jitter_u8(out, self.desc[ncrop:ncrop + n * C.sizeof(_lib.JitterDesc)])
        if self.rand_augment is not None:
            _lib.K.rand_augment_u8(out, self.desc[ncrop:ncrop + n * C.sizeof(_lib.RandAugDesc)], self.err)
        return out

    def __call__(self, clips):
        self.prepare(clips)
        return self.run()

    def __repr__(self):
        return (f'{type(self).__name__}(size={self.size}, mode={self.mode!r}, scale={self.scale}, ratio={self.ratio}, '
                f'hflip={self.hflip}, jitter={self.jitter}, rand_augment={self.rand_augment}, filter={self.filter}, '
                f'resize_to={self.resize_to})')


def create_video_transform(input_size=224, is_training=False, scale=None, ratio=None, hflip=0.5, color_jitter=0.4,
                           auto_augment=None, interpolation='bilinear', mean=IMAGENET_DEFAULT_MEAN,
                           std=IMAGENET_DEFAULT_STD, objective='supervised', crop_pct=None, device=None) -> ClipTransform:
    """data_transform.create_video_transform with the same arguments and defaults, on the GPU.  The `mim` objective
    returns one transform (the reference returns [crop + flip, ToTensor + Normalize]; here Normalize is the model's, via
    set_input_normalization(tf.mean, tf.std)), and the HOG targets are computed from its output.

    A truthy auto_augment selects torchvision's RandAugment() with its defaults in place of ColorJitter, as the
    reference's transforms_train does for every truthy value.  timm policy strings ('rand-m9-mstd0.5-inc1', ...) raise
    NotImplementedError: the reference would silently ignore their magnitude noise and severity fields."""
    img_size = input_size[-1] if isinstance(input_size, (tuple, list)) else input_size
    if isinstance(input_size, (tuple, list)) and input_size[-1] != input_size[-2]:
        raise ValueError('the GPU transforms produce square clips')
    if is_training:
        rand_augment = None
        if auto_augment:
            if isinstance(auto_augment, str) and auto_augment.startswith('rand-'):
                raise NotImplementedError(
                    f'auto_augment={auto_augment!r}: timm RandAugment policy strings are not implemented on the GPU.  The '
                    f'reference builds torchvision\'s RandAugment() for any auto_augment and silently ignores the '
                    f'string\'s magnitude noise and increasing-severity fields; pass auto_augment=\'rand_aug\' (or True) '
                    f'for that transform.')
            rand_augment, color_jitter = RANDAUG_DEFAULTS, None
        return ClipTransform(img_size, 'train', scale=tuple(scale or (0.08, 1.0)), ratio=tuple(ratio or (3. / 4., 4. / 3.)),
                             hflip=hflip, color_jitter=color_jitter, interpolation=interpolation, mean=mean, std=std,
                             rand_augment=rand_augment, device=device)
    crop_pct = crop_pct or DEFAULT_CROP_PCT
    return ClipTransform(img_size, 'center', interpolation=interpolation, resize_to=int(math.floor(img_size / crop_pct)),
                         mean=mean, std=std, device=device)


def _pack_randaug(d, ops, S: int):
    """Fill one RandAugDesc from [(op, signed magnitude), ...] as _apply_op would apply them to an S x S frame."""
    d.n_ops = len(ops)
    for s, (op, m) in enumerate(ops):
        d.op[s] = op
        if 1 <= op <= 5:
            for k, v in enumerate(randaug_theta(op, m, S)):
                d.theta[s][k] = v
        elif 6 <= op <= 9:                            # _blend(img, ., 1.0 + m): fp32 ratio and fp32 (1.0 - ratio)
            d.arg[s] = np.float32(1.0 + m)
            d.one_minus[s] = np.float32(1.0 - (1.0 + m))
        elif op == 10:                                # posterize(img, int(m)): img & -2 ** (8 - bits)
            d.arg[s] = float(-int(2 ** (8 - int(m))) & 0xFF)
        elif op == 11:                                # solarize: an fp32 threshold
            d.arg[s] = m


def ThreeCropTest(short_side=256, size=224, mean=IMAGENET_DEFAULT_MEAN, std=IMAGENET_DEFAULT_STD, device=None):
    """The reference's test transform (data_trainer.py:110-115): Resize(short_side) with torchvision's default bilinear
    filter, then ThreeCrop(size); outputs clip-major [B * 3, T, size, size, 3] (left, right, centre per clip)."""
    return ClipTransform(size, 'three', interpolation='bilinear', resize_to=short_side, mean=mean, std=std, device=device)
