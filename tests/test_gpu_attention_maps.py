"""cls-row attention (vt_attn_cls_probs) and show_attn's threshold masks (vt_attn_mass_mask) on the GPU.  -m gpu"""
import ctypes

import numpy as np
import pytest
import torch

from tests.emu_attention_maps import mass_mask_rows
from tests.test_attention_maps_host import check_against_show_attn

pytestmark = pytest.mark.gpu

DEV = 'cuda'


def _ts(kind, T=4, img=32, D=64, heads=2, layers=2):
    from videotransformer_pytorch_b200 import TimeSformer
    torch.manual_seed(0)
    m = TimeSformer(num_frames=T, img_size=img, patch_size=16, embed_dims=D, num_heads=heads, num_transformer_layers=layers,
                    attention_type=kind)
    with torch.no_grad():                   # spread the attention (zero-init temporal_fc / small pos_embed give flat maps)
        for n, p in m.named_parameters():
            if 'temporal_fc' in n or 'qkv' in n:
                p.normal_(std=0.08)
    return m.to(DEV).eval()


def _vivit(kind, T=4, img=32, D=64, heads=2, layers=2):
    from videotransformer_pytorch_b200 import ViViT
    torch.manual_seed(0)
    m = ViViT(num_frames=T, img_size=img, patch_size=16, embed_dims=D, num_heads=heads, num_transformer_layers=layers,
              attention_type=kind)
    with torch.no_grad():
        for n, p in m.named_parameters():
            if 'qkv' in n:
                p.normal_(std=0.08)
    return m.to(DEV).eval()


TS_KINDS = ['divided_space_time', 'space_only', 'joint_space_time']
# (T, img, embed_dims, heads, input side): the tiny, n289 and 8 x 224^2 golden geometries (embed_dims a multiple of 128,
# which the divided blocks' row-mapped LayerNorm needs), the four head widths at 8 x 224^2, and a 320^2 input to a 224^2
# model (interpolated pos_embed)
TS_CONFIGS = [(4, 32, 128, 2, 32), (8, 96, 128, 2, 96), (8, 224, 768, 12, 224), (8, 224, 384, 12, 224),
              (8, 224, 384, 4, 224), (8, 224, 384, 3, 224), (8, 224, 768, 12, 320)]


@pytest.mark.parametrize('cfg', TS_CONFIGS, ids=lambda c: 'T{}_img{}_D{}_h{}_in{}'.format(*c))
@pytest.mark.parametrize('kind', TS_KINDS)
def test_timesformer_cls_attention_is_row_zero(kind, cfg):
    T, img, D, heads, side = cfg
    m = _ts(kind, T, img, D, heads)
    x = torch.randn(2, T, 3, side, side, device=DEV)
    full = m.get_last_selfattention(x)
    row = m.cls_attention(x)
    assert row.shape == full.shape[:3]
    assert torch.equal(row, full[:, :, 0, :])


@pytest.mark.parametrize('kind', ['fact_encoder', 'joint_space_time', 'divided_space_time'])
@pytest.mark.parametrize('D,heads', [(128, 2), (384, 12), (384, 3)])
def test_vivit_cls_attention_is_row_zero(kind, D, heads):
    m = _vivit(kind, T=16, img=64, D=D, heads=heads)
    x = torch.randn(2, 16, 3, 64, 64, device=DEV)
    full = m.get_last_selfattention(x)
    assert torch.equal(m.cls_attention(x), full[:, :, 0, :])


def test_cls_attention_byte_and_mixed_clips():
    from videotransformer_pytorch_b200.mixup import MixedClip
    m = _ts('divided_space_time', 4, 32, 128, 2)
    u8 = torch.randint(0, 256, (2, 4, 32, 32, 3), dtype=torch.uint8, device=DEV)
    assert torch.equal(m.cls_attention(u8), m.get_last_selfattention(u8)[:, :, 0, :])
    mc = MixedClip(u8, 2, 0.6, (0, 16, 0, 16))
    assert torch.equal(m.cls_attention(mc), m.get_last_selfattention(mc)[:, :, 0, :])


@pytest.mark.parametrize('N,hd', [(1, 64), (9, 32), (197, 96), (256, 128), (257, 64), (1569, 128), (3137, 32),
                                  (12545, 128)])
def test_kernel_row_equals_vt_attn_fwd_row(N, hd):
    """vt_attn_cls_probs == row 0 of vt_attn_fwd's probs, through both routes (N <= 256 generic, above row-tile); at
    N = 12545 the full map does not fit the row-tile kernel, so the row is checked against fp64"""
    from videotransformer_pytorch_b200 import _lib, attn_maps_lib
    k = _lib.K
    H, Bp = 2, 2
    torch.manual_seed(N)
    qkv = (torch.randn(Bp, N, 3, H, hd, device=DEV) * 1.5).to(torch.bfloat16)
    row = attn_maps_lib.K.attn_cls_probs(qkv, Bp, N, H, hd, hd ** -0.5)
    if N <= 5000:
        full = k.attn_fwd(qkv, Bp, N, H, hd, hd ** -0.5, want_probs=True)[2]
        assert torch.equal(row, full[:, :, 0, :])
    q = qkv.double()
    s = torch.einsum('bhd,bnhd->bhn', q[:, 0, 0], q[:, :, 1]) * hd ** -0.5
    ref = torch.softmax(s, dim=-1)
    assert float((row.double() - ref).abs().max()) < 1e-5


def test_masks_match_show_attn_outside_the_bound():
    m = _ts('joint_space_time', 8, 64, 64, 2)
    x = torch.randn(2, 8, 3, 64, 64, device=DEV)
    cls = m.cls_attention(x)
    for threshold in (0.6, 0.9):
        heat, mask = m.attention_maps(x, threshold)
        pat = cls[:, :, 1:].reshape(-1, cls.shape[2] - 1)
        rows_mask = _lib_mask(pat, threshold)
        # in the map's layout: token order p * T + t -> [T, w, h]
        T = 8
        want = rows_mask.reshape(2, 2, -1, T).transpose(2, 3).reshape(mask.shape)
        assert torch.equal(mask, want)
        # the kernel is its restatement, bit for bit, and show_attn's arithmetic outside the bound
        assert torch.equal(rows_mask.cpu(), torch.from_numpy(mass_mask_rows(pat.cpu().numpy(), 1 - threshold)))
        check_against_show_attn(pat.cpu(), threshold, rows_mask.cpu())
    # long rows and ties straight through the kernel
    g = torch.Generator().manual_seed(3)
    for n in (8, 196, 1568, 12544):
        p = torch.softmax(torch.randn(3, n, generator=g, dtype=torch.float64) * 4, -1).float()
        p[1] = torch.tensor([1., 2., 2., 5.])[torch.randint(0, 4, (n,), generator=g)] / n
        got = _lib_mask(p.to(DEV), 0.6).cpu()
        assert torch.equal(got, torch.from_numpy(mass_mask_rows(p.numpy(), 1 - 0.6)))
        check_against_show_attn(p, 0.6, got)


def _lib_mask(rows, threshold):
    from videotransformer_pytorch_b200 import attn_maps_lib
    return attn_maps_lib.K.attn_mass_mask(rows, threshold)


def test_get_last_selfattention_forward_only_is_identical_and_smaller():
    m = _ts('divided_space_time', 8, 224, 384, 6, layers=3)
    x = torch.randn(2, 8, 3, 224, 224, device=DEV)
    with torch.no_grad():                   # warm-up of both forms: shadows, index maps, kernel attributes
        m.get_last_selfattention(x)
    m.get_last_selfattention(x)
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    full = m.get_last_selfattention(x)
    torch.cuda.synchronize()
    peak_grad = torch.cuda.max_memory_allocated() - base
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    with torch.no_grad():
        fo = m.get_last_selfattention(x)
    torch.cuda.synchronize()
    peak_fo = torch.cuda.max_memory_allocated() - base
    assert torch.equal(fo, full)
    assert peak_fo < peak_grad, (peak_fo, peak_grad)


def test_cls_attention_peak_is_below_one_full_map():
    m = _ts('joint_space_time', 8, 224, 768, 12, layers=2)
    x = torch.randn(2, 8, 3, 224, 224, device=DEV)
    m.cls_attention(x)                      # warm-up: shadows, index maps, kernel attributes
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    row = m.cls_attention(x)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    N = row.shape[-1]
    assert N == 1569
    assert peak < 2 * 12 * N * N * 4, peak


def test_cls_attention_in_a_captured_graph():
    from videotransformer_pytorch_b200.graph import GraphedForward
    m = _ts('joint_space_time', 4, 64, 128, 2)
    x = torch.randn(2, 4, 3, 64, 64, device=DEV)
    g = GraphedForward(m.cls_attention, (x,))
    for trial in range(2):
        x2 = torch.randn(2, 4, 3, 64, 64, device=DEV)
        out = g(x2).clone()
        assert torch.equal(out, m.cls_attention(x2))


def test_bad_parameters_are_refused():
    from videotransformer_pytorch_b200 import _lib, attn_maps_lib
    lib = attn_maps_lib.library()
    qkv = torch.zeros(2, 8, 3, 2, 64, dtype=torch.bfloat16, device=DEV)
    out = torch.zeros(2, 2, 8, device=DEV)
    stream = _lib._stream()

    def cls_rc(**kw):
        p = attn_maps_lib.AttnClsProbsParams()
        p.qkv, p.probs, p.Bp, p.N, p.H, p.hd, p.scale = qkv.data_ptr(), out.data_ptr(), 2, 8, 2, 64, 0.125
        for k, v in kw.items():
            setattr(p, k, v)
        return lib.vt_attn_cls_probs(ctypes.byref(p), stream)

    assert cls_rc() == 0
    assert cls_rc(N=0) != 0
    assert cls_rc(hd=48) != 0
    assert cls_rc(qkv=None) != 0
    assert cls_rc(probs=None) != 0
    assert cls_rc(Bp=0) != 0

    rows = torch.rand(4, 100, device=DEV)
    mask = torch.zeros_like(rows)

    def mm_rc(**kw):
        p = attn_maps_lib.AttnMassMaskParams()
        p.probs, p.ld, p.mask, p.ldm, p.rows, p.n, p.thresh = rows.data_ptr(), 100, mask.data_ptr(), 100, 4, 100, 0.4
        for k, v in kw.items():
            setattr(p, k, v)
        return lib.vt_attn_mass_mask(ctypes.byref(p), stream)

    assert mm_rc() == 0
    assert mm_rc(n=0) != 0
    assert mm_rc(n=16385, ld=16385, ldm=16385) != 0
    assert mm_rc(mask=None) != 0
    assert mm_rc(ld=50) != 0
    assert mm_rc(rows=0) != 0
    torch.cuda.synchronize()
    assert float(out.sum()) == pytest.approx(4.0, rel=1e-5)      # the accepted calls ran: rows of probabilities
