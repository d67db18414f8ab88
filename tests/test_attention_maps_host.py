"""cls-row attention and show_attn's threshold masks on the CPU: the model surface (cls_attention, attention_maps) on the
CPU kernel tables, the mass-mask kernel's restatement (tests/emu_attention_maps.mass_mask_rows) against show_attn's own torch
code (reference visualize_attention.py:73-82) within the bound derived in vt_attn_maps.cu, and a walk-through of the new
kernels' index arithmetic."""
import math

import numpy as np
import pytest
import torch

from tests.emu_attention_maps import emu_maps, mass_mask_rows  # noqa: F401  (emu_maps: fixture)

TS_TYPES = ['divided_space_time', 'space_only', 'joint_space_time']
VV_TYPES = ['fact_encoder', 'joint_space_time', 'divided_space_time']


def beta(n):
    """vt_attn_maps.cu's bound on |kernel cumulative mass - show_attn's|"""
    return 1.01 * (n + 5) * 2.0 ** -24


def show_attn_masks(attentions, threshold, stable=False):
    """show_attn's thresholding, literally (visualize_attention.py:73-80), on [nh, n] -> (th_attn in patch order, cumval in
    sorted order, idx)"""
    val, idx = torch.sort(attentions, stable=stable) if stable else torch.sort(attentions)
    val /= torch.sum(val, dim=1, keepdim=True)
    cumval = torch.cumsum(val, dim=1)
    th_attn = cumval > (1 - threshold)
    idx2 = torch.argsort(idx)
    for head in range(attentions.shape[0]):
        th_attn[head] = th_attn[head][idx2[head]]
    return th_attn.float(), cumval, idx


def check_against_show_attn(x, threshold, mask):
    """mask (patch order) == show_attn's, except patches whose cumulative mass lies within beta(n) of 1 - threshold; tie
    runs may keep other members, never another count.  -> number of patches the bound excused"""
    n = x.shape[1]
    tau = float(np.float32(1 - threshold))
    ref, cum, idx = show_attn_masks(x.clone(), threshold)
    ref_st, cum_st, idx_st = show_attn_masks(x.clone(), threshold, stable=True)
    assert torch.equal(cum, cum_st)                       # the tie order moves members, not cumulative values
    near = torch.zeros_like(ref, dtype=torch.bool)
    near.scatter_(1, idx_st, (cum_st - tau).abs() <= beta(n))
    # stable order (the kernel's): equal outside the bound
    assert torch.equal(mask[~near], ref_st[~near])
    # torch's default order: the same count kept in every run of equal values that has no patch within the bound
    for r in range(x.shape[0]):
        for v in torch.unique(x[r]):
            run = x[r] == v
            if not bool(near[r][run].any()):
                assert int(mask[r][run].sum()) == int(ref[r][run].sum())
    return int(near.sum())


def softmax_rows(logits):
    return torch.softmax(logits.double(), dim=-1).float()


@pytest.mark.parametrize('n', [8, 196, 1000, 1025, 3136, 12544])
def test_mass_mask_restatement_matches_show_attn(n):
    g = torch.Generator().manual_seed(n)
    x = softmax_rows(torch.randn(6, n, generator=g) * 3)
    for threshold in (0.6, 0.9, 0.1):
        mask = torch.from_numpy(mass_mask_rows(x.numpy(), 1 - threshold))
        check_against_show_attn(x, threshold, mask)


def test_mass_mask_ties_and_threshold_on_a_cumulative_value():
    # ties: a handful of distinct values repeated, in shuffled patch order
    g = torch.Generator().manual_seed(1)
    vals = torch.tensor([1., 2., 2., 3., 5., 5., 5., 8.]) / 64
    x = vals[torch.randint(0, len(vals), (4, 196), generator=g)]
    x = x / x.sum(1, keepdim=True)
    for threshold in (0.6, 0.3, 0.95):
        check_against_show_attn(x, threshold, torch.from_numpy(mass_mask_rows(x.numpy(), 1 - threshold)))
    # dyadic rows whose cumulative sums are exact: 1 - threshold = 0.5 falls exactly on a cumulative value, which is
    # not kept (strict >) by either side
    x = torch.tensor([[1., 1., 2., 4.], [4., 2., 1., 1.], [2., 2., 2., 2.]]) / 8
    mask = torch.from_numpy(mass_mask_rows(x.numpy(), 0.5))
    ref, cum, _ = show_attn_masks(x.clone(), 0.5, stable=True)
    assert bool((cum == 0.5).any(dim=1).all())
    assert torch.equal(mask, ref)
    assert mask.tolist() == [[0., 0., 0., 1.], [1., 0., 0., 0.], [0., 0., 1., 1.]]


def test_mass_mask_uniform_row_keeps_the_last_indices():
    """a row of equal values: ties sort by patch index, so the highest indices carry the largest cumulative mass"""
    x = np.full((1, 1000), 1 / 1000, dtype=np.float32)
    mask = mass_mask_rows(x, 0.4)
    kept = int(mask.sum())
    assert kept in (599, 600, 601)
    assert np.all(mask[0, -kept:] == 1) and np.all(mask[0, :-kept] == 0)


def _emu_model(cls, kind, hd=16, **kw):
    torch.manual_seed(0)
    if cls == 'ts':
        from videotransformer_pytorch_b200 import TimeSformer
        m = TimeSformer(num_frames=4, img_size=32, patch_size=16, embed_dims=2 * hd, num_heads=2, num_transformer_layers=2,
                        attention_type=kind, **kw)
        x = torch.randn(2, 4, 3, 32, 32)
    else:
        from videotransformer_pytorch_b200 import ViViT
        m = ViViT(num_frames=4, img_size=32, patch_size=16, embed_dims=2 * hd, num_heads=2, num_transformer_layers=2,
                  attention_type=kind, **kw)
        x = torch.randn(2, 4, 3, 32, 32)
    return m.eval(), x


@pytest.mark.parametrize('cls,kind', [('ts', k) for k in TS_TYPES] + [('vv', k) for k in VV_TYPES])
def test_cls_attention_is_row_zero_of_get_last_selfattention(emu, emu_maps, cls, kind):
    m, x = _emu_model(cls, kind)
    full = m.get_last_selfattention(x)
    with torch.no_grad():
        full_ng = m.get_last_selfattention(x)
    row = m.cls_attention(x)
    assert row.shape == full.shape[:3] and torch.equal(row, full[:, :, 0, :])
    assert torch.equal(full_ng, full)
    assert ('attn_cls_probs', full.shape[-1]) in emu_maps.calls


def test_cls_attention_resized_timesformer_and_byte_clips(emu, emu_maps):
    m, _ = _emu_model('ts', 'divided_space_time')
    x = torch.randn(1, 4, 3, 48, 64)                        # interpolated pos_embed: 3 x 4 patches
    assert torch.equal(m.cls_attention(x), m.get_last_selfattention(x)[:, :, 0, :])
    from videotransformer_pytorch_b200.mixup import MixedClip
    u8 = torch.randint(0, 256, (2, 4, 32, 32, 3), dtype=torch.uint8)
    assert torch.equal(m.cls_attention(u8), m.get_last_selfattention(u8)[:, :, 0, :])
    mc = MixedClip(u8, 1, 0.7, (0, 0, 0, 0))
    assert torch.equal(m.cls_attention(mc), m.get_last_selfattention(mc)[:, :, 0, :])


@pytest.mark.parametrize('cls,kind', [('ts', k) for k in TS_TYPES] + [('vv', k) for k in VV_TYPES])
def test_attention_maps_layout(emu, emu_maps, cls, kind):
    m, _ = _emu_model(cls, kind)
    x = torch.randn(1, 4, 3, 32, 48)
    if cls == 'vv':
        x = torch.randn(1, 4, 3, 32, 32)
    wf, hf = x.shape[3] // 16, x.shape[4] // 16
    c = m.cls_attention(x)
    heat, mask = m.attention_maps(x, threshold=0.6)
    nh = c.shape[1]
    if kind == 'fact_encoder':
        assert heat.shape == (1, nh, c.shape[2] - 1) and torch.equal(heat, c[:, :, 1:])
    elif kind == 'joint_space_time':
        T = (c.shape[2] - 1) // (wf * hf)
        assert heat.shape == (1, nh, T, wf, hf)
        for t in range(T):
            for i in range(wf):
                for j in range(hf):
                    assert torch.equal(heat[0, :, t, i, j], c[0, :, 1 + (i * hf + j) * T + t])
    else:
        assert heat.shape == (c.shape[0], nh, wf, hf)
        assert torch.equal(heat.reshape(c.shape[0], nh, -1), c[:, :, 1:])
    assert mask.shape == heat.shape and set(mask.unique().tolist()) <= {0.0, 1.0}
    # the mask is show_attn's on each (frame or clip, head) row, in the heatmap's layout
    rows = c[:, :, 1:].reshape(-1, c.shape[2] - 1)
    want = torch.from_numpy(mass_mask_rows(rows.numpy(), 0.4)).reshape(c[:, :, 1:].shape)
    if kind == 'joint_space_time':
        T = (c.shape[2] - 1) // (wf * hf)
        want = want.reshape(1, nh, wf * hf, T).transpose(2, 3).reshape(mask.shape)
    assert torch.equal(mask, want.reshape(mask.shape))
    assert m.attention_maps(x, threshold=None)[1] is None


# ------------------------------------------------------------------------------------------------------------------
# index arithmetic of the new kernels
# ------------------------------------------------------------------------------------------------------------------
def sim_bitonic(keys):
    """mass_mask_kernel's sort: pair p of step (k, j) -> i = p with a zero inserted at bit log2(j), partner i + j"""
    keys = list(keys)
    npad = len(keys)
    for k in (2 ** e for e in range(1, int(math.log2(npad)) + 1)):
        j = k >> 1
        while j > 0:
            touched = []
            for p in range(npad // 2):
                i = ((p & ~(j - 1)) << 1) | (p & (j - 1))
                assert i & j == 0
                touched += [i, i + j]
                a, b = keys[i], keys[i + j]
                if (a > b) == ((i & k) == 0):
                    keys[i], keys[i + j] = b, a
            assert sorted(touched) == list(range(npad))       # each position in exactly one pair per step
            j >>= 1
    return keys


@pytest.mark.parametrize('n', [1, 7, 8, 100, 1024, 1025])
def test_mass_mask_sort_chunks_and_scatter(n):
    rng = np.random.default_rng(n)
    x = rng.integers(0, 5, n).astype(np.float32) / 7          # ties
    npad = max(1024, 1 << (n - 1).bit_length())
    u = x.view(np.uint32).astype(np.uint64)
    ob = np.where(u & 0x80000000, ~u & 0xffffffff, u | 0x80000000)
    keys = [(int(b) << 32) | i for i, b in enumerate(ob)] + [2 ** 64 - 1] * (npad - n)
    got = sim_bitonic(keys)
    assert got == sorted(keys)
    order = [kk & 0xffffffff for kk in got[:n]]
    assert order == list(np.argsort(x, kind='stable'))       # ascending, ties by patch index
    # thread t owns sorted positions [t * chunk, (t + 1) * chunk): every position once, in order
    chunk = npad // 1024
    owned = [t * chunk + e for t in range(1024) for e in range(chunk)]
    assert owned == list(range(npad))
    # the scatter writes position k's flag to patch order[k]: a permutation of the row
    assert sorted(order) == list(range(n))


@pytest.mark.parametrize('N', [1, 9, 197, 256, 257, 1569, 12545])
def test_cls_kernels_cover_every_key_once(N):
    if N <= 256:
        # generic row: lane owns keys lane + 32 jj, jj < MAX_N / 32
        owners = [j for lane in range(32) for jj in range(256 // 32) if (j := lane + 32 * jj) < N]
    else:
        # tiled: thread t scores key j0 + t of each 256-key tile; the softmax warp reads lanes' strided keys
        owners = [j for j0 in range(0, N, 256) for t in range(256) if (j := j0 + t) < N]
        assert sorted(j for lane in range(32) for j in range(lane, N, 32)) == list(range(N))
    assert sorted(owners) == list(range(N))
    # shared memory of the tiled kernel at head dim 128 stays within the 227 KB a CTA may opt into
    if N > 256:
        assert (N + 128 + 256 * 129) * 4 <= 227 * 1024
