"""MViT / MaskFeat kernels against the ORACLE's own functions (oracle/mvit_oracle.py), not the kernel emulation.  -m gpu

tests/test_gpu_mvit.py checks every kernel of csrc/vt_mvit.cu / vt_xattention_tc.cu against tests/emu_kernels.py (a CPU
statement of each kernel's contract, written with the kernels).  This file closes the loop to the restated reference
algorithm: the same kernels — and whole MultiScaleBlocks at the MViT-B stage shapes — are compared with
`mvit_oracle.attention_pool`, `multiscale_attention`'s softmax core, `multiscale_block`, `cls_positional_encoding`,
`maskfeat_forward_features`' mask mixing and `maskfeat_forward`'s loss, forward and (through torch autograd over the oracle)
backward.  Operands are rounded to bf16 once and fed to both sides, so fp32-output quantities agree to ~1e-5 and
bf16-output quantities to bf16 resolution.
"""
import math

import pytest
import torch

from tests.conftest import rel_err

pytestmark = pytest.mark.gpu
HD = 96


def K():
    from videotransformer_pytorch_b200 import _lib
    return _lib.K


def rn(shape, seed, scale=1.0):
    return torch.randn(shape, generator=torch.Generator().manual_seed(seed)) * scale


@pytest.mark.parametrize('thw,stride,H,B', [((8, 14, 14), (1, 2, 2), 4, 2), ((8, 28, 28), (1, 4, 4), 2, 1),
                                            ((4, 16, 16), (1, 8, 8), 1, 2), ((2, 5, 7), (1, 1, 1), 2, 1)])
def test_pool_kernels_vs_oracle_attention_pool(thw, stride, H, B):
    from oracle import mvit_oracle as MO
    N1 = 1 + thw[0] * thw[1] * thw[2]
    d = H * HD
    qkv = rn((B * N1, 3 * d), 10).bfloat16()
    w = rn((HD, 1, 3, 3, 3), 11, 0.3)
    gamma, beta = 1 + rn((HD,), 12, 0.1), rn((HD,), 13, 0.1)
    slot = 1
    # oracle: [B, heads, N, hd] view of the k slice, autograd for the adjoints
    t = qkv.float().view(B, N1, 3, H, HD)[:, :, slot].permute(0, 2, 1, 3).clone().requires_grad_(True)
    wr, gr, br = w.clone().requires_grad_(True), gamma.clone().requires_grad_(True), beta.clone().requires_grad_(True)
    out_o, othw = MO.attention_pool(t, thw, conv_w=wr, stride=stride, norm_w=gr, norm_b=br, eps=1e-5)
    dout = rn(tuple(out_o.shape), 14)
    out_o.backward(dout)
    qg = qkv.cuda()
    src = qg.view(B, N1, 3 * d)[:, :, slot * d:(slot + 1) * d]
    out, pooled, mean, rstd, othw_g = K().pool_fwd(src, H, HD, thw, stride, w.reshape(HD, 27).cuda(), gamma.cuda(),
                                                   beta.cuda(), 1e-5)
    assert tuple(othw_g) == tuple(othw)
    assert rel_err(out.float().cpu(), out_o.detach()) < 4e-3                  # bf16 output
    dq = torch.zeros((B * N1, 3 * d), dtype=torch.bfloat16, device='cuda')
    din = dq.view(B, N1, 3 * d)[:, :, slot * d:(slot + 1) * d]
    dw, dg, db = K().pool_bwd(dout.cuda(), pooled, mean, rstd, gamma.cuda(), src, w.reshape(HD, 27).cuda(), din, H, HD,
                              thw, stride)
    din_o = t.grad.permute(0, 2, 1, 3).reshape(B, N1, d)
    assert rel_err(din.float().cpu(), din_o) < 5e-3
    assert rel_err(dw.cpu(), wr.grad.reshape(HD, 27)) < 1e-4
    assert rel_err(dg.cpu(), gr.grad) < 1e-4 and rel_err(db.cpu(), br.grad) < 1e-4


@pytest.mark.parametrize('B,H,Nq,Nk', [(1, 1, 2000, 393), (2, 2, 1569, 393), (1, 8, 393, 393), (1, 4, 700, 1569)])
def test_pooling_attention_vs_oracle_softmax_core(B, H, Nq, Nk):
    """softmax((q k^T) * hd^-0.5) v as mvit_oracle.multiscale_attention states it, at the MViT-B stage sizes."""
    scale = HD ** -0.5
    q, k, v = (rn((B, H, n, HD), s).bfloat16() for n, s in ((Nq, 20), (Nk, 21), (Nk, 22)))
    qr, kr, vr = (t.float().requires_grad_(True) for t in (q, k, v))
    attn = ((qr @ kr.transpose(-2, -1)) * scale).softmax(dim=-1)
    o_o = (attn @ vr).transpose(1, 2).reshape(B, Nq, H * HD)
    dout = rn((B, Nq, H * HD), 23).bfloat16()
    o_o.backward(dout.float())
    o, lse = K().xattn_fwd(q.cuda(), k.cuda(), v.cuda(), scale)
    assert rel_err(o.float().cpu(), o_o.detach()) < 1e-2
    dq = torch.empty((B, H, Nq, HD), dtype=torch.bfloat16, device='cuda')
    dk, dv = K().xattn_bwd(q.cuda(), k.cuda(), v.cuda(), o, dout.cuda(), lse, scale, dq)
    assert rel_err(dq.float().cpu(), qr.grad) < 2e-2
    assert rel_err(dk.cpu(), kr.grad) < 2e-2 and rel_err(dv.cpu(), vr.grad) < 2e-2


@pytest.mark.parametrize('thw,stride,D,B', [((8, 56, 56), (1, 2, 2), 96, 1), ((8, 28, 28), (1, 2, 2), 192, 2)])
def test_skip_maxpool_vs_oracle(thw, stride, D, B):
    from oracle import mvit_oracle as MO
    kernel = tuple(s + 1 if s > 1 else s for s in stride)
    x = rn((B, 1 + thw[0] * thw[1] * thw[2], D), 30).requires_grad_(True)
    y_o, othw = MO.attention_pool(x, thw, max_kernel=kernel, stride=stride)
    dy = rn(tuple(y_o.shape), 31)
    y_o.backward(dy)
    y, idx, othw_g = K().maxpool_fwd(x.detach().cuda(), thw, kernel, stride)
    assert tuple(othw) == tuple(othw_g) and torch.equal(y.cpu(), y_o.detach())
    dx = K().maxpool_bwd(dy.cuda(), idx, thw, kernel, stride)
    assert rel_err(dx.cpu(), x.grad) < 1e-6


def test_token_preparation_vs_oracle():
    """mask-token mixing (video_transformer.py:917-919) + SpatioTemporalClsPositionalEncoding."""
    from oracle import mvit_oracle as MO
    B, T, H, W, C = 2, 4, 6, 6, 96
    HW, L = H * W, T * H * W
    t = rn((B, L, C), 40)
    mask = (torch.rand(B, T, H // 2, W // 2, generator=torch.Generator().manual_seed(41)) < 0.4).float()
    dense = mask.repeat_interleave(2, dim=2).repeat_interleave(2, dim=3).flatten(1)
    sd = {'mask_token': rn((1, 1, C), 42), 'p.cls_token': rn((1, 1, C), 43), 'p.pos_embed_spatial': rn((1, HW, C), 44),
          'p.pos_embed_temporal': rn((1, T, C), 45), 'p.pos_embed_class': rn((1, 1, C), 46)}
    w = dense.unsqueeze(-1)
    mixed = t * (1 - w) + sd['mask_token'] * w
    ref = MO.cls_positional_encoding(sd, 'p.', mixed, (T, H, W))
    got = K().mvit_tokens_fwd(t.reshape(B * L, C).cuda(), dense.contiguous().cuda(), sd['mask_token'].reshape(C).cuda(),
                              sd['p.cls_token'].reshape(C).cuda(), sd['p.pos_embed_spatial'].reshape(HW, C).cuda(),
                              sd['p.pos_embed_temporal'].reshape(T, C).cuda(), sd['p.pos_embed_class'].reshape(C).cuda(),
                              B, T, HW)
    assert rel_err(got.cpu(), ref) < 1e-6


def test_masked_mse_vs_oracle_loss():
    """Loss half of mvit_oracle.maskfeat_forward (video_transformer.py:882-901) incl. the centre-frame mask."""
    from oracle import mvit_oracle as MO
    B, t, dt, h, w, dc = 2, 8, 2, 14, 14, 108
    L1 = 1 + t * h * w
    pred_rows = rn((B, L1, dt * dc), 60).requires_grad_(True)
    target = rn((B, t * dt, h, w, dc), 61)
    mask = (torch.rand(B, t, h, w, generator=torch.Generator().manual_seed(62)) < 0.3).float()
    markers = [[[0, 2], [5, 1]], [[3, 3]]]
    m = MO.center_frame_mask(mask, markers, dt, t * dt)
    p = pred_rows[:, 1:].reshape(B, t, h, w, dt, dc).permute(0, 1, 4, 2, 3, 5).reshape(B, t * dt, h, w, dc)
    loss_o = (((p - target) ** 2).mean(dim=-1) * m).sum() / (m.sum() + 1e-5)
    loss_o.backward()
    dims = (B, t, dt, h, w, dc)
    num = K().mse_fwd(pred_rows.detach().reshape(B * L1, dt * dc).cuda(), target.cuda(), m.cuda(), dims)
    loss = num[0].item() / (m.sum().item() + 1e-5)
    assert abs(loss - loss_o.item()) < 1e-5 * abs(loss_o.item())
    coef = torch.tensor([(2.0 / dc) / (m.sum().item() + 1e-5)])       # d loss / d (pred - target)^2-sum, as MaskedMSEFn passes it
    dp = K().mse_bwd(pred_rows.detach().reshape(B * L1, dt * dc).cuda(), target.cuda(), m.cuda(), coef.cuda(), dims)
    assert rel_err(dp.float().cpu(), pred_rows.grad.reshape(B * L1, dt * dc)) < 4e-3


# MViT-B blocks as the reference configures them (model_trainer.py:54): (block index, input thw)
STAGE_BLOCKS = [(0, (8, 56, 56)), (1, (8, 56, 56)), (2, (8, 28, 28)), (3, (8, 28, 28)), (14, (8, 14, 14)), (15, (8, 14, 14))]


@pytest.mark.parametrize('index,thw', STAGE_BLOCKS)
def test_multiscale_block_vs_oracle_at_mvit_b_shapes(index, thw):
    """One whole MultiScaleBlock (LN, fused q/k/v GEMM, pooling, tensor-core pooling attention, proj, max-pool skip, MLP, width
    change) forward + all gradients against mvit_oracle.multiscale_block at the real token counts."""
    from oracle import mvit_oracle as MO
    from videotransformer_pytorch_b200.maskfeat import MultiScaleBlock
    cfg = MO.maskfeat_config(img_size=224, num_frames=16, feature_dim=216, pool_q_stride_size=[[1, 1, 2, 2], [3, 1, 2, 2]])
    sd_all = MO.random_maskfeat_state(cfg, seed=31, dtype=torch.float32)
    blk = cfg['blocks'][index]
    pre = f'mvit.blocks.{index}.'
    sd = {k[len(pre):]: v for k, v in sd_all.items() if k.startswith(pre)}
    sq = tuple(blk['stride_q']) if len(blk['stride_q']) > 0 else None
    mod = MultiScaleBlock(blk['dim'], blk['dim_out'], blk['heads'], int(blk['dim'] * 4), sq, tuple(blk['stride_kv']))
    mod.load_state_dict(sd, strict=True)
    mod = mod.cuda().train()
    B = 1
    N1 = 1 + math.prod(thw)
    x = rn((B, N1, blk['dim']), 70 + index)
    xg = x.clone().cuda().requires_grad_(True)
    y, othw = mod(xg, thw)
    wgt = rn(tuple(y.shape), 90 + index) / 30
    (y * wgt.cuda()).sum().backward()
    s = {k: v.clone().requires_grad_(True) for k, v in sd_all.items() if k.startswith(pre)}
    xr = x.clone().requires_grad_(True)
    y_o, othw_o = MO.multiscale_block(s, pre, xr, thw, blk, cfg['block_norm_eps'], cfg['pool_norm_eps'])
    (y_o * wgt).sum().backward()
    assert tuple(othw) == tuple(othw_o)
    e_y, e_dx = rel_err(y.detach().cpu(), y_o.detach()), rel_err(xg.grad.cpu(), xr.grad)
    errs = sorted(((rel_err(p.grad.cpu(), s[pre + n].grad), n) for n, p in mod.named_parameters()
                   if not n.endswith('attn.norm_k.bias')), reverse=True)
    print(f'block {index} thw {thw}: y {e_y:.2e}  dx {e_dx:.2e}  worst param grad {errs[0][0]:.2e} ({errs[0][1]})')
    assert e_y < 5e-3 and e_dx < 2e-2
    assert errs[0][0] < 5e-2, errs[:4]


def test_masked_mse_fp64_targets():
    """fp64 targets (the reference's numpy default): differences and sums in fp64 on the device, fp64 loss; gradient as fp32."""
    B, t, dt, h, w, dc = 2, 8, 2, 14, 14, 108
    L1 = 1 + t * h * w
    pred = rn((B * L1, dt * dc), 63)
    target = torch.randn(B, t * dt, h, w, dc, generator=torch.Generator().manual_seed(64), dtype=torch.float64)
    mask = (torch.rand(B, t * dt, h, w, generator=torch.Generator().manual_seed(65)) < 0.2).float()
    dims = (B, t, dt, h, w, dc)
    num = K().mse_fwd(pred.cuda(), target.cuda(), mask.cuda(), dims)
    assert num.dtype == torch.float64
    p = pred.view(B, L1, dt * dc)[:, 1:].reshape(B, t, h, w, dt, dc).permute(0, 1, 4, 2, 3, 5).reshape(B, t * dt, h, w, dc)
    ref = (((p.double() - target) ** 2).mean(-1) * mask.double()).sum()
    assert abs(num[0].item() - ref.item()) < 1e-12 * abs(ref.item())
    coef = torch.tensor([0.01])
    d64 = K().mse_bwd(pred.cuda(), target.cuda(), mask.cuda(), coef.cuda(), dims)
    d32 = K().mse_bwd(pred.cuda(), target.float().cuda(), mask.cuda(), coef.cuda(), dims)
    assert rel_err(d64.float().cpu(), d32.float().cpu()) < 4e-3
