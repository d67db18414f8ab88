"""Classification head, softmax-CE, long-sequence attention maps and the Mixup/CutMix operand kernel vs fp32 torch.  -m gpu"""
import os

import numpy as np
import pytest
import torch

from tests.conftest import load_golden, rel_err

pytestmark = pytest.mark.gpu


def K():
    from videotransformer_pytorch_b200 import _lib
    return _lib.K


@pytest.mark.parametrize('M,N,Kd', [(8, 400, 768), (1, 400, 768), (16, 174, 768), (72, 10, 128), (3, 1000, 96)])
def test_linear_small_fwd_bwd(M, N, Kd):
    g = torch.Generator().manual_seed(M * 1000 + N)
    x, w, b = torch.randn(M, Kd, generator=g), torch.randn(N, Kd, generator=g) * 0.05, torch.randn(N, generator=g)
    dy = torch.randn(M, N, generator=g)
    y = K().linear_small_fwd(x.cuda(), w.cuda(), b.cuda())
    assert rel_err(y.cpu(), x.double() @ w.double().t() + b.double()) < 1e-6
    dx, dw, db = K().linear_small_bwd(dy.cuda(), x.cuda(), w.cuda())
    assert rel_err(dx.cpu(), dy.double() @ w.double()) < 1e-6
    assert rel_err(dw.cpu(), dy.double().t() @ x.double()) < 1e-6
    assert rel_err(db.cpu(), dy.double().sum(0)) < 1e-6
    y0 = K().linear_small_fwd(x.cuda(), w.cuda(), None)
    assert rel_err(y0.cpu(), x.double() @ w.double().t()) < 1e-6


@pytest.mark.parametrize('M,N', [(8, 400), (16, 174), (2, 7), (64, 1000)])
def test_softmax_ce_hard_and_soft(M, N):
    g = torch.Generator().manual_seed(M + N)
    z = torch.randn(M, N, generator=g) * 3
    y = torch.randint(0, N, (M,), generator=g)
    zr = z.double().requires_grad_(True)
    ref = torch.nn.functional.cross_entropy(zr, y)
    ref.backward()
    loss, dz, row = K().softmax_ce(z.cuda(), labels=y.cuda())
    assert abs(float(loss) - float(ref)) < 1e-5 * abs(float(ref))
    assert rel_err(dz.cpu(), zr.grad) < 1e-5
    assert rel_err(row.cpu(), torch.nn.functional.cross_entropy(z.double(), y, reduction='none')) < 1e-5
    soft = torch.rand(M, N, generator=g)
    soft = soft / soft.sum(-1, keepdim=True)
    zr = z.double().requires_grad_(True)
    ref = torch.sum(-soft.double() * torch.log_softmax(zr, dim=-1), dim=-1).mean()     # timm SoftTargetCrossEntropy
    ref.backward()
    loss, dz, _ = K().softmax_ce(z.cuda(), soft_targets=soft.cuda())
    assert abs(float(loss) - float(ref)) < 1e-5 * abs(float(ref))
    assert rel_err(dz.cpu(), zr.grad) < 1e-5


def test_head_module_and_fused_loss_autograd():
    from videotransformer_pytorch_b200 import ClassificationHead, cross_entropy
    torch.manual_seed(0)
    head = ClassificationHead(400, 768)
    with torch.no_grad():
        head.cls_head.bias.normal_(std=0.1)
    ref = torch.nn.Linear(768, 400)
    ref.load_state_dict(head.cls_head.state_dict())
    head = head.cuda()
    x = torch.randn(8, 768)
    y = torch.randint(0, 400, (8,))
    xg = x.cuda().requires_grad_(True)
    loss = head.loss(xg, y.cuda())
    (2.5 * loss).backward()
    xr = x.clone().requires_grad_(True)
    lr = torch.nn.functional.cross_entropy(ref(xr), y)
    (2.5 * lr).backward()
    assert abs(float(loss) - float(lr)) < 1e-5 * abs(float(lr))
    assert rel_err(xg.grad.cpu(), xr.grad) < 1e-5
    assert rel_err(head.cls_head.weight.grad.cpu(), ref.weight.grad) < 1e-5
    assert rel_err(head.cls_head.bias.grad.cpu(), ref.bias.grad) < 1e-5
    # logits through forward() + torch's own loss (the reference trainer's flow, model_trainer.py:207-208)
    logits = head(x.cuda())
    assert rel_err(logits.cpu(), ref(x)) < 1e-5
    assert abs(float(cross_entropy(logits, y.cuda())) - float(lr)) < 1e-5 * abs(float(lr))


@pytest.mark.parametrize('Bp,H,N', [(1, 12, 1569), (2, 2, 289), (1, 1, 77), (1, 3, 2049)])
def test_attn_fwd_probabilities_long_sequences(Bp, H, N):
    hd = 64
    g = torch.Generator().manual_seed(N)
    qkv = (torch.randn(Bp * N, 3 * H * hd, generator=g)).bfloat16()
    q5 = qkv.float().view(Bp, N, 3, H, hd)
    q, k = q5[:, :, 0].permute(0, 2, 1, 3), q5[:, :, 1].permute(0, 2, 1, 3)
    ref = ((q.double() @ k.double().transpose(-1, -2)) * hd ** -0.5).softmax(dim=-1)
    # impl 2, the tensor-core path: the row-tile probability kernel at every N, as the automatic choice takes it past 256
    _, _, got = K().attn_fwd(qkv.cuda(), Bp, N, H, hd, hd ** -0.5, want_probs=True, impl=2)
    assert got.shape == (Bp, H, N, N)
    assert rel_err(got.cpu(), ref) < 1e-5
    assert float((got.sum(-1) - 1).abs().max()) < 1e-5


def test_get_last_selfattention_joint_space_time_1569_tokens():
    """TimeSformer joint_space_time at 8x224 (1569 tokens): get_last_selfattention (video_transformer.py:258-261) returns the
    [B, 12, 1569, 1569] map of the last layer — served by the row-tile kernel, checked against the fp64 oracle."""
    from oracle import vt_oracle as O
    from videotransformer_pytorch_b200 import TimeSformer
    cfg = dict(num_frames=8, img_size=224, patch_size=16, embed_dims=768, num_heads=12, num_transformer_layers=1)
    sd = O.random_timesformer_state(dict(cfg), seed=9)
    sd = {k: v for k, v in sd.items() if 'attentions.1' not in k and 'temporal_fc' not in k}
    m = TimeSformer(attention_type='joint_space_time', **cfg)
    m.load_state_dict(sd, strict=True)
    m = m.cuda().eval()
    x = torch.randn(1, 8, 3, 224, 224, generator=torch.Generator().manual_seed(3))
    with torch.no_grad():
        attn = m.get_last_selfattention(x.cuda())
        tok = O.timesformer_tokens({k: v.double() for k, v in sd.items()}, x.double(), cfg)
        ref = O.container(tok, {k: v.double() for k, v in sd.items()}, 'transformer_layers.', 1, ['self_attn', 'ffn'], 8, 12,
                          False, return_attention=True)
    assert attn.shape == (1, 12, 1569, 1569) == ref.shape
    e = rel_err(attn.cpu(), ref)
    print(f'joint_space_time last attention (1569 tokens): rel-L2 {e:.2e}')
    assert e < 1e-2


def test_attention_module_long_sequence_forward_backward():
    """Stand-alone Attention.forward (transformer.py:165-177) past 256 tokens: context from the tiled tensor-core kernels,
    probabilities from the row-tile kernel, gradients through the tiled backward."""
    from videotransformer_pytorch_b200 import Attention
    torch.manual_seed(1)
    a = Attention(128, num_heads=2, qkv_bias=True)
    ref_qkv, ref_proj = torch.nn.Linear(128, 384), torch.nn.Linear(128, 128)
    ref_qkv.load_state_dict(a.qkv.state_dict()); ref_proj.load_state_dict(a.proj.state_dict())
    x = torch.randn(2, 300, 128)
    xg = x.cuda().requires_grad_(True)
    a = a.cuda()
    out, attn = a(xg)
    out.square().sum().backward()
    xr = x.double().requires_grad_(True)
    qkv = (xr @ ref_qkv.weight.double().t() + ref_qkv.bias.double()).reshape(2, 300, 3, 2, 64).permute(2, 0, 3, 1, 4)
    p = ((qkv[0] @ qkv[1].transpose(-1, -2)) * 64 ** -0.5).softmax(-1)
    o = (p @ qkv[2]).transpose(1, 2).reshape(2, 300, 128) @ ref_proj.weight.double().t() + ref_proj.bias.double()
    o.square().sum().backward()
    assert rel_err(out.detach().cpu(), o.detach()) < 1e-2 and rel_err(attn.cpu(), p.detach()) < 1e-2
    assert rel_err(xg.grad.cpu(), xr.grad) < 3e-2


def test_mixup_cutmix_operand_kernel_vs_reference_goldens():
    """vt_im2col_u8_mix_bf16 against clips mixed by the reference's Mixup class (tests/golden/mixup.npz)."""
    from videotransformer_pytorch_b200 import Mixup
    gold = load_golden('mixup')
    scale = torch.full((3,), 1.0 / (255.0 * 0.225)).cuda()
    shift = torch.full((3,), -0.45 / 0.225).cuda()
    for seed in gold['seeds']:
        u8, labels = torch.from_numpy(gold[f'u8_{seed}']), torch.from_numpy(gold[f'labels_{seed}'])
        np.random.seed(int(seed))
        mixed, tgt = Mixup(num_classes=int(gold['num_classes']))(u8.cuda(), labels.cuda())
        assert torch.equal(tgt.cpu(), torch.from_numpy(gold[f'target_{seed}']))
        cols = K().im2col_u8_mix(mixed.clip, scale, shift, mixed.plan, 1, 16, 16)
        ref = K().im2col(torch.from_numpy(gold[f'mixed_{seed}']).cuda(), 1, 16, 16)
        assert rel_err(cols.float().cpu(), ref.float().cpu()) < 4e-3, (seed, mixed.mode)      # bf16 rounding of both sides
        same = (cols == ref).float().mean().item()
        assert same > 0.99, (seed, same)


def test_model_consumes_mixed_uint8_clip():
    """TimeSformer(MixedClip) == TimeSformer(float clip mixed by the reference-order ops), eval mode."""
    from videotransformer_pytorch_b200 import Mixup, TimeSformer
    torch.manual_seed(2)
    m = TimeSformer(num_frames=4, img_size=48, patch_size=16, embed_dims=128, num_heads=2, num_transformer_layers=1).cuda().eval()
    u8 = torch.randint(0, 256, (4, 4, 48, 48, 3), dtype=torch.uint8)
    labels = torch.tensor([0, 1, 2, 3])
    for seed in (0, 1, 2, 3):
        np.random.seed(seed)
        mixed, t1 = Mixup(num_classes=4)(u8.cuda(), labels.cuda())
        np.random.seed(seed)
        xf = ((u8.float() / 255.0 - 0.45) / 0.225).permute(0, 1, 4, 2, 3).contiguous()
        xm, t2 = Mixup(num_classes=4)(xf.cuda(), labels.cuda())
        with torch.no_grad():
            a, b = m(mixed), m(xm)
        assert torch.equal(t1, t2)
        assert rel_err(a, b) < 2e-3, seed
