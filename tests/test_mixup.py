"""Mixup / CutMix (reference mixup.py:58-126): RNG-stream parity of the draw and the fused uint8 operand path.

tests/golden/mixup.npz was produced by the reference's own Mixup class under np.random.seed (oracle/make_golden.py mixup)."""
import os

import numpy as np
import pytest
import torch

from tests.conftest import load_golden, rel_err


@pytest.fixture(scope='module')
def gold():
    return load_golden('mixup')


def _norm(u8):
    return ((u8.float() / 255.0 - 0.45) / 0.225).permute(0, 1, 4, 2, 3).contiguous()


def test_float_clips_and_targets_equal_the_reference(gold):
    from videotransformer_pytorch_b200 import Mixup
    kinds = set()
    for seed in gold['seeds']:
        u8, labels = torch.from_numpy(gold[f'u8_{seed}']), torch.from_numpy(gold[f'labels_{seed}'])
        np.random.seed(int(seed))
        fn = Mixup(num_classes=int(gold['num_classes']))
        xm, tgt = fn(_norm(u8), labels)
        assert torch.equal(xm, torch.from_numpy(gold[f'mixed_{seed}'])), seed          # bit-identical blend
        assert torch.equal(tgt, torch.from_numpy(gold[f'target_{seed}'])), seed
        np.random.seed(int(seed))
        kinds.add(Mixup(num_classes=7).draw((32, 32))[0])
    assert kinds == {1, 2}                      # both mixup and cutmix draws are covered by the stored seeds


def test_uint8_clips_get_a_plan_that_reproduces_the_reference_blend(gold, emu):
    """The uint8 path defers the blend to the patch-operand kernel: the emulated kernel fed the plan gives im2col(reference mix)."""
    from videotransformer_pytorch_b200 import MixedClip, Mixup
    for seed in gold['seeds']:
        u8, labels = torch.from_numpy(gold[f'u8_{seed}']), torch.from_numpy(gold[f'labels_{seed}'])
        np.random.seed(int(seed))
        mixed, tgt = Mixup(num_classes=int(gold['num_classes']))(u8, labels)
        assert isinstance(mixed, MixedClip) and mixed.clip is u8
        assert torch.equal(tgt, torch.from_numpy(gold[f'target_{seed}'])), seed
        scale = torch.full((3,), 1.0 / (255.0 * 0.225))
        shift = torch.full((3,), -0.45 / 0.225)
        cols = emu.im2col_u8_mix(u8, scale, shift, mixed.plan, 1, 16, 16)
        ref = emu.im2col(torch.from_numpy(gold[f'mixed_{seed}']), 1, 16, 16)
        assert rel_err(cols, ref) < 1e-6, seed


def test_disabled_and_odd_batches():
    from videotransformer_pytorch_b200 import Mixup
    fn = Mixup(num_classes=5)
    fn.mixup_enabled = False
    x = torch.randn(2, 3, 8, 8)
    y, t = fn(x.clone(), torch.tensor([1, 3]))
    assert torch.equal(x, y)
    assert torch.allclose(t.sum(-1), torch.ones(2))
    with pytest.raises(AssertionError):
        fn(torch.randn(3, 3, 8, 8), torch.tensor([0, 1, 2]))


def test_head_loss_matches_torch_on_emulation(emu):
    """ClassificationHead.forward / .loss route through the skinny-GEMV + softmax-CE kernel table entries."""
    from videotransformer_pytorch_b200 import ClassificationHead, cross_entropy
    torch.manual_seed(0)
    head = ClassificationHead(11, 32)
    with torch.no_grad():
        head.cls_head.bias.normal_()
    ref = torch.nn.Linear(32, 11)
    ref.load_state_dict(head.cls_head.state_dict())
    x = torch.randn(6, 32, requires_grad=True)
    xr = x.detach().clone().requires_grad_(True)
    y = torch.randint(0, 11, (6,))
    loss = head.loss(x, y)
    loss_r = torch.nn.functional.cross_entropy(ref(xr), y)
    (loss * 3).backward(); (loss_r * 3).backward()
    assert abs(float(loss) - float(loss_r)) < 1e-6
    assert rel_err(x.grad, xr.grad) < 1e-5
    assert rel_err(head.cls_head.weight.grad, ref.weight.grad) < 1e-5 and rel_err(head.cls_head.bias.grad, ref.bias.grad) < 1e-5
    soft = torch.rand(6, 11); soft = soft / soft.sum(-1, keepdim=True)
    z = torch.randn(6, 11, requires_grad=True)
    ls = cross_entropy(z, soft)
    lr = torch.sum(-soft * torch.log_softmax(z.detach(), dim=-1), dim=-1).mean()          # timm SoftTargetCrossEntropy
    assert abs(float(ls) - float(lr)) < 1e-6
