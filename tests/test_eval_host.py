"""Forward-only evaluation path, host side, on CPU with the kernel table replaced by the twin of tests/emu_kernels.py with
its forward-only forms: the no_grad forward of every golden configuration against the goldens and bit for bit against
the grad-enabled forward, which kernel forms each took, the top-k counter twin against a plain-torch restatement of the
test step, inference mode between training steps, and a linear probe."""
import pytest
import torch

from tests.conftest import rel_err
from tests.emu_kernels import EmuKernels


@pytest.fixture
def emu():
    from videotransformer_pytorch_b200 import _lib
    old = _lib.K
    _lib.K = EmuKernels(exact=True, inference_forms=True)
    yield _lib.K
    _lib.K = old


def _ts(g, attention_type):
    from videotransformer_pytorch_b200 import TimeSformer
    c = g.cfg
    m = TimeSformer(num_frames=c['num_frames'], img_size=c['img_size'], patch_size=c['patch_size'], embed_dims=c['embed_dims'],
                    num_heads=c['num_heads'], num_transformer_layers=c['num_transformer_layers'], attention_type=attention_type)
    m.load_state_dict(g.sd, strict=True)
    return m


def _vv(g, attention_type):
    from videotransformer_pytorch_b200 import ViViT
    c = g.cfg
    m = ViViT(num_frames=c['num_frames_in'], img_size=c['img_size'], patch_size=c['patch_size'], embed_dims=c['embed_dims'],
              num_heads=c['num_heads'], num_transformer_layers=c['num_transformer_layers'], attention_type=attention_type)
    m.load_state_dict(g.sd, strict=True)
    return m


CONFIGS = [
    ('timesformer_tiny', _ts, 'divided_space_time'),
    ('timesformer_hd64', _ts, 'divided_space_time'),
    ('timesformer_space_only_tiny', _ts, 'space_only'),
    ('timesformer_joint_tiny', _ts, 'joint_space_time'),
    ('timesformer_joint_n289', _ts, 'joint_space_time'),
    ('vivit_tiny_b1', _vv, 'fact_encoder'),
    ('vivit_tiny_b3', _vv, 'fact_encoder'),
    ('vivit_joint_tiny', _vv, 'joint_space_time'),
    ('vivit_divided_tiny', _vv, 'divided_space_time'),
]
STAT_CALLS = ('ln_fwd', 'attn_fwd', 'xattn_fwd', 'pool_fwd', 'maxpool_fwd')


def _check_forms(calls, forward_only):
    kinds = {c[0] for c in calls}
    gemm_epis = {c[-1] for c in calls if c[0] == 'gemm'}
    stats = [c[1] for c in calls if c[0] in STAT_CALLS]
    assert stats, 'no call with statistics outputs recorded'
    if forward_only:
        assert 'gelu_h' in gemm_epis and 'gelu' not in kinds      # FC1 writes h; no stand-alone GELU
        assert not any(stats)                                       # no statistics written
    else:
        assert 'gelu_h' not in gemm_epis and 'gelu' in kinds
        assert all(stats)


@pytest.mark.parametrize('name,build,attention_type', CONFIGS, ids=[c[0] for c in CONFIGS])
def test_no_grad_forward_matches_golden_and_grad_forward(golden, emu, name, build, attention_type):
    g = golden(name)
    m = build(g, attention_type).eval()
    emu.calls.clear()
    with torch.no_grad():
        y0 = m(g.x)
    fwd_only = list(emu.calls)
    emu.calls.clear()
    y1 = m(g.x)                                       # grad enabled: the saving forward, unchanged
    saving = list(emu.calls)
    assert rel_err(y0, g.out['y_eval']) < 2e-5
    assert torch.equal(y0, y1.detach())
    _check_forms(fwd_only, True)
    _check_forms(saving, False)
    assert [c[:-1] for c in fwd_only if c[0] == 'gemm'] == [c[:-1] for c in saving if c[0] == 'gemm']   # same GEMMs
    with torch.inference_mode():
        assert torch.equal(m(g.x), y0)


@pytest.mark.parametrize('name', ['maskfeat_s32', 'maskfeat_s64', 'maskfeat_s64_3stage'])
def test_maskfeat_no_grad_forward_features(maskfeat_golden, emu, name):
    from tests.test_host_logic_mvit import build
    g = maskfeat_golden(name)
    m = build(g).eval()
    emu.calls.clear()
    with torch.no_grad():
        f0 = m.forward_features(g.x, g.mask)
    fwd_only = list(emu.calls)
    emu.calls.clear()
    f1 = m.forward_features(g.x, g.mask)
    assert rel_err(f0, g.feats) < 5e-5
    assert torch.equal(f0, f1.detach())
    _check_forms(fwd_only, True)
    _check_forms(emu.calls, False)
    assert any(c[0] == 'pool_fwd' for c in fwd_only) and any(c[0] == 'maxpool_fwd' for c in fwd_only)


def _topk_reference(logits, labels, views, ks):
    """The test step as the reference intends it (model_trainer.py:291-299): mean of the views, softmax, top-k."""
    C = logits.shape[1]
    probs = logits.view(-1, views, C).mean(1).softmax(-1)
    return {k: int((probs.topk(k, dim=-1).indices == labels[:, None]).any(-1).sum()) for k in ks}, probs


@pytest.mark.parametrize('views', [1, 3])
@pytest.mark.parametrize('C', [400, 600])
def test_topk_twin_matches_torch_test_step(emu, views, C):
    from videotransformer_pytorch_b200.metrics import TopKAccuracy
    gen = torch.Generator().manual_seed(views * 1000 + C)
    acc = TopKAccuracy(top_k=(1, 5, 10), views=views, device='cpu')
    want = {1: 0, 5: 0, 10: 0}
    seen = 0
    for B in (1, 7, 64):
        logits = torch.randn(B * views, C, generator=gen)
        labels = torch.randint(0, C, (B,), generator=gen)
        logits[torch.arange(B) * views, labels] += 2.5                  # some clips rank their label high
        probs = acc.update(logits, labels, want_probs=True)
        ref, ref_probs = _topk_reference(logits, labels, views, (1, 5, 10))
        assert (probs - ref_probs).abs().max() < 1e-6
        for k in want:
            want[k] += ref[k]
        seen += B
    got = acc.compute()
    assert got == {k: want[k] / seen for k in want}
    acc.reset()
    assert all(v != v for v in acc.compute().values())                   # NaN: nothing seen since the reset


def test_topk_twin_constructed_ties(emu):
    """Ties with the label do not push it down: rank = classes strictly above it."""
    from videotransformer_pytorch_b200.metrics import TopKAccuracy
    C = 10
    logits = torch.zeros(4, C)
    labels = torch.tensor([3, 0, 9, 5])
    # clip 0: all equal -> rank 0.  clip 1: two classes above the label, three tied with it -> rank 2
    logits[1, 0] = 1.0
    logits[1, [4, 5]] = 2.0
    logits[1, [6, 7, 8]] = 1.0
    # clip 2: label above everything -> rank 0.  clip 3: every other class above -> rank 9
    logits[2, 9] = 5.0
    logits[3] = 1.0
    logits[3, 5] = 0.0
    acc = TopKAccuracy(top_k=(1, 2, 3, 10), device='cpu')
    acc.update(logits, labels)
    assert acc.compute() == {1: 2 / 4, 2: 2 / 4, 3: 3 / 4, 10: 4 / 4}
    # where no tie touches the label the torch test step agrees
    ref, _ = _topk_reference(logits[[2, 3]], labels[[2, 3]], 1, (1, 2, 3, 10))
    assert ref == {1: 1, 2: 1, 3: 1, 10: 2}


def test_metric_updates_inside_restored_after_leave_no_trace(emu):
    """What GraphedForward's warm-up relies on: counters return to their state before the block, including a metric
    whose counters the block allocated."""
    from videotransformer_pytorch_b200.metrics import TopKAccuracy, restored_after
    logits, labels = torch.randn(4, 10), torch.tensor([1, 2, 3, 4])
    seen, fresh = TopKAccuracy(top_k=(1, 5), device='cpu'), TopKAccuracy(top_k=(1, 5))
    seen.update(logits, labels)
    before = seen.compute()
    with restored_after():
        for _ in range(2):
            seen.update(logits, labels)
            fresh.update(logits, labels)
    assert seen.compute() == before
    assert all(v != v for v in fresh.compute().values())           # nothing seen
    fresh.update(logits, labels)
    assert fresh.compute() == before


def _tiny_timesformer():
    from videotransformer_pytorch_b200 import TimeSformer
    torch.manual_seed(0)
    m = TimeSformer(num_frames=4, img_size=32, patch_size=16, embed_dims=64, num_heads=2, num_transformer_layers=2)
    with torch.no_grad():
        for n, p in m.named_parameters():
            if 'temporal_fc' in n:
                p.normal_(std=0.05)
    return m


@pytest.mark.parametrize('table', ['emu', 'emu_eval'])
def test_inference_mode_between_training_steps(table):
    """An eval forward under torch.inference_mode() (Lightning's default for validation), then a training step, then eval
    again: the cached index maps and weight shadows made under inference mode must not reach autograd."""
    from videotransformer_pytorch_b200 import _lib, ops
    old = _lib.K
    _lib.K = EmuKernels(exact=True, inference_forms=table == 'emu_eval')
    try:
        ops.token_maps.cache_clear()
        ops.frame_maps.cache_clear()
        m = _tiny_timesformer()
        x = torch.randn(2, 4, 3, 32, 32)
        m.eval()
        with torch.inference_mode():
            y0 = m(x)
        m.train()
        m(x).sum().backward()
        assert all(p.grad is not None for p in m.parameters())
        m.eval()
        with torch.inference_mode():
            y1 = m(x)
        assert torch.equal(y0, y1)
    finally:
        _lib.K = old


def test_linear_probe_head_gradients_match():
    """linear_prob (model_trainer.py:198-201): backbone under no_grad in eval mode, only the head trained.  The head's
    gradients are the same whether the backbone took the forward-only path or the saving forward."""
    from videotransformer_pytorch_b200 import _lib, cross_entropy
    from videotransformer_pytorch_b200.transformer import ClassificationHead
    m = _tiny_timesformer().eval()
    head = ClassificationHead(num_classes=10, in_channels=64)
    x = torch.randn(3, 4, 3, 32, 32)
    labels = torch.tensor([1, 7, 3])
    old = _lib.K
    grads = []
    try:
        for table in (EmuKernels(exact=True, inference_forms=True), EmuKernels(exact=True)):
            _lib.K = table
            head.zero_grad(set_to_none=True)
            with torch.no_grad():
                f = m(x)
            cross_entropy(head(f), labels).backward()
            grads.append([p.grad.clone() for p in head.parameters()])
            if table.inference_forms:
                assert any(c[-1] == 'gelu_h' for c in table.calls if c[0] == 'gemm')
    finally:
        _lib.K = old
    assert all(torch.equal(a, b) for a, b in zip(*grads))
    assert all(p.grad is None for p in m.parameters())
