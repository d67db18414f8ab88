"""The training iteration as one CUDA graph: GraphedTrainStep(optimizer=FusedSGD / FusedAdamW, clip_grad=...) replays
forward, backward, the clip norms and the update, and must give the same bits as the captured forward + backward followed
by the eager opt.step(clip_grad=...), under LR and weight-decay schedules that change between steps.  -m gpu"""
import copy
import math
import os
import socket

import pytest
import torch

from tests.test_gpu_graph import Net

pytestmark = pytest.mark.gpu

STEPS = 10


def lr_lambda(step, warmup=3, total=STEPS, base_lr=1e-2, min_lr=5e-5):
    """cosine schedule with linear warm-up, as the reference's LambdaLR lambda (model_trainer.py:20-37)"""
    step += 1
    if step <= warmup:
        return float(step) / float(max(1, warmup))
    progress = min(float(step - warmup) / float(max(1, total - warmup)), 1)
    return 0.5 * (1. + math.cos(math.pi * progress)) * (1 - min_lr / base_lr) + min_lr / base_lr


def wd_update(opt, step, base=0.05, final=0.2, total=STEPS):
    """the reference's _weight_decay_update: only the second group's weight decay follows the cosine ramp"""
    for i, g in enumerate(opt.param_groups):
        if i == 1:
            g['weight_decay'] = final - (final - base) * (math.cos(math.pi * step / total) + 1) / 2


def decay_groups(module):
    """decay / no-decay groups in the shape of the reference's get_pretrain_param_groups"""
    no, yes = [], []
    for n, p in module.named_parameters():
        if p.requires_grad:
            (no if p.ndim == 1 or n.endswith('.bias') else yes).append(p)
    return [{'params': no, 'weight_decay': 0.}, {'params': yes}]


def make_opt(kind, groups):
    from videotransformer_pytorch_b200.optim import FusedAdamW, FusedSGD
    if kind == 'sgd':
        return FusedSGD(groups, lr=0.05, momentum=0.9, nesterov=True, weight_decay=0.05)
    return FusedAdamW(groups, lr=1e-2, betas=(0.9, 0.999), weight_decay=0.05)


def schedule(opt, step):
    base = getattr(opt, '_base_lrs', None)
    if base is None:
        base = opt._base_lrs = [g['lr'] for g in opt.param_groups]
    for g, b in zip(opt.param_groups, base):
        g['lr'] = b * lr_lambda(step)
    wd_update(opt, step)


def batches(n, B=2, seed=5, shape=(4, 3, 48, 48), classes=10):
    g = torch.Generator().manual_seed(seed)
    return [(torch.randn(B, *shape, generator=g).cuda(), torch.randint(0, classes, (B,), generator=g).cuda())
            for _ in range(n)]


def state_of(opt):
    return [buf.detach().clone() for slot in opt._tab.state for buf in slot]


def run_eager_arm(net, opt, data, clip, steps, start=0, reducer=None, params=None):
    """captured forward + backward, then the eager fused step"""
    from videotransformer_pytorch_b200.graph import GraphedTrainStep
    step = GraphedTrainStep(net, data[0], reducer=reducer, params=params)
    losses, norms = [], []
    for i in range(start, start + steps):
        schedule(opt, i)
        torch.manual_seed(1000 + i)
        losses.append(step(*data[i]).detach().clone())
        t = opt.step(clip_grad=clip)
        norms.append(None if t is None else t.clone())
    return losses, norms


def run_captured_arm(net, opt, data, clip, steps, start=0, reducer=None, params=None, graph=None):
    from videotransformer_pytorch_b200.graph import GraphedTrainStep
    if graph is None:
        graph = GraphedTrainStep(net, data[0], reducer=reducer, params=params, optimizer=opt, clip_grad=clip)
    losses, norms = [], []
    for i in range(start, start + steps):
        schedule(opt, i)
        torch.manual_seed(1000 + i)
        loss, t = graph(*data[i])
        losses.append(loss.detach().clone())
        norms.append(None if t is None else t.clone())
    return losses, norms, graph


def assert_same(a, b):
    assert len(a) == len(b)
    for i, (x, y) in enumerate(zip(a, b)):
        if x is None or y is None:
            assert x is None and y is None, i
        else:
            assert torch.equal(x, y), (i, float((x.float() - y.float()).abs().max()))


def median_grad_norm(net, data):
    """a clip value that clips about half of the parameters at the first step"""
    for p in net.parameters():
        p.grad = None
    torch.manual_seed(999)
    net(*data[0]).backward()
    norms = sorted(float(p.grad.norm()) for p in net.parameters() if p.grad is not None)
    for p in net.parameters():
        p.grad = None
    return norms[len(norms) // 2]


def twin_nets(factory):
    torch.manual_seed(0)
    a = factory().cuda().train()
    b = copy.deepcopy(a)
    return a, b


@pytest.mark.parametrize('kind', ['sgd', 'adamw'])
@pytest.mark.parametrize('clip', [None, 'median'])
def test_captured_iteration_bitwise_equals_eager_optimizer(kind, clip):
    data = batches(STEPS)
    ne, nc = twin_nets(Net)
    if clip == 'median':
        clip = median_grad_norm(ne, data)
    oe, oc = make_opt(kind, decay_groups(ne)), make_opt(kind, decay_groups(nc))
    le, te = run_eager_arm(ne, oe, data, clip, STEPS)
    lc, tc, graph = run_captured_arm(nc, oc, data, clip, STEPS)
    torch.cuda.synchronize()
    assert_same(lc, le)
    assert_same(tc, te)
    for (n, p), q in zip(nc.named_parameters(), ne.parameters()):
        assert torch.equal(p.detach(), q.detach()), n
    assert_same(state_of(oc), state_of(oe))
    assert oc._steps == oe._steps == STEPS
    assert float(oc.state[next(nc.parameters())]['step']) == STEPS


def test_clip_value_clips_some_parameters_but_not_all():
    """the 'median' clip of the test above really splits the parameters"""
    data = batches(1)
    net, _ = twin_nets(Net)
    clip = median_grad_norm(net, data)
    torch.manual_seed(999)
    net(*data[0]).backward()
    norms = [float(p.grad.norm()) for p in net.parameters()]
    assert any(n > clip * 1.01 for n in norms) and any(n < clip for n in norms)


def test_optimizer_adds_only_its_own_launches_to_the_replay():
    """norm2 (two kernels) with clipping, then the update"""
    from videotransformer_pytorch_b200.graph import GraphedTrainStep
    data = batches(1)
    na, nb = twin_nets(Net)
    plain = GraphedTrainStep(na, data[0])
    assert isinstance(plain(*data[0]), torch.Tensor)
    full = GraphedTrainStep(nb, data[0], optimizer=make_opt('adamw', decay_groups(nb)), clip_grad=1.0)
    noclip = GraphedTrainStep(na, data[0], optimizer=make_opt('sgd', decay_groups(na)))
    assert full.kernels_per_replay == plain.kernels_per_replay + 3
    assert noclip.kernels_per_replay == plain.kernels_per_replay + 1


def _mvit_probe():
    from videotransformer_pytorch_b200 import ClassificationHead, MaskFeat

    class MViTFinetune(torch.nn.Module):
        """MaskFeat backbone fine-tuning as the reference builds it for arch='mvit' (model_trainer.py:72-82, :199-206):
        forward_features' cls row into the classification head; the decoder is frozen, and so is the mask token, which
        forward_features does not use (the fused step updates only parameters that get a gradient)."""

        def __init__(self):
            super().__init__()
            self.model = MaskFeat(img_size=32, num_frames=8, feature_dim=216,
                                  pool_q_stride_size=[[1, 1, 2, 2], [3, 1, 2, 2]])
            for p in self.model.decoder_pred.parameters():
                p.requires_grad = False
            self.model.mask_token.requires_grad = False
            self.cls_head = ClassificationHead(10, self.model.embed_dims)

        def forward(self, x, y):
            return torch.nn.functional.cross_entropy(self.cls_head(self.model.forward_features(x)[:, 0]), y)

    return MViTFinetune


def layer_decay_groups(module, lr, weight_decay, layer_decay=0.75, num_layers=16):
    """the layer-decay groups of the reference's build_finetune_optimizer for arch='mvit' (optimizer.py:57-158): one
    group per (layer, decay / no-decay), lr = lr * scale and lr_scale = scale, scale = layer_decay ** (L - 1 - layer)"""
    L = num_layers + 2
    scales = [layer_decay ** i for i in reversed(range(L))]
    skip = module.model.no_weight_decay_keywords()

    def layer_of(name):
        n = name.replace('mvit.', '').replace('model.', '')
        if n == 'mask_token' or n.startswith('patch_embed') or n.startswith('cls_positional_encoding'):
            return 0
        if n.startswith('blocks'):
            return int(n.split('.')[1]) + 1
        return L - 1

    groups = {}
    for name, p in module.named_parameters():
        if not p.requires_grad:
            continue
        nd = p.ndim == 1 or name.endswith('.bias') or any(k in name for k in skip)
        lid = layer_of(name)
        key = f'layer_{lid}_{"no_decay" if nd else "decay"}'
        if key not in groups:
            groups[key] = {'params': [], 'weight_decay': 0. if nd else weight_decay, 'lr': lr * scales[lid],
                           'lr_scale': scales[lid]}
        groups[key]['params'].append(p)
    return list(groups.values())


def test_mvit_layer_decay_groups_bitwise_equal_eager():
    from videotransformer_pytorch_b200.optim import FusedAdamW
    factory = _mvit_probe()
    data = batches(6, B=2, shape=(8, 3, 32, 32))
    ne, nc = twin_nets(factory)
    mk = lambda n: FusedAdamW(layer_decay_groups(n, 1e-3, 0.05), lr=1e-3, weight_decay=0.05)
    oe, oc = mk(ne), mk(nc)
    assert len(oe.param_groups) > 4 and len({g['lr_scale'] for g in oe.param_groups}) > 4
    frozen = {id(p) for p in nc.model.decoder_pred.parameters()} | {id(nc.model.mask_token)}
    le, te = run_eager_arm(ne, oe, data, 1.0, 6)
    lc, tc, _ = run_captured_arm(nc, oc, data, 1.0, 6)
    assert not frozen & {id(p) for p in oc._tab.params}
    torch.cuda.synchronize()
    assert_same(lc, le)
    assert_same(tc, te)
    for (n, p), q in zip(nc.named_parameters(), ne.parameters()):
        assert torch.equal(p.detach(), q.detach()), n
    assert_same(state_of(oc), state_of(oe))


@pytest.mark.parametrize('kind', ['sgd', 'adamw'])
def test_resume_from_state_dict_bitwise(kind):
    data = batches(STEPS)
    ref, part = twin_nets(Net)
    o_ref = make_opt(kind, decay_groups(ref))
    l_ref, t_ref, _ = run_captured_arm(ref, o_ref, data, 0.5, STEPS)
    # five captured steps, checkpoint, then a new model / optimizer / graph resumes
    o_part = make_opt(kind, decay_groups(part))
    l_a, t_a, _ = run_captured_arm(part, o_part, data, 0.5, 5)
    torch.cuda.synchronize()
    sd_model = copy.deepcopy(part.state_dict())
    sd_opt = copy.deepcopy(o_part.state_dict())
    base = o_part._base_lrs
    resumed = Net().cuda().train()
    resumed.load_state_dict(sd_model)
    o_res = make_opt(kind, decay_groups(resumed))
    o_res.load_state_dict(copy.deepcopy(sd_opt))
    o_res._base_lrs = base
    l_b, t_b, _ = run_captured_arm(resumed, o_res, data, 0.5, 5, start=5)
    # the same checkpoint loaded into an optimizer whose graph is already captured: copied into the graph's tensors
    late = Net().cuda().train()
    late.load_state_dict(sd_model)
    o_late = make_opt(kind, decay_groups(late))
    o_late._base_lrs = base
    from videotransformer_pytorch_b200.graph import GraphedTrainStep
    g_late = GraphedTrainStep(late, data[0], optimizer=o_late, clip_grad=0.5)
    live = state_of(o_late)
    ptrs = [b.data_ptr() for slot in o_late._tab.state for b in slot]
    o_late.load_state_dict(copy.deepcopy(sd_opt))
    assert [b.data_ptr() for slot in o_late._tab.state for b in slot] == ptrs
    assert o_late._steps == 5 and float(o_late.state[next(late.parameters())]['step']) == 5
    assert not all(torch.equal(a, b) for a, b in zip(live, state_of(o_late)))
    l_c, t_c, _ = run_captured_arm(late, o_late, data, 0.5, 5, start=5, graph=g_late)
    torch.cuda.synchronize()
    assert_same(l_a + l_b, l_ref)
    assert_same(t_a + t_b, t_ref)
    assert_same(l_a + l_c, l_ref)
    assert_same(t_a + t_c, t_ref)
    for p, q, r in zip(resumed.parameters(), late.parameters(), ref.parameters()):
        assert torch.equal(p.detach(), r.detach()) and torch.equal(q.detach(), r.detach())
    assert_same(state_of(o_res), state_of(o_ref))
    assert_same(state_of(o_late), state_of(o_ref))
    # a checkpoint that does not fit the captured tensors is refused
    bad = copy.deepcopy(sd_opt)
    first = bad['param_groups'][0]['params'][0]
    name = 'momentum_buffer' if kind == 'sgd' else 'exp_avg'
    bad['state'][first][name] = bad['state'][first][name].double()
    with pytest.raises(ValueError, match='captured'):
        o_late.load_state_dict(bad)
    bad['state'][first][name] = torch.zeros(3, device='cuda')
    with pytest.raises(ValueError, match='captured'):
        o_late.load_state_dict(bad)


class LinearProbe(torch.nn.Module):
    """eval_metrics='linear_prob' (model_trainer.py:195-199): the backbone runs under no_grad in eval mode, only the head
    trains"""

    def __init__(self):
        super().__init__()
        self.net = Net()

    def forward(self, x, y):
        with torch.no_grad():
            self.net.model.eval()
            feats = self.net.model(x)
        return torch.nn.functional.cross_entropy(self.net.head(feats), y)


@pytest.mark.parametrize('kind', ['sgd', 'adamw'])
def test_linear_probe_captured_equals_eager(kind):
    data = batches(6)
    ne, nc = twin_nets(LinearProbe)
    oe = make_opt(kind, decay_groups(ne.net.head))
    oc = make_opt(kind, decay_groups(nc.net.head))
    le, te = run_eager_arm(ne, oe, data, 0.05, 6, params=list(ne.net.head.parameters()))
    lc, tc, _ = run_captured_arm(nc, oc, data, 0.05, 6, params=list(nc.net.head.parameters()))
    torch.cuda.synchronize()
    assert_same(lc, le)
    assert_same(tc, te)
    for p, q in zip(nc.parameters(), ne.parameters()):
        assert torch.equal(p.detach(), q.detach())
    assert len(oc._tab.params) == len(list(nc.net.head.parameters()))


def test_refusals():
    from videotransformer_pytorch_b200.graph import GraphedTrainStep
    from videotransformer_pytorch_b200.optim import FusedSGD
    data = batches(3)
    net, _ = twin_nets(Net)
    opt = make_opt('sgd', decay_groups(net))
    graph = GraphedTrainStep(net, data[0], optimizer=opt, clip_grad=1.0)
    graph(*data[0])
    extra = torch.nn.Parameter(torch.zeros(4, device='cuda'))
    with pytest.raises(RuntimeError, match='captured'):
        opt.add_param_group({'params': [extra]})
    with pytest.raises(RuntimeError, match='closure'):
        opt.step(closure=lambda: 0.0)
    p0 = next(net.parameters())
    p0.requires_grad_(False)
    with pytest.raises(RuntimeError, match='parameter list changed'):
        graph(*data[1])
    p0.requires_grad_(True)
    with pytest.raises(RuntimeError, match='already captured'):
        GraphedTrainStep(net, data[0], optimizer=opt)
    graph(*data[2])                                   # the unchanged list replays again
    cpu = Net().train()
    with pytest.raises(RuntimeError, match='optimizer'):
        GraphedTrainStep(cpu, data[0], optimizer=FusedSGD(cpu.parameters(), lr=0.1))


def _free_port():
    s = socket.socket()
    s.bind(('127.0.0.1', 0))
    p = s.getsockname()[1]
    s.close()
    return p


def test_gradient_buckets_world_size_one_bitwise():
    """the bucket-view gradient table: GradientBuckets in a one-process NCCL group"""
    import torch.distributed as dist
    from videotransformer_pytorch_b200.ddp import GradientBuckets
    os.environ.setdefault('MASTER_ADDR', '127.0.0.1')
    os.environ['MASTER_PORT'] = str(_free_port())
    dist.init_process_group('nccl', rank=0, world_size=1, device_id=torch.device('cuda', torch.cuda.current_device()))
    try:
        data = batches(6)
        ne, nc = twin_nets(Net)
        re_, rc = GradientBuckets(ne, bucket_bytes=1 << 18), GradientBuckets(nc, bucket_bytes=1 << 18)
        assert len(rc.buckets) > 1
        oe, oc = make_opt('adamw', decay_groups(ne)), make_opt('adamw', decay_groups(nc))
        le, te = run_eager_arm(ne, oe, data, 0.5, 6, reducer=re_)
        lc, tc, _ = run_captured_arm(nc, oc, data, 0.5, 6, reducer=rc)
        torch.cuda.synchronize()
        assert_same(lc, le)
        assert_same(tc, te)
        for p, q in zip(nc.parameters(), ne.parameters()):
            assert torch.equal(p.detach(), q.detach())
        assert_same(state_of(oc), state_of(oe))
        views = {rc._view[p].data_ptr() for p in nc.parameters()}
        assert set(oc._cap['t']['gptr'].tolist()) == views
    finally:
        dist.destroy_process_group()
