"""Host side of the capturable optimizer step, on the CPU: the per-step arena (lr * lr_scale and weight decay per tensor in
table order, the hyper scalars, the three rotating staging buffers), and on the CPU kernel table the launch path a CUDA
graph records (hyper block) against the eager step (scalar fields), bit for bit over a schedule.  Capturing the graph
needs CUDA; tests/test_gpu_graph_optim.py covers it."""
import math

import pytest
import torch

from tests.emu_optim_hyper import f32
from tests.test_optim_host import make_params


@pytest.fixture
def hyper_emu():
    """the CPU kernel table with the vt_opt_params scalar contract (tests/emu_optim_hyper.py)"""
    from tests.emu_optim_hyper import HyperEmuKernels
    from videotransformer_pytorch_b200 import _lib
    old = _lib.K
    _lib.K = HyperEmuKernels(exact=True)
    yield _lib.K
    _lib.K = old


def groups(ps):
    return [{'params': [ps[0], ps[2]], 'weight_decay': 0.0, 'lr_scale': 0.5},
            {'params': [ps[1], ps[3]]},
            {'params': [ps[4]], 'weight_decay': 0.125, 'lr_scale': 0.25}]


def make(kind, ps):
    from videotransformer_pytorch_b200.optim import FusedAdamW, FusedSGD
    if kind == 'sgd':
        return FusedSGD(groups(ps), lr=0.05, momentum=0.9, nesterov=True, weight_decay=0.05)
    return FusedAdamW(groups(ps), lr=1e-2, betas=(0.9, 0.999), weight_decay=0.05)


@pytest.mark.parametrize('kind', ['sgd', 'adamw'])
def test_arena_packs_table_order_and_scalars(hyper_emu, kind):
    from videotransformer_pytorch_b200 import _lib
    from videotransformer_pytorch_b200.optim import HyperArena
    ps = make_params(0)
    ps[3].requires_grad_(False)                       # frozen: not in the table, not in the arena
    opt = make(kind, ps)
    for p in ps:
        p.grad = torch.ones_like(p)
    tab_params = opt.prepare_capture(clip_grad=0.3)
    order = [0, 2, 1, 4]
    assert [id(p) for p in tab_params] == [id(ps[i]) for i in order]
    arena = opt._cap['arena']
    n = len(order)
    assert arena.dev.numel() == 2 * n + _lib.OPT_HYPER_SIZE
    opt.param_groups[1]['lr'] = 0.03
    opt._steps = 4
    opt.refill()
    lr = [0.05 * 0.5, 0.05 * 0.5, 0.03, 0.05 * 0.25] if kind == 'sgd' else [1e-2 * 0.5, 1e-2 * 0.5, 0.03, 1e-2 * 0.25]
    wd = [0.0, 0.0, 0.05, 0.125]
    assert arena.lr.tolist() == [f32(v) for v in lr]
    assert arena.wd.tolist() == [f32(v) for v in wd]
    h = arena.hyper.tolist()
    assert h[_lib.OPT_HYPER['clip']] == f32(0.3)
    if kind == 'sgd':
        assert h[_lib.OPT_HYPER['first_step']] == 0.0
        assert h[_lib.OPT_HYPER['bc1']] == h[_lib.OPT_HYPER['bc2']] == 0.0
    else:
        assert h[_lib.OPT_HYPER['bc1']] == f32(1.0 - 0.9 ** 5)
        assert h[_lib.OPT_HYPER['bc2']] == f32(1.0 - 0.999 ** 5)
        assert h[_lib.OPT_HYPER['first_step']] == 0.0
    assert h[-1] == 0.0                                # the spare slot
    opt._steps = 0
    opt.refill()
    if kind == 'sgd':
        assert arena.hyper[_lib.OPT_HYPER['first_step']] == 1.0
    else:
        assert arena.hyper[_lib.OPT_HYPER['bc1']] == f32(1.0 - 0.9)
    # the arena alone: three staging buffers used in turn, each holding what its refill packed
    a = HyperArena(2, torch.device('cpu'))
    assert len(a.hosts) == 3 and len({h.data_ptr() for h in a.hosts}) == 3
    slots = [a.refill([0.1 * k, 0.2], [0.0, 0.01 * k], {'clip': k}) for k in range(7)]
    assert slots == [0, 1, 2, 0, 1, 2, 0]
    for k in (4, 5, 6):
        assert a.hosts[slots[k]].tolist()[:5] == [f32(0.1 * k), f32(0.2), 0.0, f32(0.01 * k), float(k)]
    assert torch.equal(a.dev, a.hosts[0])


@pytest.mark.parametrize('kind', ['sgd', 'adamw'])
@pytest.mark.parametrize('clip', [None, 1.3])
def test_hyper_block_launch_equals_scalar_launch(hyper_emu, kind, clip):
    """The eager step (scalars as kernel arguments) and the launch path a graph records (scalars from the arena), on the
    CPU kernel table, over a schedule that changes lr and weight decay every step: the same bits."""
    pe, pc = make_params(1), make_params(1)
    oe, oc = make(kind, pe), make(kind, pc)

    def grads(step, ps):
        g = torch.Generator().manual_seed(300 + step)
        for p in ps:
            p.grad = torch.randn(p.shape, generator=g) * (3.0 if step % 2 else 0.05)

    def sched(opt, step):
        for i, gr in enumerate(opt.param_groups):
            gr['lr'] = (0.05 if kind == 'sgd' else 1e-2) * 0.5 * (1 + math.cos(math.pi * step / 6))
            if i == 1:
                gr['weight_decay'] = 0.05 + 0.01 * step

    grads(0, pc)
    tab_params = oc.prepare_capture(clip)
    oc.capture_ready([p.grad for p in tab_params])
    for step in range(6):
        grads(step, pe), grads(step, pc)
        sched(oe, step), sched(oc, step)
        te = oe.step(clip_grad=clip)
        oc.refill()
        tc = oc.launch_captured()
        oc.advance()
        if clip is None:
            assert te is None and tc is None
        else:
            assert torch.equal(te, tc)
        for a, b in zip(pe, pc):
            assert torch.equal(a.detach(), b.detach()), step
        for sa, sb in zip(oe._tab.state, oc._tab.state):
            for a, b in zip(sa, sb):
                assert torch.equal(a, b)
    assert oc._steps == oe._steps == 6 and float(oc.state[pc[0]]['step']) == 6.0


def test_capture_state_refuses_changes(hyper_emu):
    import copy
    ps = make_params(2)
    opt = make('adamw', ps)
    for p in ps:
        p.grad = torch.ones_like(p)
    tab_params = opt.prepare_capture(0.5)
    opt.capture_ready([p.grad for p in tab_params])
    with pytest.raises(RuntimeError, match='captured'):
        opt.add_param_group({'params': [torch.nn.Parameter(torch.zeros(3))]})
    with pytest.raises(RuntimeError, match='closure'):
        opt.step(closure=lambda: 0.0)
    ps[1].requires_grad_(False)
    with pytest.raises(RuntimeError, match='parameter list changed'):
        opt.refill()
    ps[1].requires_grad_(True)
    opt.param_groups[0]['betas'] = (0.8, 0.999)
    with pytest.raises(RuntimeError, match='betas'):
        opt.refill()
    opt.param_groups[0]['betas'] = (0.9, 0.999)
    opt.refill()
    # load_state_dict copies into the live state tensors and takes the checkpoint's step count
    sd = copy.deepcopy(opt.state_dict())
    for i in sd['state']:
        sd['state'][i]['exp_avg'].fill_(float(i) + 0.5)
        sd['state'][i]['step'] = torch.tensor(7.0)
    live = [b for slot in opt._tab.state for b in slot]
    opt.load_state_dict(sd)
    assert all(a is b for a, b in zip(live, [b for slot in opt._tab.state for b in slot]))
    assert opt._steps == 7 and all(float(opt.state[p]['step']) == 7.0 for p in ps)
    assert all(opt.state[p]['exp_avg'] is b for p, b in zip(tab_params, opt._tab.state[0]))
    assert float(opt._tab.state[0][0][0]) == 0.5
    sd['state'][0]['exp_avg_sq'] = sd['state'][0]['exp_avg_sq'][:-1]
    with pytest.raises(ValueError, match='shape'):
        opt.load_state_dict(sd)
