"""GradientBuckets on CPU with the gloo backend, world_size 2 (host-side logic of the N>1 path)."""
import os
import socket

import torch
import torch.distributed as dist
import torch.multiprocessing as mp


def _free_port():
    s = socket.socket(); s.bind(('127.0.0.1', 0)); p = s.getsockname()[1]; s.close(); return p


def _worker(rank, world, port, q):
    os.environ['MASTER_ADDR'] = '127.0.0.1'
    os.environ['MASTER_PORT'] = str(port)
    dist.init_process_group('gloo', rank=rank, world_size=world)
    from videotransformer_pytorch_b200.ddp import GradientBuckets
    torch.manual_seed(rank)          # different init per rank: the constructor must broadcast rank 0's values
    net = torch.nn.Sequential(torch.nn.Linear(16, 32), torch.nn.GELU(), torch.nn.Linear(32, 8), torch.nn.Linear(8, 4))
    red = GradientBuckets(net, bucket_bytes=64)          # tiny buckets -> several of them
    assert len(red.buckets) >= 3
    w0 = [p.detach().clone() for p in net.parameters()]
    for step in range(2):
        red.zero_grad()
        g = torch.Generator().manual_seed(100 * step + rank)
        x = torch.randn(5, 16, generator=g)
        net(x).square().mean().backward()
        red.finish()
    grads = [p.grad.detach().clone() for p in net.parameters()]
    # every p.grad must still be a view of its flat bucket
    for p in net.parameters():
        assert any(p.grad.data_ptr() >= b.data_ptr() and p.grad.data_ptr() < b.data_ptr() + b.numel() * 4 for b in red.buckets)
    q.put((rank, [w.numpy() for w in w0], [g.numpy() for g in grads]))
    dist.barrier()
    dist.destroy_process_group()


def test_gradient_buckets_average_across_ranks():
    ctx = mp.get_context('spawn')
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = sorted([q.get(timeout=120) for _ in procs], key=lambda t: t[0])
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    (r0, w0, g0), (r1, w1, g1) = res
    import numpy as np
    for a, b in zip(w0, w1):
        assert np.array_equal(a, b)                      # parameters broadcast from rank 0
    for a, b in zip(g0, g1):
        assert np.allclose(a, b, atol=1e-7)              # identical averaged gradients on both ranks
    # reference: same net, mean of the two ranks' local gradients of the last step
    torch.manual_seed(0)
    net = torch.nn.Sequential(torch.nn.Linear(16, 32), torch.nn.GELU(), torch.nn.Linear(32, 8), torch.nn.Linear(8, 4))
    ref = None
    for rank in range(2):
        for p in net.parameters():
            p.grad = None
        g = torch.Generator().manual_seed(100 * 1 + rank)
        net(torch.randn(5, 16, generator=g)).square().mean().backward()
        cur = [p.grad.clone() for p in net.parameters()]
        ref = cur if ref is None else [a + b for a, b in zip(ref, cur)]
    for a, r in zip(g0, ref):
        assert np.allclose(a, (r / 2).numpy(), atol=1e-6)


def _train_worker(rank, world, port, q):
    """Two data-parallel ranks: bucketed gradient mean + fused clip/SGD step (kernel table = CPU emulation)."""
    os.environ['MASTER_ADDR'] = '127.0.0.1'
    os.environ['MASTER_PORT'] = str(port)
    dist.init_process_group('gloo', rank=rank, world_size=world)
    from tests.emu_kernels import EmuKernels
    from videotransformer_pytorch_b200 import _lib
    from videotransformer_pytorch_b200.ddp import GradientBuckets
    from videotransformer_pytorch_b200.optim import FusedSGD
    _lib.K = EmuKernels(exact=True)
    torch.manual_seed(7)
    net = torch.nn.Sequential(torch.nn.Linear(16, 32), torch.nn.GELU(), torch.nn.Linear(32, 4))
    red = GradientBuckets(net, bucket_bytes=256)
    opt = FusedSGD(net.parameters(), lr=0.1, momentum=0.9, nesterov=True, weight_decay=1e-3)
    norms = []
    for step in range(3):
        red.zero_grad()
        g = torch.Generator().manual_seed(10 * step + rank)
        net(torch.randn(6, 16, generator=g)).square().mean().backward()
        red.finish()
        norms.append(float(opt.step(clip_grad=0.05)))      # p.grad are views of the flat buckets
    q.put((rank, [p.detach().numpy().copy() for p in net.parameters()], norms))
    dist.barrier()
    dist.destroy_process_group()


def test_data_parallel_step_with_fused_optimizer():
    import numpy as np
    ctx = mp.get_context('spawn')
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_train_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = sorted([q.get(timeout=120) for _ in procs], key=lambda t: t[0])
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    (_, w0, n0), (_, w1, n1) = res
    for a, b in zip(w0, w1):
        assert np.allclose(a, b, atol=1e-7)                  # replicas stay in lock-step
    assert np.allclose(n0, n1, rtol=1e-6)
    # single-process reference: mean of the two ranks' gradients, reference clip flow, torch SGD
    torch.manual_seed(7)
    net = torch.nn.Sequential(torch.nn.Linear(16, 32), torch.nn.GELU(), torch.nn.Linear(32, 4))
    ref = torch.optim.SGD(net.parameters(), lr=0.1, momentum=0.9, nesterov=True, weight_decay=1e-3)
    for step in range(3):
        acc = None
        for rank in range(2):
            for p in net.parameters():
                p.grad = None
            g = torch.Generator().manual_seed(10 * step + rank)
            net(torch.randn(6, 16, generator=g)).square().mean().backward()
            cur = [p.grad.clone() for p in net.parameters()]
            acc = cur if acc is None else [a + b for a, b in zip(acc, cur)]
        for p, gsum in zip(net.parameters(), acc):
            p.grad = gsum / 2
            nrm = torch.norm(p.grad, 2)
            coef = 0.05 / (nrm + 1e-6)
            if coef < 1:
                p.grad.mul_(coef)
        ref.step()
    for a, p in zip(w0, net.parameters()):
        assert np.allclose(a, p.detach().numpy(), atol=2e-6)


def _none_grad_worker(rank, world, port, q):
    """A foreign `zero_grad(set_to_none=True)` (torch / Lightning default) between steps must not lose the exchange."""
    os.environ['MASTER_ADDR'] = '127.0.0.1'
    os.environ['MASTER_PORT'] = str(port)
    dist.init_process_group('gloo', rank=rank, world_size=world)
    from videotransformer_pytorch_b200.ddp import GradientBuckets
    torch.manual_seed(3)
    net = torch.nn.Sequential(torch.nn.Linear(16, 32), torch.nn.GELU(), torch.nn.Linear(32, 4))
    red = GradientBuckets(net, bucket_bytes=128)
    opt = torch.optim.SGD(net.parameters(), lr=0.1)
    for step in range(2):
        opt.zero_grad()                      # set_to_none=True: p.grad is no longer the bucket view
        assert all(p.grad is None for p in net.parameters())
        red._pending = [len(ps) for ps in red._bucket_params]
        g = torch.Generator().manual_seed(10 * step + rank)
        net(torch.randn(6, 16, generator=g)).square().mean().backward()
        red.finish()
        for p in net.parameters():           # re-attached to the flat buckets, holding the MEAN gradient
            assert any(b.data_ptr() <= p.grad.data_ptr() < b.data_ptr() + b.numel() * 4 for b in red.buckets)
    q.put((rank, [p.grad.detach().numpy().copy() for p in net.parameters()]))
    dist.barrier()
    dist.destroy_process_group()


def test_buckets_survive_set_to_none_zero_grad():
    import numpy as np
    ctx = mp.get_context('spawn')
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_none_grad_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = sorted([q.get(timeout=120) for _ in procs], key=lambda t: t[0])
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    (_, g0), (_, g1) = res
    torch.manual_seed(3)
    net = torch.nn.Sequential(torch.nn.Linear(16, 32), torch.nn.GELU(), torch.nn.Linear(32, 4))
    acc = None
    for rank in range(2):
        for p in net.parameters():
            p.grad = None
        g = torch.Generator().manual_seed(10 + rank)
        net(torch.randn(6, 16, generator=g)).square().mean().backward()
        cur = [p.grad.clone() for p in net.parameters()]
        acc = cur if acc is None else [a + b for a, b in zip(acc, cur)]
    for a, b, r in zip(g0, g1, acc):
        assert np.allclose(a, b, atol=1e-7)
        assert np.allclose(a, (r / 2).numpy(), atol=1e-6)


def _stock_ddp_worker(rank, world, port, q):
    """The package's modules under the stock torch DistributedDataParallel wrapper, as Lightning's DDPPlugin applies it
    to the reference (model_pretrain.py:200-204): every gradient flows through ordinary autograd, so the stock reducer's
    hooks fire.  Kernel table = CPU emulation (host logic only)."""
    os.environ['MASTER_ADDR'] = '127.0.0.1'
    os.environ['MASTER_PORT'] = str(port)
    dist.init_process_group('gloo', rank=rank, world_size=world)
    from tests.emu_kernels import EmuKernels
    from videotransformer_pytorch_b200 import TimeSformer, _lib
    _lib.K = EmuKernels(exact=True)
    cfg = dict(num_frames=2, img_size=32, patch_size=16, embed_dims=32, num_heads=2, num_transformer_layers=1)
    torch.manual_seed(5 + rank)                    # DDP broadcasts rank 0's parameters
    net = TimeSformer(**cfg).eval()
    with torch.no_grad():
        for n, p in net.named_parameters():
            if 'temporal_fc' in n:
                p.normal_(std=0.05)
    ddp = torch.nn.parallel.DistributedDataParallel(net)
    g = torch.Generator().manual_seed(50 + rank)
    x = torch.randn(2, 2, 3, 32, 32, generator=g)
    ddp(x).square().mean().backward()
    q.put((rank, {n: p.grad.detach().numpy().copy() for n, p in net.named_parameters()},
           {n: p.detach().numpy().copy() for n, p in net.named_parameters()}))
    dist.barrier()
    dist.destroy_process_group()


def test_modules_work_under_stock_distributed_data_parallel():
    import numpy as np
    from tests.emu_kernels import EmuKernels
    from videotransformer_pytorch_b200 import TimeSformer, _lib
    ctx = mp.get_context('spawn')
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_stock_ddp_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = sorted([q.get(timeout=180) for _ in procs], key=lambda t: t[0])
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    (_, g0, w0), (_, g1, w1) = res
    for n in g0:
        assert np.array_equal(w0[n], w1[n]), n
        assert np.allclose(g0[n], g1[n], atol=1e-7), n
    # single-process reference with rank 0's weights: mean of the two ranks' gradients
    old = _lib.K
    _lib.K = EmuKernels(exact=True)
    try:
        cfg = dict(num_frames=2, img_size=32, patch_size=16, embed_dims=32, num_heads=2, num_transformer_layers=1)
        net = TimeSformer(**cfg).eval()
        net.load_state_dict({k: torch.from_numpy(v) for k, v in w0.items()}, strict=False)
        acc = None
        for rank in range(2):
            for p in net.parameters():
                p.grad = None
            g = torch.Generator().manual_seed(50 + rank)
            net(torch.randn(2, 2, 3, 32, 32, generator=g)).square().mean().backward()
            cur = {n: p.grad.clone() for n, p in net.named_parameters()}
            acc = cur if acc is None else {n: acc[n] + cur[n] for n in cur}
    finally:
        _lib.K = old
    for n in g0:
        assert np.allclose(g0[n], (acc[n] / 2).numpy(), atol=1e-6, rtol=1e-5), n


def _captured_body_worker(rank, world, port, q):
    """The body of a captured data-parallel step (GradientBuckets.backward_into_buckets): weight-gradient GEMMs write into
    the bucket slices directly, everything else is copied, buckets are averaged — on the CPU emulation of the kernel table."""
    os.environ['MASTER_ADDR'] = '127.0.0.1'
    os.environ['MASTER_PORT'] = str(port)
    dist.init_process_group('gloo', rank=rank, world_size=world)
    from tests.emu_kernels import EmuKernels
    from videotransformer_pytorch_b200 import TimeSformer, _lib, ops
    from videotransformer_pytorch_b200.ddp import GradientBuckets
    _lib.K = EmuKernels(exact=True)
    cfg = dict(num_frames=2, img_size=32, patch_size=16, embed_dims=32, num_heads=2, num_transformer_layers=1)
    torch.manual_seed(9)
    net = TimeSformer(**cfg).eval()
    with torch.no_grad():
        for n, p in net.named_parameters():
            if 'temporal_fc' in n:
                p.normal_(std=0.05)
    red = GradientBuckets(net, bucket_bytes=4096)
    params = [p for p in net.parameters() if p.requires_grad]
    g = torch.Generator().manual_seed(70 + rank)
    x = torch.randn(2, 2, 3, 32, 32, generator=g)
    local = torch.autograd.grad(net(x).square().mean(), params)          # plain local gradients (no registry active)
    direct = []
    real_gemm = _lib.K.gemm

    spans = [(b.data_ptr(), b.data_ptr() + b.numel() * 4) for b in red.buckets]

    def spy(a, b, M, N, Kd, **kw):
        o = kw.get('out')                      # a GEMM whose output lies inside a bucket = a gradient written in place
        if o is not None and any(lo <= o.data_ptr() < hi for lo, hi in spans):
            direct.append((M, N))
        return real_gemm(a, b, M, N, Kd, **kw)
    _lib.K.gemm = spy
    with torch.no_grad():                      # no gradient may depend on zeroed buckets
        for p in params:
            p.grad.fill_(float('nan'))
    grads = red.backward_into_buckets(net(x).square().mean(), params)
    assert ops.GRAD_DEST is None
    aliased = sum(1 for p, gr in zip(params, grads) if gr.data_ptr() == p.grad.data_ptr())
    q.put((rank, [lg.numpy().copy() for lg in local], [p.grad.detach().numpy().copy() for p in params], len(direct), aliased))
    dist.barrier()
    dist.destroy_process_group()


def test_captured_step_body_always_writes_weight_gradients_into_buckets():
    import numpy as np
    ctx = mp.get_context('spawn')
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_captured_body_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = sorted([q.get(timeout=180) for _ in procs], key=lambda t: t[0])
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    (_, l0, b0, d0, a0), (_, l1, b1, d1, a1) = res
    assert d0 >= 7 and a0 >= 7            # qkv x2, proj x2, temporal_fc, fc1, fc2 landed in the buckets without a copy
    # (proj / temporal_fc of the temporal pass through the 768^3 GEMMs of the product-weight form)
    for x0, x1, y0, y1 in zip(l0, l1, b0, b1):
        assert np.allclose(y0, y1, atol=1e-7)                       # same averaged gradient on both ranks
        assert np.allclose(y0, (x0 + x1) / 2, atol=1e-6, rtol=1e-5)
