"""Data-parallel gradient exchange: bucketed all-reduce (mean) of parameter gradients over NCCL,
overlapped with the backward pass.

Replaces what PyTorch-Lightning's DDPPlugin gives the reference (model_pretrain.py:200-204,
SURVEY.md §2.2 C1): one process per GPU, full replica, one all-reduce of the gradients per step and
nothing else on the data path.  Design for NVLink 5 / NVSwitch:

  * parameters are grouped into flat fp32 buckets in *reverse registration order* (the order backward
    produces them), one bucket ~= one transformer layer (default 32 MiB), and every `p.grad` is a view
    into its bucket, so wgrad results land in the bucket without a gather copy;
  * a post-accumulate-grad hook counts ready parameters; when a bucket is complete its all-reduce is
    issued on a dedicated communication stream (ordered after the producing kernels by an event), so
    NCCL (NVLS in-switch reduction when available) runs under the remaining backward compute;
  * `finish()` makes the compute stream wait for the communication stream.

`torch.nn.parallel.DistributedDataParallel` also works with these modules (all gradients flow through
ordinary autograd); this class exists so the exchange is explicit, allocation-free per step and
measurable.  Works with the `gloo` backend on CPU tensors (tests), where the overlap degenerates to
synchronous calls.
"""
from __future__ import annotations

from typing import List

import torch
import torch.distributed as dist


class GradientBuckets:
    def __init__(self, module: torch.nn.Module, bucket_bytes: int = 32 << 20, process_group=None,
                 broadcast_parameters: bool = True):
        if not dist.is_initialized():
            raise RuntimeError('GradientBuckets needs an initialised torch.distributed process group')
        self.group = process_group
        self.world = dist.get_world_size(process_group)
        params = [p for p in module.parameters() if p.requires_grad]
        if not params:
            raise RuntimeError('module has no trainable parameters')
        self.device = params[0].device
        self.cuda = self.device.type == 'cuda'
        if broadcast_parameters:                       # DDP constructor semantics (SURVEY C2)
            with torch.no_grad():
                for p in module.parameters():
                    dist.broadcast(p.data, src=0, group=process_group)
                for b in module.buffers():
                    dist.broadcast(b.data, src=0, group=process_group)
        # bucket assignment in reverse order
        self.buckets: List[torch.Tensor] = []
        self._bucket_params: List[List[torch.nn.Parameter]] = []
        cur, cur_bytes = [], 0
        for p in reversed(params):
            cur.append(p)
            cur_bytes += p.numel() * 4
            if cur_bytes >= bucket_bytes:
                self._bucket_params.append(cur)
                cur, cur_bytes = [], 0
        if cur:
            self._bucket_params.append(cur)
        self._owner = {}
        self._view = {}
        for bi, ps in enumerate(self._bucket_params):
            # every slice starts on a 16-byte boundary (the weight-gradient GEMMs store into them by TMA); the padding
            # elements stay zero and ride along in the all-reduce
            n = sum((p.numel() + 3) // 4 * 4 for p in ps)
            flat = torch.zeros(n, dtype=torch.float32, device=self.device)
            off = 0
            for p in ps:
                p.grad = flat[off:off + p.numel()].view_as(p)
                self._view[p] = p.grad
                off += (p.numel() + 3) // 4 * 4
                self._owner[p] = bi
                p.register_post_accumulate_grad_hook(self._hook)
            self.buckets.append(flat)
        self._pending = [len(ps) for ps in self._bucket_params]
        self._arrived = [[] for _ in self._bucket_params]
        self._works = []
        self.comm_stream = torch.cuda.Stream(device=self.device) if self.cuda else None
        self.bytes_per_step = sum(b.numel() * 4 for b in self.buckets)

    # -- per step -------------------------------------------------------------------------------
    def zero_grad(self):
        """Gradients live in the buckets: zero them in place and make sure every p.grad is its bucket view again
        (a foreign zero_grad(set_to_none=True) is tolerated: see _hook)."""
        for b in self.buckets:
            b.zero_()
        for p, view in self._view.items():
            if p.grad is not view:
                p.grad = view
        self._pending = [len(ps) for ps in self._bucket_params]

    def reset_counters(self):
        """CUDA-graph replays run no Python hooks: the captured graph already contains the gradient writes and the
        all-reduces in the right order; only the host-side bookkeeping is reset."""
        self._pending = [0 for _ in self._bucket_params]

    def _hook(self, p):
        bi = self._owner[p]
        view = self._view[p]
        if p.grad is not view and (p.grad is None or p.grad.data_ptr() != view.data_ptr()):
            # something replaced p.grad (optimizer.zero_grad(set_to_none=True), Lightning's default): autograd then
            # accumulated into a fresh tensor.  Move it into the bucket and re-attach the view, otherwise the bucket
            # would be all-reduced without this rank's gradient and the optimizer would consume the unsynchronised one.
            with torch.no_grad():
                view.copy_(p.grad)
            p.grad = view
        self._pending[bi] -= 1
        if self._pending[bi] == 0:
            self._launch(bi)

    def _launch(self, bi: int):
        flat = self.buckets[bi]
        if self.world == 1:
            return
        if self.cuda:
            ready = torch.cuda.Event()
            ready.record(torch.cuda.current_stream(self.device))
            with torch.cuda.stream(self.comm_stream):
                self.comm_stream.wait_event(ready)
                dist.all_reduce(flat, op=dist.ReduceOp.AVG, group=self.group)
        else:
            dist.all_reduce(flat, op=dist.ReduceOp.SUM, group=self.group)
            flat.div_(self.world)

    def grad_ready(self, p, grad):
        """Tensor-hook entry (graph capture with torch.autograd.grad): copy one finished gradient into its bucket
        view and, when the bucket is complete, start its all-reduce on the communication stream — so the
        exchange overlaps the rest of the backward pass inside the captured graph."""
        bi = self._owner[p]
        self._arrived[bi].append((p, grad))
        self._pending[bi] -= 1
        if self._pending[bi] == 0:
            # one multi-tensor copy per bucket (not one tiny kernel per parameter), then the bucket's all-reduce
            ps = [q for q, g in self._arrived[bi] if g.data_ptr() != q.grad.data_ptr()]
            gs = [g for q, g in self._arrived[bi] if g.data_ptr() != q.grad.data_ptr()]
            if ps:
                with torch.no_grad():
                    torch._foreach_copy_([q.grad for q in ps], gs)
            self._arrived[bi] = []
            self._launch(bi)

    def backward_into_buckets(self, loss, params):
        """Backward of `loss` with the gradients landing in the flat buckets and every bucket's all-reduce issued as soon as
        it is complete (the body of a captured data-parallel step, graph.GraphedTrainStep; also usable eagerly while every
        p.grad is its bucket view, as zero_grad() leaves it).  Uses torch.autograd.grad, so nothing is ACCUMULATED:
        weight-gradient GEMMs therefore write directly into their bucket slice (ops.GRAD_DEST), other gradients are copied
        in by grad_ready().  Writing in place instead of copying measured 19.70 vs 20.00 ms per step at 2 GPUs (before the
        port to H100; not re-measured since), bucket contents equal to 8e-9 (bench.py ddp_check).  Every parameter's slice
        is overwritten in full, so the buckets need no zeroing first."""
        from . import ops
        params = list(params)
        self._pending = [len(ps) for ps in self._bucket_params]
        self._arrived = [[] for _ in self._bucket_params]
        handles = [p.register_hook(lambda g, p=p: self.grad_ready(p, g)) for p in params]
        ops.set_grad_destinations({p.data_ptr(): v for p, v in self._view.items()})
        try:
            grads = torch.autograd.grad(loss, params)
        finally:
            ops.set_grad_destinations(None)
            for h in handles:
                h.remove()
        self.finish()
        return grads

    def reduce_into_buckets(self, params, grads):
        """Graph-capture path: gradients arrive as a list (torch.autograd.grad); copy them into the flat buckets
        (p.grad stays the bucket view) and all-reduce bucket by bucket on the communication stream."""
        by_param = {id(p): g for p, g in zip(params, grads)}
        for bi, ps in enumerate(self._bucket_params):
            torch._foreach_copy_([p.grad for p in ps], [by_param[id(p)] for p in ps])
            self._pending[bi] = 0
            self._launch(bi)
        self.finish()

    def finish(self):
        """Call after backward(): the compute stream waits for all bucket reductions."""
        missing = [i for i, n in enumerate(self._pending) if n != 0]
        if missing:
            raise RuntimeError(f'buckets {missing} did not receive all gradients this step '
                               '(every parameter must get a gradient, as in the reference with '
                               'find_unused_parameters=False)')
        if self.cuda and self.world > 1:
            torch.cuda.current_stream(self.device).wait_stream(self.comm_stream)
