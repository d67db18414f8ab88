"""CUDA-graph capture of one training step (forward + backward [+ gradient all-reduce]), and of one forward alone
(`GraphedForward`: validation / test steps).

A TimeSformer-B step is ~850 kernel launches of 5-150 us each; issued one by one from Python they make the
step launch-bound long before the kernels are.  `GraphedTrainStep` records the whole step once and replays
it with a single launch; per replay the host only
  * draws the DropPath masks on the CPU default generator, in the reference's order and shapes
    (transformer.py:34-42 — keeps bit-parity of the masks with an eager reference run under the same seed),
    and ships them in ONE pinned host->device copy into a static mask arena the captured kernels read;
  * copies the new batch into the static input buffers.
bf16 weight shadows are re-cast from the fp32 parameters *inside* the graph, so optimizer updates between
replays are picked up.  Gradients land in static `.grad` tensors (or in the `GradientBuckets` flat buffers,
whose NCCL all-reduces are captured on their side stream and overlap the backward).
With `optimizer=` (optim.FusedSGD / FusedAdamW) the graph also records the per-parameter clip norms and the update after
the backward, so one replay is the whole training iteration; the optimizer's per-step values (lr, weight decay, bias
corrections) are refilled from its param_groups with one more copy before each replay.
"""
from __future__ import annotations

from typing import Callable, Optional, Sequence

import torch

from . import metrics, ops


class MaskArena:
    """Static device buffer for per-step DropPath factors + the recipe to refill it."""

    def __init__(self, device, capacity: int = 1 << 20):
        self.device = device
        self.dev = torch.ones(capacity, dtype=torch.float32, device=device)
        # pinned staging is rotated over three buffers, each guarded by an event recorded after its upload: the host may
        # run ahead of the GPU (back-to-back replays without a sync) and must not rewrite a buffer whose copy is pending
        cuda = device.type == 'cuda'
        self.hosts = [torch.ones(capacity, dtype=torch.float32).pin_memory() if cuda else torch.ones(capacity)
                      for _ in range(3 if cuda else 1)]
        self.uploaded = [torch.cuda.Event() if cuda else None for _ in self.hosts]
        self._slot = 0
        self.entries = []      # (offset, n0, keep)
        self.used = 0
        self.recording = False

    def register(self, n0: int, keep: float) -> torch.Tensor:
        off = self.used
        if off + n0 > self.dev.numel():
            raise RuntimeError('MaskArena capacity exceeded')
        self.entries.append((off, n0, keep))
        self.used += n0
        return self.dev[off:off + n0]

    def refill(self):
        """Draw this step's masks exactly like the reference does (one torch.rand((n0,1,1)) per active DropPath,
        in forward order) and upload them with one copy."""
        slot = self._slot
        self._slot = (slot + 1) % len(self.hosts)
        host, ev = self.hosts[slot], self.uploaded[slot]
        if ev is not None:
            ev.synchronize()          # no-op unless this buffer's previous upload (3 steps ago) is still in flight
        for off, n0, keep in self.entries:
            r = (keep + torch.rand((n0, 1, 1))).floor_().reshape(n0) / keep
            host[off:off + n0] = r
        if self.used:
            self.dev[:self.used].copy_(host[:self.used], non_blocking=True)
            if ev is not None:
                ev.record(torch.cuda.current_stream(self.device))


class GraphedTrainStep:
    """loss = step(*inputs): replays  `loss = loss_fn(*static_inputs); loss.backward()`  as one CUDA graph.

    loss_fn   : callable taking the input tensors and returning a scalar loss (typically an nn.Module whose
                forward computes the loss); its parameters' .grad are (re)written by every call.
    reducer   : optional ddp.GradientBuckets — the bucket all-reduces become part of the graph.
    optimizer : optional optim.FusedSGD / FusedAdamW — the graph also records `optimizer.step(clip_grad=clip_grad)` after
                the backward (and after the bucket all-reduces), and a call returns `(loss, total_norm)`; total_norm is
                None when clip_grad is None, as from step().  Its param_groups' lr / weight_decay may change between
                calls.  Every parameter of its table must get a gradient from this step; frozen parameters
                (requires_grad False) are never in the table.
    """

    def __init__(self, loss_fn: Callable, example_inputs: Sequence[torch.Tensor], reducer=None,
                 params: Optional[Sequence[torch.nn.Parameter]] = None, warmup: int = 3, optimizer=None,
                 clip_grad: Optional[float] = None):
        self.loss_fn = loss_fn
        self.reducer = reducer
        self.optimizer = optimizer
        dev = example_inputs[0].device
        if dev.type != 'cuda':
            raise RuntimeError('GraphedTrainStep needs CUDA tensors')
        if optimizer is not None:
            bad = [p for g in optimizer.param_groups for p in g['params'] if p.requires_grad and p.device != dev]
            if bad:
                raise RuntimeError(f'GraphedTrainStep: the optimizer has parameters on {bad[0].device}; a captured '
                                   f'optimizer step needs them on {dev}')
        self.static_inputs = [t.clone() for t in example_inputs]
        if params is None:
            params = list(loss_fn.parameters()) if isinstance(loss_fn, torch.nn.Module) else []
        self.params = [p for p in params if p.requires_grad]
        self.arena = MaskArena(dev)
        opt_params = None
        if optimizer is not None:
            opt_params = optimizer.prepare_capture(clip_grad)
            known = {id(p) for p in self.params}
            if any(id(p) not in known for p in opt_params):
                raise RuntimeError('GraphedTrainStep: an optimizer parameter gets no gradient from this step (pass it in '
                                   '`params`, or freeze it)')

        # warm-up and capture share one side stream: autograd's AccumulateGrad nodes are bound to the stream
        # they were created on, and a node bound to a non-capturing stream would run outside the graph
        side = torch.cuda.Stream(device=dev)
        self._stream = side
        side.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(side):
            for _ in range(warmup):          # eager warm-up: lazy kernel attributes, index maps, allocator
                self._zero()
                loss_fn(*self.static_inputs).backward()
                if reducer is not None:
                    reducer.finish()
        torch.cuda.current_stream(dev).wait_stream(side)
        torch.cuda.synchronize(dev)

        from . import _lib
        self.graph = torch.cuda.CUDAGraph()
        launches_before = _lib.launch_count()
        self._zero(set_to_none=True)
        ops.set_mask_arena(self.arena)
        self.arena.recording = True
        try:
            with torch.cuda.graph(self.graph, stream=side):
                self.static_loss = loss_fn(*self.static_inputs)
                # torch.autograd.grad instead of .backward(): the gradients come back as plain tensors produced by
                # captured kernels.  (.backward() would route them through per-parameter AccumulateGrad nodes, which
                # are bound to the stream they were first created on and may execute outside the capture.)
                if reducer is None:
                    # the gradients are allocated in the graph's private pool, so every replay rewrites the same tensors
                    grads = torch.autograd.grad(self.static_loss, self.params)
                else:
                    # per-parameter tensor hooks fire as soon as a gradient is final: weight gradients are written by
                    # their GEMM straight into the flat buckets, the rest is copied there, and completed buckets are
                    # all-reduced on the side stream while backward continues
                    grads = reducer.backward_into_buckets(self.static_loss, self.params)
                if optimizer is not None:
                    # after the backward; with a reducer, backward_into_buckets has already made this stream wait for
                    # every bucket's all-reduce (GradientBuckets.finish)
                    self.static_total_norm = optimizer.launch_captured()
        finally:
            self.arena.recording = False
            ops.set_mask_arena(None)
        # drop the captured autograd graph (its kernels are recorded; keeping the Python graph alive would pin
        # AccumulateGrad nodes to the capture stream for later eager steps)
        self.static_loss = self.static_loss.detach()
        # libvt_b200 kernels recorded in the graph == launched by every replay
        self.kernels_per_replay = _lib.launch_count() - launches_before
        if reducer is None:
            self.static_grads = [g.detach() for g in grads]
            for p_, g_ in zip(self.params, self.static_grads):
                p_.grad = g_                                             # rewritten in place by every replay
        if optimizer is not None:
            # the update reads the graph's own gradients: the static tensors, or the bucket views
            by_id = {id(p): g for p, g in zip(self.params, self.static_grads)} if reducer is None else \
                {id(p): reducer._view[p] for p in self.params}
            optimizer.capture_ready([by_id[id(p)] for p in opt_params])
            torch.cuda.synchronize(dev)

    def _zero(self, set_to_none=True):
        if self.reducer is not None:
            self.reducer.zero_grad()
        else:
            for p in self.params:
                p.grad = None

    def __call__(self, *inputs):
        if self.optimizer is not None:
            self.optimizer.refill()       # first: it refuses a changed parameter list before anything is issued
        for dst, src in zip(self.static_inputs, inputs):
            if dst.data_ptr() != src.data_ptr():
                dst.copy_(src, non_blocking=True)
        self.arena.refill()
        if self.reducer is not None:
            self.reducer.reset_counters()
        self.graph.replay()
        if self.reducer is None:
            for p_, g_ in zip(self.params, self.static_grads):
                if p_.grad is not g_:
                    p_.grad = g_
        if self.optimizer is not None:
            self.optimizer.advance()
            return self.static_loss, self.static_total_norm
        return self.static_loss


class _NoMasks:
    """Mask arena of GraphedForward: a forward that would draw DropPath masks (training mode) is refused."""
    recording = True

    def register(self, n0: int, keep: float):
        raise RuntimeError('GraphedForward: the forward draws DropPath masks; put the model in eval mode')


class GraphedForward:
    """out = fwd(*inputs): replays  `with torch.no_grad(): out = fn(*static_inputs)`  as one CUDA graph.

    For evaluation: the model must be in eval mode (a captured forward that draws DropPath masks is refused).  The module
    forwards take their forward-only form under no_grad (ops.run), and the bf16 weight shadows are re-cast from the fp32
    parameters inside the graph, so training steps between two replays are picked up.  `fn` may also update device-side
    metrics (metrics.TopKAccuracy.update) from its inputs; those launches are replayed with the rest.  The eager warm-up
    runs on the example inputs leave those metrics as they found them, so after construction they count the replayed
    batches only.  The returned output is a static tensor, rewritten by the next replay.
    """

    def __init__(self, fn: Callable, example_inputs: Sequence[torch.Tensor], warmup: int = 2):
        self.fn = fn
        dev = example_inputs[0].device
        if dev.type != 'cuda':
            raise RuntimeError('GraphedForward needs CUDA tensors')
        self.static_inputs = [t.clone() for t in example_inputs]
        side = torch.cuda.Stream(device=dev)
        from . import _lib
        ops.set_mask_arena(_NoMasks())
        try:
            side.wait_stream(torch.cuda.current_stream(dev))
            with torch.cuda.stream(side), torch.no_grad(), metrics.restored_after():
                for _ in range(max(warmup, 1)):  # eager warm-up: kernel attributes, index maps, allocator, metric counters
                    fn(*self.static_inputs)
            torch.cuda.current_stream(dev).wait_stream(side)
            torch.cuda.synchronize(dev)
            self.graph = torch.cuda.CUDAGraph()
            launches_before = _lib.launch_count()
            with torch.cuda.graph(self.graph, stream=side), torch.no_grad():
                self.static_output = fn(*self.static_inputs)
        finally:
            ops.set_mask_arena(None)
        # libvt_b200 kernels recorded in the graph == launched by every replay
        self.kernels_per_replay = _lib.launch_count() - launches_before

    def __call__(self, *inputs):
        for dst, src in zip(self.static_inputs, inputs):
            if dst.data_ptr() != src.data_ptr():
                dst.copy_(src, non_blocking=True)
        self.graph.replay()
        return self.static_output
