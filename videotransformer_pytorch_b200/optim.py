"""Fused gradient clipping + optimizer step on the sm_90a kernels (SURVEY §8f rank 1).

Drop-in for the two optimizers the reference builds (optimizer.py:33-38) and for `VideoTransformer.clip_gradients`
(model_trainer.py:155-170):

    opt = FusedSGD(param_groups, lr=..., momentum=0.9, nesterov=True, weight_decay=...)     # or FusedAdamW(...)
    total_norm = opt.step(clip_grad=0.3)        # == clip_gradients(0.3) followed by optimizer.step()

`param_groups` is whatever the reference's get_pretrain_param_groups / get_finetune_param_groups return (per-group
`weight_decay`, `lr`, optional `lr_scale`), so schedulers that rewrite group['lr'] / group['weight_decay']
(model_trainer.py:150-153) keep working.  One norm launch + one update launch replace 247 `torch.norm` launches, 247
host comparisons and the foreach optimizer kernels.  Gradients are taken from `p.grad` (plain tensors, the static
gradients of a captured step, or views of the DDP flat buckets).

Both optimizers are also capturable: `graph.GraphedTrainStep(..., optimizer=opt, clip_grad=c)` records the norm and the
update launches after the backward, and every replay then runs the whole iteration.  For that path the per-step values
(each tensor's `lr * lr_scale` and `weight_decay`, the clip value, AdamW's bias corrections `1 - beta^t` computed on the
host in double, SGD's first-step flag) live in a static device block, `HyperArena`, that the graph refills with one copy
before each replay from `param_groups` and the host step count, so LR and weight-decay schedules keep working.  The
kernels read the block through `vt_opt_params.hyper`; the eager `step()` passes the same values as kernel arguments, so a
captured and an eager step give the same bits.  Once captured, the parameter list is fixed (`add_param_group` or a
`requires_grad` flip raises), and `load_state_dict` copies into the state tensors the graph writes.
"""
from __future__ import annotations

import torch

from . import _lib

CHUNK = 1 << 16


class TensorTable:
    """Device-side description of a list of (param, grad, state...) tensors for the multi-tensor kernels.
    `state` = one list of tensors per state slot (momentum | exp_avg, exp_avg_sq), owned by the optimizer's
    torch.optim.Optimizer.state so that state_dict() / load_state_dict() round-trip them."""

    def __init__(self, params, state):
        self.params = list(params)
        dev = self.params[0].device
        self.device = dev
        rows = []
        for i, p in enumerate(self.params):
            if p.dtype != torch.float32 or not p.is_contiguous():
                raise RuntimeError('fused optimizer: parameters must be contiguous fp32')
            n = p.numel()
            for off in range(0, n, CHUNK):
                rows.append((i, min(CHUNK, n - off), off))
        # rows of {int32 tensor, int32 len, int64 offset} = 16 bytes, built as int64 pairs (little endian)
        tbl = torch.tensor([[(ln << 32) | i, off] for i, ln, off in rows], dtype=torch.int64)
        n = len(self.params)
        self.state = [list(slot) for slot in state]
        for slot in self.state:
            for p, s_ in zip(self.params, slot):
                if s_.dtype != torch.float32 or not s_.is_contiguous() or s_.device != p.device or s_.shape != p.shape:
                    raise RuntimeError('fused optimizer: state tensors must be contiguous fp32 like their parameter')
        self.t = {
            'chunks': tbl.to(dev), 'n_chunks': len(rows), 'n_tensors': n,
            'pptr': torch.tensor([p.data_ptr() for p in self.params], dtype=torch.int64, device=dev),
            'gptr': torch.zeros(n, dtype=torch.int64, device=dev),
            's1ptr': torch.tensor([s.data_ptr() for s in self.state[0]], dtype=torch.int64, device=dev),
            'norm2': torch.zeros(n, dtype=torch.float32, device=dev),
            'partials': torch.zeros(len(rows), dtype=torch.float32, device=dev),    # vt_opt_norm2: one sum per chunk
            'lr': torch.zeros(n, dtype=torch.float32, device=dev),
            'wd': torch.zeros(n, dtype=torch.float32, device=dev),
        }
        # python-side handles (used by the CPU emulation of the kernel table in tests; the CUDA path reads the pointer arrays)
        self.t['_params'], self.t['_state'] = self.params, self.state
        self.t['_grads'] = lambda: [p.grad for p in self.params]
        if len(self.state) > 1:
            self.t['s2ptr'] = torch.tensor([s.data_ptr() for s in self.state[1]], dtype=torch.int64, device=dev)
        self._gptr_host = None
        self._hp_host = None

    def bind_grads(self):
        """Refresh the gradient pointer table (eager steps allocate new .grad tensors; captured steps keep them)."""
        ptrs = []
        for p in self.params:
            g = p.grad
            if g is None:
                raise RuntimeError('fused optimizer: a parameter has no gradient (the fused step updates every tensor)')
            if g.dtype != torch.float32 or not g.is_contiguous() or g.device != p.device:
                raise RuntimeError('fused optimizer: gradients must be contiguous fp32 on the parameter device')
            ptrs.append(g.data_ptr())
        if ptrs != self._gptr_host:
            self.t['gptr'].copy_(torch.tensor(ptrs, dtype=torch.int64), non_blocking=True)
            self._gptr_host = ptrs

    def bind_hyper(self, lrs, wds):
        key = (tuple(lrs), tuple(wds))
        if key != self._hp_host:
            self.t['lr'].copy_(torch.tensor(lrs, dtype=torch.float32), non_blocking=True)
            self.t['wd'].copy_(torch.tensor(wds, dtype=torch.float32), non_blocking=True)
            self._hp_host = key


class HyperArena:
    """Static device block of one step's optimizer values: lr[n] | wd[n] | the vt_opt_params.hyper scalars, in table order,
    and the recipe to refill it (the counterpart of graph.MaskArena for the captured optimizer launches).  `refill()`
    packs the values into one of three pinned staging buffers and issues one host->device copy; each buffer is guarded
    by an event recorded after its copy, so the host may run replays ahead of the GPU without rewriting a buffer whose
    copy is still pending."""

    def __init__(self, n, device):
        self.n = n
        size = 2 * n + _lib.OPT_HYPER_SIZE
        self.dev = torch.zeros(size, dtype=torch.float32, device=device)
        self.lr, self.wd, self.hyper = self.dev[:n], self.dev[n:2 * n], self.dev[2 * n:]
        cuda = device.type == 'cuda'
        self.hosts = [torch.zeros(size, dtype=torch.float32, pin_memory=cuda) for _ in range(3)]
        self.uploaded = [torch.cuda.Event() if cuda else None for _ in self.hosts]
        self._slot = 0

    def refill(self, lrs, wds, scalars):
        """lrs / wds: per-tensor python floats in table order; scalars: {name in _lib.OPT_HYPER: value}, rounded to fp32
        here exactly as ctypes rounds the scalar fields of the eager launch"""
        slot = self._slot
        self._slot = (slot + 1) % len(self.hosts)
        host, ev = self.hosts[slot], self.uploaded[slot]
        if ev is not None:
            ev.synchronize()          # no-op unless this buffer's previous copy (three refills ago) is still in flight
        n = self.n
        host[:n] = torch.tensor(lrs, dtype=torch.float32)
        host[n:2 * n] = torch.tensor(wds, dtype=torch.float32)
        host[2 * n:] = 0.0
        for k, v in scalars.items():
            host[2 * n + _lib.OPT_HYPER[k]] = float(v)
        self.dev.copy_(host, non_blocking=True)
        if ev is not None:
            ev.record(torch.cuda.current_stream(self.dev.device))
        return slot


class _FusedBase(torch.optim.Optimizer):
    state_names = ('momentum_buffer',)       # keys in self.state[p], same names as torch.optim.SGD / AdamW
    fixed_names = ()                         # group values recorded into a captured launch as kernel arguments

    def _trainable(self):
        return [p for g in self.param_groups for p in g['params'] if p.requires_grad]

    def _hyper_lists(self):
        lrs, wds = [], []
        for g in self.param_groups:
            for p in g['params']:
                if p.requires_grad:
                    lrs.append(float(g['lr']) * float(g.get('lr_scale', 1.0)))
                    wds.append(float(g['weight_decay']))
        return lrs, wds

    def _table(self):
        tab = self._bind_table()
        tab.bind_hyper(*self._hyper_lists())
        tab.bind_grads()
        return tab

    def _bind_table(self):
        params = self._trainable()
        tab = getattr(self, '_tab', None)
        if tab is None or [id(p) for p in tab.params] != [id(p) for p in params]:
            if self._captured():
                raise RuntimeError('fused optimizer: the parameter list changed after the optimizer was captured in a '
                                   'CUDA graph (add_param_group or a requires_grad flip); build a new optimizer and graph')
            # (re)bind: the per-parameter buffers live in torch.optim.Optimizer.state, so they survive
            # state_dict()/load_state_dict() (checkpoint resume) and changes of the parameter list (add_param_group)
            had_all = True
            slots = [[] for _ in self.state_names]
            steps = 0
            for p in params:
                st = self.state[p]
                for si, name in enumerate(self.state_names):
                    buf = st.get(name)
                    if buf is None:
                        had_all = False
                        buf = torch.zeros_like(p, memory_format=torch.contiguous_format)
                    elif buf.dtype != torch.float32 or buf.device != p.device or not buf.is_contiguous():
                        buf = buf.to(device=p.device, dtype=torch.float32).contiguous()
                    st[name] = buf
                    slots[si].append(buf)
                if 'step' in st:
                    steps = max(steps, int(float(st['step'])))
            tab = self._tab = TensorTable(params, slots)
            # fresh buffers start the count at 0; restored buffers without a counter (torch.optim.SGD keeps none) are
            # past their first step
            self._steps = steps if steps > 0 else (1 if had_all else 0)
            self._step_tensor = torch.tensor(float(self._steps))
            for p in params:
                self.state[p]['step'] = self._step_tensor        # one shared host scalar (torch keeps one per tensor)
        return tab

    def _captured(self):
        c = getattr(self, '_cap', None)
        return c is not None and c['ready']

    def add_param_group(self, param_group):
        if self._captured():
            raise RuntimeError('fused optimizer: add_param_group after the optimizer was captured in a CUDA graph; '
                               'build a new optimizer and graph')
        super().add_param_group(param_group)

    def load_state_dict(self, state_dict):
        if self._captured():
            self._load_in_place(state_dict)
            return
        super().load_state_dict(state_dict)
        self._tab = None              # pointer tables are rebuilt from the restored self.state on the next step

    def _load_in_place(self, state_dict):
        """Captured optimizer: the graph writes the state tensors it was recorded with, so the checkpoint's values are
        copied into them (and the host step count follows the checkpoint's) instead of rebinding new tensors."""
        tab = self._tab
        saved_ids = [i for g in state_dict['param_groups'] for i in g['params']]
        params = [p for g in self.param_groups for p in g['params']]
        if len(saved_ids) != len(params):
            raise ValueError('fused optimizer: the state dict has a different number of parameters')
        index = {id(p): i for p, i in zip(params, saved_ids)}
        incoming, steps = [], 0
        for p, *bufs in zip(tab.params, *tab.state):
            st = state_dict['state'].get(index[id(p)], {})
            row = []
            for name, buf in zip(self.state_names, bufs):
                v = st.get(name)
                if not isinstance(v, torch.Tensor) or v.shape != buf.shape or v.dtype != buf.dtype:
                    raise ValueError(f'fused optimizer: state {name!r} of a captured parameter must be a {buf.dtype} '
                                     f'tensor of shape {tuple(buf.shape)}, got '
                                     f'{(v.dtype, tuple(v.shape)) if isinstance(v, torch.Tensor) else type(v).__name__}')
                row.append(v)
            incoming.append(row)
            if 'step' in st:
                steps = max(steps, int(float(st['step'])))
        with torch.no_grad():
            for row, *bufs in zip(incoming, *tab.state):
                for v, buf in zip(row, bufs):
                    buf.copy_(v, non_blocking=False)
        live = {p: {n: s_ for n, s_ in zip(self.state_names, bufs)} for p, *bufs in zip(tab.params, *tab.state)}
        super().load_state_dict(state_dict)            # param_groups (lr, weight_decay, ...) and any other state
        self._steps = steps if steps > 0 else 1        # every state buffer was restored: past the first step
        self._step_tensor.fill_(float(self._steps))
        for p, st in live.items():
            self.state[p].update(st)
            self.state[p]['step'] = self._step_tensor

    # -- the capturable launch path (graph.GraphedTrainStep(optimizer=...)) --------------------------------------------
    def prepare_capture(self, clip_grad=None):
        """Bind the table and allocate the static buffers of the captured launches.  Call before the capture; returns
        the table's parameters, whose gradients capture_ready() takes in this order."""
        if self._captured():
            raise RuntimeError('fused optimizer: already captured in a CUDA graph')
        tab = self._bind_table()
        n, dev = len(tab.params), tab.device
        t = dict(tab.t)
        t['gptr'] = torch.zeros(n, dtype=torch.int64, device=dev)       # this graph's gradients, bound by capture_ready
        t['norm2'] = torch.zeros(n, dtype=torch.float32, device=dev)
        t['partials'] = torch.zeros(tab.t['n_chunks'], dtype=torch.float32, device=dev)
        arena = HyperArena(n, dev)
        t['lr'], t['wd'], t['hyper'] = arena.lr, arena.wd, arena.hyper     # the kernels take the per-step scalars from here
        g0 = self.param_groups[0]
        self._cap = dict(tab=tab, t=t, arena=arena, clip=clip_grad, fixed={k: g0[k] for k in self.fixed_names},
                         ready=False)
        return tab.params

    @torch.no_grad()
    def launch_captured(self):
        """Issue the capturable work only: the norms (with clipping), the total norm into a tensor of the capture's pool,
        and the update reading the arena.  Returns the total norm tensor, or None without clipping (as step())."""
        c = self._cap
        total = None
        if c['clip'] is not None:
            n2 = _lib.K.opt_norm2(c['t'])
            total = n2.sum().sqrt()
        self._update_captured(c['t'], c['fixed'])
        return total

    def capture_ready(self, grads):
        """After the capture: bind the gradient pointer table once (the graph's static gradients or the bucket views, one
        per table parameter and in table order); from here on the optimizer is captured."""
        c = self._cap
        if len(grads) != len(c['tab'].params):
            raise RuntimeError('fused optimizer: one gradient per table parameter expected')
        for p, g in zip(c['tab'].params, grads):
            if g.dtype != torch.float32 or not g.is_contiguous() or g.device != p.device or g.shape != p.shape:
                raise RuntimeError('fused optimizer: gradients must be contiguous fp32 like their parameter')
        c['t']['gptr'].copy_(torch.tensor([g.data_ptr() for g in grads], dtype=torch.int64))
        c['ready'] = True

    def refill(self):
        """Before each replay: this step's lr / wd / scalars into the arena (one copy)."""
        c = self._cap
        if [id(p) for p in self._trainable()] != [id(p) for p in c['tab'].params]:
            raise RuntimeError('fused optimizer: the parameter list changed after the optimizer was captured in a '
                               'CUDA graph (add_param_group or a requires_grad flip); build a new optimizer and graph')
        g0 = self.param_groups[0]
        for k, v in c['fixed'].items():
            if g0[k] != v:
                raise RuntimeError(f'fused optimizer: {k!r} is recorded in the captured update and cannot change')
        scalars = dict(clip=float(c['clip'] or 0.0), **self._hyper_scalars())
        c['arena'].refill(*self._hyper_lists(), scalars)

    def advance(self):
        """After each replay: the host step count and the parameters' version counters, as step() leaves them."""
        self._steps += 1
        self._step_tensor.fill_(float(self._steps))
        for p in self._cap['tab'].params:
            torch.autograd.graph.increment_version(p)

    @torch.no_grad()
    def step(self, closure=None, clip_grad=None):
        """Returns the total gradient norm (sqrt of the sum of squared per-parameter norms, before clipping — what
        clip_gradients returns, model_trainer.py:169) as a device scalar when `clip_grad` is not None."""
        if closure is not None:
            if self._captured():
                raise RuntimeError('fused optimizers do not take a closure (and a captured step replays a fixed forward '
                                   'and backward: call the GraphedTrainStep instead)')
            raise RuntimeError('fused optimizers do not take a closure')
        tab = self._table()
        total = None
        if clip_grad is not None:
            n2 = _lib.K.opt_norm2(tab.t)
            total = n2.sum().sqrt()
        self._update(tab, float(clip_grad or 0.0))
        self._steps += 1
        self._step_tensor.fill_(float(self._steps))
        # the kernels wrote the parameters through raw pointers: bump the autograd version counters so everything keyed
        # on them (the bf16 weight shadows of transformer.ShadowWeights, saved-tensor checks) sees the update
        for p in tab.params:
            torch.autograd.graph.increment_version(p)
        return total


class FusedSGD(_FusedBase):
    """torch.optim.SGD(momentum, nesterov, weight_decay; dampening 0) with the reference's per-parameter clipping."""

    fixed_names = ('momentum', 'nesterov')

    def __init__(self, params, lr, momentum=0.9, nesterov=True, weight_decay=0.0):
        super().__init__(params, dict(lr=lr, momentum=momentum, nesterov=nesterov, weight_decay=weight_decay))
        if len({g['momentum'] for g in self.param_groups}) > 1 or len({g['nesterov'] for g in self.param_groups}) > 1:
            raise NotImplementedError('per-group momentum / nesterov')

    def _update(self, tab, clip):
        g0 = self.param_groups[0]
        _lib.K.opt_sgd(tab.t, clip, float(g0['momentum']), bool(g0['nesterov']), self._steps == 0)

    def _hyper_scalars(self):
        return dict(first_step=float(self._steps == 0))

    def _update_captured(self, t, fixed):
        # clip and first_step come from t['hyper']
        _lib.K.opt_sgd(t, 0.0, float(fixed['momentum']), bool(fixed['nesterov']), False)

    def momentum_buffers(self):
        return dict(zip((id(p) for p in self._tab.params), self._tab.state[0]))


class FusedAdamW(_FusedBase):
    """torch.optim.AdamW(betas, eps, weight_decay) with the reference's per-parameter clipping."""
    state_names = ('exp_avg', 'exp_avg_sq')
    fixed_names = ('betas', 'eps')

    def __init__(self, params, lr, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.01):
        super().__init__(params, dict(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay))
        if len({tuple(g['betas']) for g in self.param_groups}) > 1 or len({g['eps'] for g in self.param_groups}) > 1:
            raise NotImplementedError('per-group betas / eps')

    def _update(self, tab, clip):
        g0 = self.param_groups[0]
        b1, b2 = g0['betas']
        t = self._steps + 1
        _lib.K.opt_adamw(tab.t, clip, float(b1), float(b2), float(g0['eps']), 1.0 - b1 ** t, 1.0 - b2 ** t)

    def _hyper_scalars(self):
        # the same double-precision expressions as _update: the fp32 values in the arena are the eager kernel arguments
        b1, b2 = self.param_groups[0]['betas']
        t = self._steps + 1
        return dict(bc1=1.0 - b1 ** t, bc2=1.0 - b2 ** t)

    def _update_captured(self, t, fixed):
        # clip, bc1 and bc2 come from t['hyper']
        b1, b2 = fixed['betas']
        _lib.K.opt_adamw(t, 0.0, float(b1), float(b2), float(fixed['eps']), 1.0, 1.0)
