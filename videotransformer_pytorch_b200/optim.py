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


class _FusedBase(torch.optim.Optimizer):
    state_names = ('momentum_buffer',)       # keys in self.state[p], same names as torch.optim.SGD / AdamW

    def _table(self):
        params = [p for g in self.param_groups for p in g['params'] if p.requires_grad]
        tab = getattr(self, '_tab', None)
        if tab is None or [id(p) for p in tab.params] != [id(p) for p in params]:
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
        lrs, wds = [], []
        for g in self.param_groups:
            for p in g['params']:
                if p.requires_grad:
                    lrs.append(float(g['lr']) * float(g.get('lr_scale', 1.0)))
                    wds.append(float(g['weight_decay']))
        tab.bind_hyper(lrs, wds)
        tab.bind_grads()
        return tab

    def load_state_dict(self, state_dict):
        super().load_state_dict(state_dict)
        self._tab = None              # pointer tables are rebuilt from the restored self.state on the next step

    @torch.no_grad()
    def step(self, closure=None, clip_grad=None):
        """Returns the total gradient norm (sqrt of the sum of squared per-parameter norms, before clipping — what
        clip_gradients returns, model_trainer.py:169) as a device scalar when `clip_grad` is not None."""
        if closure is not None:
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

    def __init__(self, params, lr, momentum=0.9, nesterov=True, weight_decay=0.0):
        super().__init__(params, dict(lr=lr, momentum=momentum, nesterov=nesterov, weight_decay=weight_decay))
        if len({g['momentum'] for g in self.param_groups}) > 1 or len({g['nesterov'] for g in self.param_groups}) > 1:
            raise NotImplementedError('per-group momentum / nesterov')

    def _update(self, tab, clip):
        g0 = self.param_groups[0]
        _lib.K.opt_sgd(tab.t, clip, float(g0['momentum']), bool(g0['nesterov']), self._steps == 0)

    def momentum_buffers(self):
        return dict(zip((id(p) for p in self._tab.params), self._tab.state[0]))


class FusedAdamW(_FusedBase):
    """torch.optim.AdamW(betas, eps, weight_decay) with the reference's per-parameter clipping."""
    state_names = ('exp_avg', 'exp_avg_sq')

    def __init__(self, params, lr, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.01):
        super().__init__(params, dict(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay))
        if len({tuple(g['betas']) for g in self.param_groups}) > 1 or len({g['eps'] for g in self.param_groups}) > 1:
            raise NotImplementedError('per-group betas / eps')

    def _update(self, tab, clip):
        g0 = self.param_groups[0]
        b1, b2 = g0['betas']
        t = self._steps + 1
        _lib.K.opt_adamw(tab.t, clip, float(b1), float(b2), float(g0['eps']), 1.0 - b1 ** t, 1.0 - b2 ** t)
