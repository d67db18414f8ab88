"""Evaluation metrics computed on the device.

`TopKAccuracy` is the accuracy of the reference trainer's validation and test steps (model_trainer.py:254-269 and
:291-299): with views=1 the top-k accuracy of the logits; with views=V the test step over V crops of each clip,
preds.view(-1, V, C).mean(1) -> softmax -> top-k.  Every update is one vt_topk_hits launch adding integer hit counts
to device counters: no host synchronisation per batch, so updates can be captured in a graph.GraphedForward along
with the forward that produces the logits.  compute() reads the counters once.
"""
from __future__ import annotations

import contextlib

import torch

from . import _lib


# {id(metric): (metric, its counters before its first update in the block)} inside restored_after(), else None
_SNAPSHOTS = None


@contextlib.contextmanager
def restored_after():
    """Metric updates made inside the block leave no trace: every TopKAccuracy updated in it gets back the counters it
    had before its first update there (graph.GraphedForward wraps its eager warm-up runs in this).  The snapshots and the
    restore are enqueued on the current stream, in order with the updates."""
    global _SNAPSHOTS
    outer, _SNAPSHOTS = _SNAPSHOTS, {}
    try:
        yield
    finally:
        snaps, _SNAPSHOTS = _SNAPSHOTS, outer
        for metric, before in snaps.values():
            if before is None:
                metric._counts.zero_()
            else:
                metric._counts.copy_(before)


class TopKAccuracy:
    """Running top-k accuracy over the clips seen since the last reset().

    top_k: up to four k values.  views: logit rows per clip (row b*views + v is view v of clip b).
    A clip counts as a hit for k when fewer than k classes have a strictly larger mean logit than its label; this
    equals torch.topk on the softmax probabilities except at near-ties: probabilities that round to the same float, or a
    class within one ulp of the label's mean when torch sums the views in another order (include/vt_b200.h, vt_topk_hits).
    """

    def __init__(self, top_k=(1, 5), views: int = 1, device=None):
        self.top_k = tuple(int(k) for k in top_k)
        if not 1 <= len(self.top_k) <= 4 or min(self.top_k) < 1:
            raise ValueError(f'top_k must hold one to four positive k values, got {top_k}')
        if views < 1:
            raise ValueError(f'views must be >= 1, got {views}')
        self.views = int(views)
        self._counts = None        # int64 [len(top_k) hit counters, 1 sample counter], on the logits' device
        if device is not None:
            self._alloc(torch.device(device))

    def _alloc(self, device):
        with torch.inference_mode(False):
            self._counts = torch.zeros(len(self.top_k) + 1, dtype=torch.int64, device=device)

    def update(self, logits: torch.Tensor, labels: torch.Tensor, want_probs: bool = False):
        """logits [B*views, C] (fp32, or cast to it), labels int64 [B].  Returns softmax of the view mean, fp32 [B, C],
        when want_probs, else None."""
        if _SNAPSHOTS is not None and id(self) not in _SNAPSHOTS:
            _SNAPSHOTS[id(self)] = (self, None if self._counts is None else self._counts.clone())
        if self._counts is None:
            if torch.cuda.is_available() and torch.cuda.is_current_stream_capturing():
                raise RuntimeError('TopKAccuracy: the counters are allocated by the first update, which must not be captured')
            self._alloc(logits.device)
        n = len(self.top_k)
        z = logits.reshape(-1, logits.shape[-1])
        if z.dtype != torch.float32 or not z.is_contiguous():
            z = z.float().contiguous()
        probs = None
        if want_probs:
            probs = torch.empty((labels.numel(), z.shape[1]), dtype=torch.float32, device=z.device)
        _lib.K.topk_hits(z, labels.reshape(-1), self.views, self.top_k, self._counts[:n], self._counts[n:], probs=probs)
        return probs

    def compute(self) -> dict:
        """{k: accuracy in [0, 1]} over the clips seen so far (one device -> host copy); NaN before any update."""
        if self._counts is None:
            return {k: float('nan') for k in self.top_k}
        c = self._counts.tolist()
        seen = c[-1]
        return {k: (c[i] / seen if seen else float('nan')) for i, k in enumerate(self.top_k)}

    def reset(self) -> None:
        if self._counts is not None:
            self._counts.zero_()
