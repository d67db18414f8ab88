"""The q/k/v pooling kernels (vt_pool_fwd / vt_pool_bwd) element by element against fp64 at grid edges.  -m gpu

Every output is checked per element against the bounds of tests/mvit_pool_ref.py (shown to hold for an fp32 evaluation
and to reject seeded defects in tests/test_mvit_pool_bounds.py), each stage against fp64 computed from the kernel's own
outputs of the stage before.  The kernels are driven through ctypes: every output sits between NaN guard rows and starts
as NaN, the other two slots of a packed q/k/v input hold NaN, and so do the rows past the last token, the dout rows past
the end and the whole scratch, so a missing store, a store outside the output, or a read of the wrong slot, past the end
or of scratch nobody wrote shows.  Both kernel generations of the backward run: the second on 8-byte aligned views, the
first on the same problem as a view 4 bytes into its row.  Their din must agree bit for bit, each must give the same dw
bits over two calls, and dgamma / dbeta must not depend on whether they are adjacent.
"""
import math

import pytest
import torch

from tests import mvit_pool_ref as R
from tests.test_gpu_attention_edges import Guarded, _call, _lib

pytestmark = pytest.mark.gpu

HD = R.HD
PAD = 8                      # rows past the end of every input, NaN


def _sm_count():
    return _lib()[1].vt_sm_count()


class PoolRun:
    """inputs of one pooling problem on the GPU: x [B, N, H*96] (bf16, CPU) placed as `layout` (a slot 0 / 1 / 2 of a
    [B*N, 3*H*96] projection or 'contig'); misalign: the view starts 4 bytes into its row (4- but not 8-byte aligned)"""

    def __init__(self, x, w, gam, bet, H, thw, stride, layout, misalign=False):
        self.B, self.N1, d = x.shape
        self.H, self.thw, self.stride, self.layout, self.d = H, thw, stride, layout, d
        self.To, self.Ho, self.Wo = R.out_thw(thw, stride)
        self.Lo1 = 1 + self.To * self.Ho * self.Wo
        self.rows = self.B * H * self.Lo1
        if layout == 'contig':
            self.width, self.col = d + (4 if misalign else 0), (2 if misalign else 0)
        else:
            self.width, self.col = 3 * d + (4 if misalign else 0), layout * d + (2 if misalign else 0)
        self.xbuf = torch.full((self.B * self.N1 + PAD, self.width), float('nan'), dtype=torch.bfloat16, device='cuda')
        self.xbuf[:self.B * self.N1, self.col:self.col + d] = x.reshape(-1, d).cuda()
        self.w, self.gam, self.bet = w.cuda().contiguous(), gam.cuda(), bet.cuda()

    def _dims(self, p):
        p.B, p.H, p.hd, p.T, p.Hin, p.Win = self.B, self.H, HD, *self.thw
        p.st, p.sh, p.sw = self.stride
        p.To, p.Ho, p.Wo = self.To, self.Ho, self.Wo

    def fwd(self):
        lib_, _ = _lib()
        self.pooled, self.out = Guarded(self.rows, HD, torch.float32), Guarded(self.rows, HD, torch.bfloat16)
        self.mean, self.rstd = Guarded(self.rows, 1, torch.float32), Guarded(self.rows, 1, torch.float32)
        p = lib_.PoolFwdParams()
        p.inp, p.in_bs, p.in_rs = self.xbuf.data_ptr() + 2 * self.col, self.N1 * self.width, self.width
        p.w, p.gamma, p.beta = self.w.data_ptr(), self.gam.data_ptr(), self.bet.data_ptr()
        p.pooled, p.out, p.mean, p.rstd = (t.inner.data_ptr() for t in (self.pooled, self.out, self.mean, self.rstd))
        self._dims(p)
        p.eps = R.EPS
        _call('vt_pool_fwd', p, 'vt_pool_fwd')
        for n in ('pooled', 'out', 'mean', 'rstd'):
            getattr(self, n).check(n)
        shp = (self.B, self.H, self.Lo1)
        return dict(pooled=self.pooled.inner.view(*shp, HD).cpu(), out=self.out.inner.view(*shp, HD).cpu(),
                    mean=self.mean.inner.view(shp).cpu(), rstd=self.rstd.inner.view(shp).cpu())

    def bwd(self, dout, separate=False, sentinel=None):
        """dout [B, H, 1+Lo, 96] fp32 or bf16 (CPU) -> dict of CPU dpooled (the scratch), din [B, H, N, 96] bf16, dw,
        dgamma, dbeta.  separate: dgamma and dbeta in two buffers instead of one [2, 96]"""
        lib_, lib = _lib()
        dbuf = torch.full((self.rows + PAD, HD), float('nan'), dtype=dout.dtype, device='cuda')
        dbuf[:self.rows] = dout.reshape(self.rows, HD).cuda()
        din = Guarded(self.B * self.N1, self.width, torch.bfloat16)
        need = lib.vt_pool_bwd_scratch(self.rows, HD)
        scratch = torch.full((need,), float('nan'), dtype=torch.float32, device='cuda')
        dw = Guarded(HD, 27, torch.float32)
        if separate:
            dg, db = Guarded(1, HD, torch.float32), Guarded(1, HD, torch.float32)
            dg_ptr, db_ptr, gb = dg.inner.data_ptr(), db.inner.data_ptr(), (dg, db)
        else:
            dgb = Guarded(2, HD, torch.float32)
            dg_ptr, db_ptr, gb = dgb.inner.data_ptr(), dgb.inner.data_ptr() + 4 * HD, (dgb,)
        if sentinel is not None:
            for t in (dw,) + gb:
                t.inner.fill_(sentinel)
        p = lib_.PoolBwdParams()
        p.dout, p.dout_fp32 = dbuf.data_ptr(), int(dout.dtype == torch.float32)
        p.pooled, p.mean, p.rstd = self.pooled.inner.data_ptr(), self.mean.inner.data_ptr(), self.rstd.inner.data_ptr()
        p.gamma, p.w = self.gam.data_ptr(), self.w.data_ptr()
        p.inp, p.in_bs, p.in_rs = self.xbuf.data_ptr() + 2 * self.col, self.N1 * self.width, self.width
        p.din, p.din_bs, p.din_rs = din.inner.data_ptr() + 2 * self.col, self.N1 * self.width, self.width
        p.dw, p.dgamma, p.dbeta = dw.inner.data_ptr(), dg_ptr, db_ptr
        p.scratch, p.scratch_floats = scratch.data_ptr(), need
        self._dims(p)
        try:
            _call('vt_pool_bwd', p, 'vt_pool_bwd')
        finally:
            self.last = dict(dw=dw, gb=gb)
        full = self.width == self.d and self.col == 0
        din.check('din', None if full else torch.arange(self.col, self.col + self.d))     # other slots keep their NaN bits
        dw.check('dw')
        for t in gb:
            t.check('dgamma / dbeta')
        dp = scratch[:self.rows * HD]
        assert bool(torch.isfinite(dp).all()), 'dpooled: scratch not written'
        g = torch.cat([t.inner for t in gb]).cpu()
        return dict(dpooled=dp.view(self.B, self.H, self.Lo1, HD).cpu(), dw=dw.inner.view(HD, 27).cpu(), dgamma=g[:HD], dbeta=g[HD:],
                    din=din.inner.view(-1, self.width)[:, self.col:self.col + self.d].reshape(self.B, self.N1, self.H, HD)
                    .permute(0, 2, 1, 3).cpu())


def _bits(t):
    return t.contiguous().view(torch.int16 if t.dtype == torch.bfloat16 else torch.int32)


@pytest.mark.parametrize('case', R.CASES, ids=R.case_id)
def test_pool_kernels_against_fp64(case):
    thw, stride, H, B, layout, regime = case
    x, w, gam, bet, dout = R.make_inputs(B, H, thw, stride, regime, seed=sum(thw) * 7 + H)
    runs = {gen: PoolRun(x, w, gam, bet, H, thw, stride, layout, misalign=gen == 1) for gen in (1, 2)}
    fwds = {gen: run.fwd() for gen, run in runs.items()}
    fwd = fwds[2]
    for n in fwd:
        assert torch.equal(_bits(fwds[1][n]), _bits(fwd[n])), f'{n}: the forward depends on the alignment of its input'
    xh = R.heads(x, H)
    rep = R.Report()
    R.check_forward(xh, w, gam, bet, thw, stride, fwd, rep)
    sm = _sm_count()
    for dt in (torch.float32, torch.bfloat16):
        d = dout.to(dt)
        got = {}
        for gen, run in runs.items():
            got[gen] = run.bwd(d)
            again = run.bwd(d)
            for n in got[gen]:
                assert torch.equal(_bits(got[gen][n]), _bits(again[n])), f'gen{gen} {n}: two calls differ'
        assert torch.equal(_bits(got[1]['dpooled']), _bits(got[2]['dpooled']))
        assert torch.equal(_bits(got[1]['din']), _bits(got[2]['din'])), 'din: the two generations differ'
        R.check_backward(xh, w, gam, thw, stride, fwd, d, got[1], 1, sm, rep)
        R.check_backward(xh, w, gam, thw, stride, fwd, d, got[2], 2, sm, rep, parts=('dw', 'dgb'))
    print(f'[mvit-edges] {R.case_id(case)}: {rep}')


def test_misaligned_view_takes_first_generation():
    """a view 4 bytes into its row cannot take the 8-byte loads of the second generation: it must take the first, whose
    dw bits differ from the second's at this shape (dw sums in another order), and give the aligned view's other bits"""
    thw, stride, H, B = (4, 16, 16), (1, 2, 2), 2, 1
    x, w, gam, bet, dout = R.make_inputs(B, H, thw, stride, seed=21)
    res = {}
    for key, mis in (('aligned', False), ('mis', True)):
        run = PoolRun(x, w, gam, bet, H, thw, stride, 0, misalign=mis)
        fwd = run.fwd()
        res[key] = (fwd, run.bwd(dout))
    for n in ('pooled', 'out', 'mean', 'rstd'):
        assert torch.equal(_bits(res['mis'][0][n]), _bits(res['aligned'][0][n])), n
    assert not torch.equal(_bits(res['mis'][1]['dw']), _bits(res['aligned'][1]['dw']))
    for n in ('din', 'dpooled', 'dgamma', 'dbeta'):
        assert torch.equal(_bits(res['mis'][1][n]), _bits(res['aligned'][1][n])), n
    rep = R.Report()
    xh = R.heads(x, H)
    R.check_forward(xh, w, gam, bet, thw, stride, res['mis'][0], rep)
    R.check_backward(xh, w, gam, thw, stride, res['mis'][0], dout, res['mis'][1], 1, _sm_count(), rep)
    print(f'[mvit-edges] misaligned {R.case_id((thw, stride, H, B, 0, "randn"))}: {rep}')


@pytest.mark.parametrize('gen', [1, 2])
def test_dgamma_dbeta_separate_buffers(gen):
    """dgamma and dbeta in separate buffers (two reductions) give the bits of the adjacent [2, 96] form (one reduction)"""
    thw, stride, H, B = (8, 14, 14), (1, 2, 2), 4, 3
    x, w, gam, bet, dout = R.make_inputs(B, H, thw, stride, seed=22)
    run = PoolRun(x, w, gam, bet, H, thw, stride, 2, misalign=gen == 1)
    fwd = run.fwd()
    a, b = run.bwd(dout), run.bwd(dout, separate=True)
    for n in a:
        assert torch.equal(_bits(a[n]), _bits(b[n])), n
    rep = R.Report()
    R.check_backward(R.heads(x, H), w, gam, thw, stride, fwd, dout, b, gen, _sm_count(), rep, parts=('dgb',))


@pytest.mark.parametrize('thw', [(1, 65, 2), (2, 3, 65), (65, 1, 1)])
def test_backward_refuses_grid_over_64_before_any_launch(thw):
    """the backward takes at most 64 per axis; a larger grid raises RuntimeError and leaves dw / dgamma / dbeta as they were"""
    stride, H, B = (1, 8, 8), 1, 1
    x, w, gam, bet, dout = R.make_inputs(B, H, thw, stride, seed=23)
    run = PoolRun(x, w, gam, bet, H, thw, stride, 'contig')
    run.fwd()                                          # the forward takes any grid
    with pytest.raises(RuntimeError, match='exceeds 64 per axis'):
        run.bwd(dout, sentinel=1234.5)
    torch.cuda.synchronize()
    for t in (run.last['dw'],) + run.last['gb']:
        assert bool((t.inner == 1234.5).all()), 'an output was written before the refusal'
