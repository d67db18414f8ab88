"""The per-element bounds of tests/mvit_pool_ref.py, on the CPU: they hold for an fp32 evaluation of every stage of the
q/k/v pooling at every shape of tests/test_gpu_mvit_edges.py, and the checker rejects seeded defects of the kinds the
kernels could have.  No GPU needed."""
import math

import pytest
import torch
import torch.nn.functional as F

from oracle.mvit_oracle import attention_pool
from tests import mvit_pool_ref as R

HD = R.HD
SM = 132                       # SM count of an H100 SXM: fixes the CTA partition the fp32 model sums by


def model(x, w, gam, bet, dout, H, thw, stride, gen=1, dw_double=None):
    """fp32 evaluation of vt_pool_fwd / vt_pool_bwd (bf16 out and din, like the kernels).  x bf16 [B, N, H*96];
    dout fp32 or bf16.  dw is summed per CTA as the kernel of generation `gen` partitions the rows, then over the CTAs;
    dw_double = k counts CTA k's partial twice."""
    B = x.shape[0]
    xh = R.heads(x, H).float()
    w5 = w.reshape(HD, 1, 3, 3, 3)
    To, Ho, Wo = R.out_thw(thw, stride)
    vol = xh[:, :, 1:].reshape(B * H, *thw, HD).permute(0, 4, 1, 2, 3)
    body = F.conv3d(vol, w5, stride=stride, padding=1, groups=HD).reshape(B, H, HD, -1).transpose(2, 3)
    p = torch.cat([xh[:, :, :1], body], 2)
    mu = p.sum(-1) * R.INV_HD32
    rs = torch.rsqrt((p - mu[..., None]).square().sum(-1) * R.INV_HD32 + R.EPS32)
    xhat = (p - mu[..., None]) * rs[..., None]
    out = (xhat * gam + bet).bfloat16()
    d = dout.float()
    gy = d * gam
    m1, m2 = gy.sum(-1, keepdim=True) * R.INV_HD32, (gy * xhat).sum(-1, keepdim=True) * R.INV_HD32
    dp = rs[..., None] * (gy - m1 - xhat * m2)
    dpv = dp[:, :, 1:].transpose(2, 3).reshape(B * H, HD, To, Ho, Wo)
    gin = torch.nn.grad.conv3d_input((B * H, HD, *thw), w5, dpv, stride=stride, padding=1, groups=HD)
    din = torch.cat([dp[:, :, :1], gin.reshape(B, H, HD, -1).transpose(2, 3)], 2).bfloat16()
    rows = B * H * To * Ho * Wo
    blocks, rpc = R.dw_plan(rows, gen, SM)
    xp = F.pad(vol, (1, 1, 1, 1, 1, 1))
    dw = torch.empty(HD, 27)
    for tap in range(27):
        kt, kh, kw = tap // 9, tap // 3 % 3, tap % 3
        xs = xp[:, :, kt:kt + stride[0] * (To - 1) + 1:stride[0], kh:kh + stride[1] * (Ho - 1) + 1:stride[1],
                kw:kw + stride[2] * (Wo - 1) + 1:stride[2]]
        prod = (xs * dpv).reshape(B * H, HD, -1).transpose(1, 2).reshape(rows, HD)
        part = F.pad(prod, (0, 0, 0, blocks * rpc - rows)).reshape(blocks, rpc, HD).sum(1)
        dw[:, tap] = part.sum(0) + (part[dw_double] if dw_double is not None else 0)
    return dict(pooled=p, mean=mu, rstd=rs, out=out, dpooled=dp, din=din, dw=dw,
                dgamma=(d * xhat).sum((0, 1, 2)), dbeta=d.sum((0, 1, 2)))


def run_checks(x, w, gam, bet, dout, got, H, thw, stride, gen=1, parts=('dpooled', 'din', 'dw', 'dgb')):
    rep = R.Report()
    xh = R.heads(x, H)
    R.check_forward(xh, w, gam, bet, thw, stride, got, rep)
    R.check_backward(xh, w, gam, thw, stride, got, dout, got, gen, SM, rep, parts)
    return rep


@pytest.mark.parametrize('case', R.CASES, ids=R.case_id)
def test_fp32_evaluation_sits_inside_every_bound(case):
    thw, stride, H, B, _, regime = case
    x, w, gam, bet, dout = R.make_inputs(B, H, thw, stride, regime, seed=1)
    for dt in (torch.float32, torch.bfloat16):
        d = dout.to(dt)
        for gen in (1, 2):
            got = model(x, w, gam, bet, d, H, thw, stride, gen)
            rep = run_checks(x, w, gam, bet, d, got, H, thw, stride, gen, ('dw',) if gen == 2 else ('dpooled', 'din', 'dw', 'dgb'))
            print(f'[pool-bounds] {R.case_id(case)} dout {dt} gen{gen}: {rep}')


def test_offset_rows_have_large_mean_next_to_spread():
    """the 'offset' regime makes rows whose mean is far above their spread (the rstd bound's delta^2 term matters there)"""
    thw, stride = (3, 9, 8), (1, 2, 2)
    x, w, gam, bet, dout = R.make_inputs(1, 1, thw, stride, 'offset')
    p, _ = R.pool_forward(R.heads(x, 1), w, thw, stride)
    assert float((p.mean(-1).abs() / p.std(-1)).median()) > 50


def test_reference_matches_the_oracle_pooling():
    """the fp64 reference is the oracle's attention_pool (conv + LayerNorm with the cls row), forward and backward"""
    thw, stride, H = (3, 9, 7), (1, 2, 4), 2
    x, w, gam, bet, dout = R.make_inputs(2, H, thw, stride, seed=3)
    xh = R.heads(x, H).requires_grad_(True)
    w5 = w.double().reshape(HD, 1, 3, 3, 3).requires_grad_(True)
    g64, b64 = gam.double().requires_grad_(True), bet.double().requires_grad_(True)
    ref, new_thw = attention_pool(xh, thw, conv_w=w5, stride=stride, norm_w=g64, norm_b=b64, eps=R.EPS)
    assert new_thw == R.out_thw(thw, stride)
    pooled, out = R.pool_forward(xh.detach(), w, thw, stride, gam, bet)
    assert float((out - ref.detach()).abs().max()) < 1e-12
    ref.backward(dout.double())
    p = pooled
    mu, rs = p.mean(-1), (p.var(-1, unbiased=False) + R.EPS).rsqrt()
    dp, xhat, _, _, _ = R.ln_backward(p, mu, rs, gam, dout)
    din = torch.cat([dp[:, :, :1], R.conv_adjoint(dp[:, :, 1:], w, thw, stride)], 2)
    assert float((din - xh.grad).abs().max()) < 1e-12
    assert float((R.conv_wgrad(xh.detach()[:, :, 1:], dp[:, :, 1:], thw, stride) - w5.grad.reshape(HD, 27)).abs().max()) < 1e-12
    d = dout.double()
    assert float(((d * xhat).sum((0, 1, 2)) - g64.grad).abs().max()) < 1e-12
    assert float((d.sum((0, 1, 2)) - b64.grad).abs().max()) < 1e-12


def test_config_shapes_include_the_stage_one_kv_pooling():
    shapes = R.config_shapes()
    assert ((8, 56, 56), (1, 8, 8), 1) in shapes
    assert ((8, 28, 28), (1, 4, 4), 2) in shapes and ((8, 14, 14), (1, 2, 2), 8) in shapes


# ---- seeded defects ---------------------------------------------------------------------------------------------------
THW, STRIDE, H, B = (3, 8, 10), (1, 2, 4), 2, 2         # (Win - 1) % 4 != 0: the last output column's window lies inside the grid


def _setup():
    x, w, gam, bet, dout = R.make_inputs(B, H, THW, STRIDE, seed=7)
    return x, w, gam, bet, dout, model(x, w, gam, bet, dout, H, THW, STRIDE)


def _bump_bf16(t, idx, ulps):
    v = t[idx].view(torch.int16)
    t[idx] = (v + ulps).view(torch.bfloat16)


def _rejects(name, x, w, gam, bet, dout, got, **kw):
    with pytest.raises(AssertionError, match=f'^{name}: '):
        run_checks(x, w, gam, bet, dout, got, H, THW, STRIDE, **kw)


def test_clean_run_passes():
    x, w, gam, bet, dout, got = _setup()
    run_checks(x, w, gam, bet, dout, got, H, THW, STRIDE)


@pytest.mark.parametrize('name', ['din', 'out'])
def test_rejects_cls_row_off_by_four_ulps(name):
    x, w, gam, bet, dout, got = _setup()
    _bump_bf16(got[name], (1, 1, 0, 37), 4)
    _rejects(name, x, w, gam, bet, dout, got)


def test_rejects_tap_dropped_at_last_output_column():
    x, w, gam, bet, dout, got = _setup()
    To, Ho, Wo = R.out_thw(THW, STRIDE)
    wi = (Wo - 1) * STRIDE[2] + 1                     # tap dw = 2 of the last column
    assert wi < THW[2]
    xh = R.heads(x, H).float()
    for ot in range(To):
        for oh in range(Ho):
            hi = oh * STRIDE[1]                       # tap dh = 1
            o = 1 + (ot * Ho + oh) * Wo + Wo - 1
            got['pooled'][:, :, o] -= w[:, 9 * 1 + 3 * 1 + 2] * xh[:, :, 1 + (ot * THW[1] + hi) * THW[2] + wi]
    _rejects('pooled', x, w, gam, bet, dout, got)


def test_rejects_tap_dropped_at_last_input_row_of_din():
    x, w, gam, bet, dout, got = _setup()
    To, Ho, Wo = R.out_thw(THW, STRIDE)
    hi = THW[1] - 1                                   # last input row: reached by output row (hi + 1 - dh) / 2
    oh, dh = (hi + 1 - 2) // STRIDE[1], 2
    assert oh * STRIDE[1] - 1 + dh == hi
    dp = got['dpooled']
    din = got['din'].float()
    for ti in range(THW[0]):
        for wi in range(0, THW[2], STRIDE[2]):        # dw = 1: ow = wi / 4
            n = 1 + (ti * THW[1] + hi) * THW[2] + wi
            din[:, :, n] -= w[:, 9 * 1 + 3 * dh + 1] * dp[:, :, 1 + (ti * Ho + oh) * Wo + wi // STRIDE[2]]
    got['din'] = din.bfloat16()
    _rejects('din', x, w, gam, bet, dout, got)


def test_rejects_uncovered_token_set_non_zero():
    x, w, gam, bet, dout, got = _setup()
    n = int((~R.covered(THW, STRIDE)).nonzero()[0])
    got['din'][0, 1, 1 + n, 5] = 1e-3
    _rejects('din', x, w, gam, bet, dout, got)


def test_rejects_uncovered_token_set_to_negative_zero():
    x, w, gam, bet, dout, got = _setup()
    n = int((~R.covered(THW, STRIDE)).nonzero()[0])
    got['din'][1, 0, 1 + n, 0] = -0.0
    with pytest.raises(AssertionError, match='^din: .* not \\+0'):
        run_checks(x, w, gam, bet, dout, got, H, THW, STRIDE)


def test_rejects_two_heads_swapped():
    x, w, gam, bet, dout, _ = _setup()
    xs = x.reshape(B, -1, H, HD)[:, :, [1, 0]].reshape(x.shape)          # the kernel read head 1 for head 0 and back
    got = model(xs, w, gam, bet, dout, H, THW, STRIDE)
    _rejects('pooled', x, w, gam, bet, dout, got)


def test_rejects_neighbouring_slot_read():
    x, w, gam, bet, dout, _ = _setup()
    qkv = torch.cat([x, R.make_inputs(B, H, THW, STRIDE, seed=8)[0], R.make_inputs(B, H, THW, STRIDE, seed=9)[0]], 2)
    d = H * HD
    got = model(qkv[:, :, d:2 * d], w, gam, bet, dout, H, THW, STRIDE)   # slot 1 read where slot 0 was asked for
    _rejects('pooled', qkv[:, :, :d], w, gam, bet, dout, got)


def test_rejects_dw_partial_counted_twice():
    x, w, gam, bet, dout, _ = _setup()
    rows = B * H * math.prod(R.out_thw(THW, STRIDE))
    blocks, _ = R.dw_plan(rows, 1, SM)
    got = model(x, w, gam, bet, dout, H, THW, STRIDE, dw_double=blocks - 1)
    _rejects('dw', x, w, gam, bet, dout, got)
