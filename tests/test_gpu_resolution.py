"""TimeSformer at input sizes other than img_size on the kernels.  -m gpu

vt_pos_resize_fwd / _bwd against fp64 F.interpolate and its autograd (with the reference's scale factors), the models
against the reference-generated goldens (tests/resize_golden.py), TimeSformer-B geometry at 16 x 448^2 and 8 x 320^2
against the fp64 oracle, and the resize inside a captured training step."""
import math

import pytest
import torch
import torch.nn.functional as F

from tests.conftest import check_grads, rel_err
from tests.resize_golden import PARAMS, family

pytestmark = pytest.mark.gpu

GUARD = 3
PAIRS = [(14, (16, 16)), (14, (20, 20)), (14, (28, 28)), (14, (7, 7)), (14, (20, 14)), (14, (14, 20)), (2, (3, 3)),
         (2, (1, 1))]


def _scales(g, out_grid):
    """The reference's scale_factor ((n + 0.1) / sqrt(N)) for an output grid"""
    return tuple((n + 0.1) / math.sqrt(g * g) for n in out_grid)


def _guarded(rows, D, fill=float('nan')):
    """[GUARD + rows + GUARD, D] fp32 buffer filled with `fill`, and its middle rows"""
    buf = torch.full((rows + 2 * GUARD, D), fill, dtype=torch.float32, device='cuda')
    return buf, buf[GUARD:GUARD + rows]


def _interp64(rows, g, out_grid, scales):
    D = rows.shape[1]
    y = F.interpolate(rows.reshape(g, g, D).permute(2, 0, 1)[None], scale_factor=scales, mode='bicubic',
                      align_corners=False)
    assert tuple(y.shape[-2:]) == tuple(out_grid)
    return y[0].permute(1, 2, 0).reshape(-1, D)


@pytest.mark.parametrize('D', [128, 768])
@pytest.mark.parametrize('g,out_grid', PAIRS, ids=[f'{g}to{o[0]}x{o[1]}' for g, o in PAIRS])
def test_pos_resize_fwd_matches_fp64_interpolate(g, out_grid, D):
    from videotransformer_pytorch_b200 import _lib
    torch.manual_seed(0)
    x = torch.randn(g * g, D)
    sbuf, src = _guarded(g * g, D)
    src.copy_(x)
    n_out = out_grid[0] * out_grid[1]
    obuf, out = _guarded(n_out, D)
    sc = _scales(g, out_grid)
    _lib.K.pos_resize_fwd(src, (g, g), out_grid, sc, out=out)
    ref = _interp64(x.double(), g, out_grid, sc)
    err = (out.cpu().double() - ref).abs().max().item()
    print(f'{g}->{out_grid} D={D}: max abs err {err:.2e} (max|x| {x.abs().max().item():.2f})')
    assert err <= 4e-6 * x.abs().max().item()
    assert torch.isnan(obuf[:GUARD]).all() and torch.isnan(obuf[GUARD + n_out:]).all()
    again = _lib.K.pos_resize_fwd(src, (g, g), out_grid, sc)
    assert torch.equal(again, out)


@pytest.mark.parametrize('D', [128, 768])
@pytest.mark.parametrize('g,out_grid', PAIRS, ids=[f'{g}to{o[0]}x{o[1]}' for g, o in PAIRS])
def test_pos_resize_bwd_is_the_adjoint(g, out_grid, D):
    from videotransformer_pytorch_b200 import _lib
    torch.manual_seed(1)
    n_out = out_grid[0] * out_grid[1]
    sc = _scales(g, out_grid)
    x, dy = torch.randn(g * g, D), torch.randn(n_out, D)
    dbuf, dsrc = _guarded(n_out, D)
    dsrc.copy_(dy)
    gbuf, gx = _guarded(g * g, D)
    _lib.K.pos_resize_bwd(dsrc, (g, g), out_grid, sc, out=gx)
    x64 = x.double().requires_grad_(True)
    (ref,) = torch.autograd.grad(_interp64(x64, g, out_grid, sc), x64, dy.double())
    err = (gx.cpu().double() - ref).abs().max().item()
    print(f'{g}->{out_grid} D={D}: adjoint max abs err {err:.2e} (max|ref| {ref.abs().max().item():.2f})')
    assert err <= 4e-6 * ref.abs().max().item() + 4e-6 * dy.abs().max().item()
    assert torch.isnan(gbuf[:GUARD]).all() and torch.isnan(gbuf[GUARD + g * g:]).all()
    # <R x, y> == <x, R^T y>
    rx = _lib.K.pos_resize_fwd(x.cuda(), (g, g), out_grid, sc)
    lhs = (rx.double() * dy.cuda().double()).sum().item()
    rhs = (x.cuda().double() * gx.double()).sum().item()
    assert abs(lhs - rhs) <= 1e-5 * (rx.double().norm() * dy.double().norm()).item()
    for _ in range(3):                                          # deterministic: no atomics
        assert torch.equal(_lib.K.pos_resize_bwd(dsrc, (g, g), out_grid, sc), gx)


@pytest.mark.parametrize('name,tag', PARAMS)
def test_timesformer_resize_golden(name, tag):
    fam = family(name)
    case = fam.cases[tag]
    m = fam.model(case.learnable).cuda().eval()
    x = case.x.cuda()
    with torch.no_grad():
        e_eval = rel_err(m(x).cpu(), case.y_eval)
    m.train()
    torch.manual_seed(case.train_seed)
    y = m(x)
    e_tr = rel_err(y.detach().cpu(), case.y_train)
    (y.double() * case.loss_w.cuda()).sum().backward()
    grads = {n: p.grad for n, p in m.named_parameters()}
    worst = check_grads(grads, case, 5e-2)
    print(f'{name}:{tag}: eval {e_eval:.2e} train {e_tr:.2e} worst grad {worst:.2e}'
          + (f' pos_embed grad {rel_err(grads["pos_embed"].cpu(), case.grad["pos_embed"]):.2e}' if case.learnable else ''))
    assert e_eval < 1.5e-2 and e_tr < 1.5e-2
    assert ('pos_embed' in case.grad) == case.learnable


def _timesformer_b(T, seed):
    from videotransformer_pytorch_b200 import TimeSformer
    torch.manual_seed(seed)
    m = TimeSformer(num_frames=T, img_size=224, patch_size=16, embed_dims=768, num_heads=12, num_transformer_layers=1)
    with torch.no_grad():
        for n, p in m.named_parameters():
            if 'temporal_fc' in n or n.endswith('bias'):
                p.normal_(std=0.02)
    sd = {k: v.detach().clone() for k, v in m.state_dict().items()}
    cfg = dict(num_frames=T, img_size=224, patch_size=16, embed_dims=768, num_heads=12, num_transformer_layers=1)
    return m.cuda().eval(), sd, cfg


@pytest.mark.parametrize('T,side', [(16, 448), (8, 320)])
def test_timesformer_b_larger_inputs_vs_oracle(T, side, monkeypatch):
    """img_size 224, one layer, B = 1: 448^2 gives spatial N = 785 (tiled tensor-core kernels), 320^2 gives N = 401.  The fp64
    oracle runs on the GPU for speed, except its pos_embed resize, which runs on the CPU like the reference's."""
    from oracle import resize_oracle as O
    cpu_resize = O.interpolate_pos_encoding
    monkeypatch.setattr(O, 'interpolate_pos_encoding',
                        lambda pos, *a: cpu_resize(pos.cpu(), *a).to(pos.device))
    m, sd, cfg = _timesformer_b(T, 9)
    x = torch.randn(1, T, 3, side, side, generator=torch.Generator().manual_seed(10))
    with torch.no_grad():
        got = m(x.cuda()).cpu()
        ref = O.timesformer_forward({k: v.cuda().double() for k, v in sd.items()}, x.cuda().double(), cfg).cpu()
    e = rel_err(got, ref)
    print(f'TimeSformer-B {T}x{side}^2: {e:.2e}')
    assert e < 5e-3
    if side == 320:
        with torch.no_grad():
            attn = m.get_last_selfattention(x.cuda()).cpu()
            ref_a = O.timesformer_last_selfattention({k: v.cuda().double() for k, v in sd.items()}, x.cuda().double(),
                                                     cfg).cpu()
        assert attn.shape == ref_a.shape == (T, 12, 401, 401)
        ea = rel_err(attn, ref_a)
        print(f'TimeSformer-B {T}x{side}^2 last self-attention: {ea:.2e}')
        assert ea < 1e-2


class _Net(torch.nn.Module):
    def __init__(self):
        super().__init__()
        from videotransformer_pytorch_b200 import ClassificationHead, TimeSformer
        self.model = TimeSformer(num_frames=2, img_size=224, patch_size=16, embed_dims=128, num_heads=2,
                                 num_transformer_layers=2)
        self.head = ClassificationHead(10, 128)
        with torch.no_grad():
            for n, p in self.model.named_parameters():
                if 'temporal_fc' in n:
                    p.normal_(std=0.05)

    def forward(self, x, y):
        return torch.nn.functional.cross_entropy(self.head(self.model(x)), y)


def test_graphed_step_at_320_contains_the_resize():
    from videotransformer_pytorch_b200.graph import GraphedTrainStep
    torch.manual_seed(0)
    net = _Net().cuda().train()
    x = torch.randn(2, 2, 3, 320, 320, device='cuda')
    y = torch.tensor([1, 7], device='cuda')
    step = GraphedTrainStep(net, (x, y))

    def eager():
        for p in net.parameters():
            p.grad = None
        torch.manual_seed(5)
        loss = net(x, y)
        loss.backward()
        return loss.detach(), {n: p.grad.clone() for n, p in net.named_parameters()}

    for trial in range(2):
        torch.manual_seed(5)
        loss_g = step(x, y).clone()
        gg = {n: p.grad.clone() for n, p in net.named_parameters()}
        loss_e, ge = eager()
        print(f'trial {trial}: graph loss {loss_g.item():.6f} eager {loss_e.item():.6f}')
        assert torch.equal(loss_g, loss_e)
        assert torch.equal(gg['model.pos_embed'], ge['model.pos_embed'])
        bad = [n for n in gg if not torch.allclose(gg[n], ge[n], rtol=1e-4, atol=1e-6)]
        assert not bad, bad
        before = loss_g
        with torch.no_grad():
            net.model.pos_embed.add_(0.5 * torch.randn_like(net.model.pos_embed))    # in place: the graph reads it
    torch.manual_seed(5)
    assert not torch.equal(step(x, y), before)


def test_uint8_clip_at_new_size_matches_float_clip():
    from videotransformer_pytorch_b200 import TimeSformer
    torch.manual_seed(2)
    m = TimeSformer(num_frames=2, img_size=32, patch_size=16, embed_dims=128, num_heads=2,
                    num_transformer_layers=1).cuda().eval()
    mean, std = (0.485, 0.456, 0.406), (0.229, 0.224, 0.225)
    m.set_input_normalization(mean, std)
    u8 = torch.randint(0, 256, (2, 2, 48, 64, 3), dtype=torch.uint8, generator=torch.Generator().manual_seed(0))
    xf = ((u8.float() / 255.0 - torch.tensor(mean)) / torch.tensor(std)).permute(0, 1, 4, 2, 3).contiguous()
    with torch.no_grad():
        y8, yf = m(u8.cuda()), m(xf.cuda())
    e = rel_err(y8.cpu(), yf.cpu())
    print(f'uint8 vs float clip at 48x64: {e:.2e}')
    assert e < 2e-3


def test_training_grid_step_runs_no_resize(monkeypatch):
    """At the training grid the step launches exactly what it did before: PosResizeFn is never reached."""
    from videotransformer_pytorch_b200 import TimeSformer, _lib, ops

    def refuse(*a, **k):
        raise AssertionError('resize at the training grid')
    monkeypatch.setattr(ops.PosResizeFn, 'apply', refuse)
    m = TimeSformer(num_frames=2, img_size=32, patch_size=16, embed_dims=128, num_heads=2,
                    num_transformer_layers=1).cuda().train()
    x = torch.randn(2, 2, 3, 32, 32, device='cuda')
    counts = []
    for _ in range(3):                  # the first step also builds per-stream scratch state
        n0 = _lib.launch_count()
        m(x).sum().backward()
        torch.cuda.synchronize()
        counts.append(_lib.launch_count() - n0)
    assert counts[1] == counts[2] > 0
