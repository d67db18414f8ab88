"""FP8 inference forms on the GPU: the e4m3 GEMM element by element against fp64 (every epilogue of the forward forms,
tile edges, NaN guards), the row quantiser bit for bit against its CPU twin, the fp8 forward of the models against a
quantising fp64 emulation and the fp64 oracle goldens, and GraphedForward with fp8 around training steps.

GEMM gate: the operands are e4m3 values times power-of-two scales, so every product is exact in fp64 and
    |c - c64| <= 2^-9 * sum_k |a_k b_k| + (the epilogue's output rounding).
The 2^-12 gate that fp32 accumulation inside each 128-wide k-block would allow does not hold on the H100: at K = 96 (one
k-block, so no promotion is involved) the e4m3 wgmma's error reached 3.57 x 2^-12 sum|ab| (about 2^-10.2), while the bf16
GEMM on the same values stays below 0.01 x 2^-12.  The fp8 MMA does not accumulate in full fp32 within an instruction
sequence; the promotion into the fp32 tile accumulator every 128 K keeps the error from growing with K.  The gate is
2^-9, twice the worst seen.  The same values also run through the bf16 GEMM (e4m3 values are exact in bf16), a second
reference held to 2^-12; the worst ratios are printed (FP8-REPORT lines)."""
import pytest
import torch

from tests.conftest import rel_err
from tests.emu_fp8 import E4M3_MAX, quant_rows_twin
from tests.emu_kernels import EmuKernels

pytestmark = pytest.mark.gpu

GATE = 2.0 ** -9            # e4m3 GEMM accumulation (module docstring)
GATE_BF16 = 2.0 ** -12      # bf16 GEMM: fp32 accumulation
U_BF16 = 2.0 ** -8          # one bf16 ulp relative (twice the unit roundoff: covers the ties-to-even bound with slack)


def _k():
    from videotransformer_pytorch_b200 import _lib
    return _lib.K


def _rand_e4m3(rows, cols, gen, pad_rows=0, pad_cols=16):
    """e4m3 values (no NaN) [rows, cols] as a view into a NaN-filled [rows + pad_rows, cols + pad_cols] buffer, and the values
    in fp64.  Magnitudes span the e4m3 range, half of them below 1."""
    from videotransformer_pytorch_b200._lib import E4M3  # noqa: F401
    buf = torch.full((rows + pad_rows, cols + pad_cols), 0x7F, dtype=torch.uint8)      # 0x7F: e4m3 NaN
    b = torch.randint(0, 256, (rows, cols), generator=gen, dtype=torch.int64).to(torch.uint8)
    b = torch.where((b & 0x7F) == 0x7F, b & 0xF0, b)                                    # drop NaN codes
    buf[:rows, :cols] = b
    q = buf.view(torch.float8_e4m3fn)
    return q.cuda()[:rows, :cols], q[:rows, :cols].double()


def _scales(n, gen, pad=8):
    s = torch.full((n + pad,), float('nan'))
    s[:n] = torch.ldexp(torch.ones(n), torch.randint(-6, 3, (n,), generator=gen)).float()
    return s.cuda(), s[:n].double()


def _operands(M, N, K, seed):
    from videotransformer_pytorch_b200._lib import E4M3
    gen = torch.Generator().manual_seed(seed)
    qa, a64 = _rand_e4m3(M, K, gen, pad_rows=8)
    qb, b64 = _rand_e4m3(N, K, gen, pad_rows=64)
    sa, sa64 = _scales(M, gen)
    sb, sb64 = _scales(N, gen)
    A = a64 * sa64[:, None]
    B = b64 * sb64[:, None]
    acc = A @ B.t()
    mag = A.abs() @ B.abs().t()
    return E4M3(qa, sa[:M]), E4M3(qb, sb[:N]), A, B, acc, mag


def _guarded_out(M, N, dtype):
    full = torch.full((M + 8, N + 16), float('nan'), dtype=dtype, device='cuda')
    return full, full[:M, :N]


def _guards_intact(full, M, N):
    return bool(torch.isnan(full[M:].float()).all()) and bool(torch.isnan(full[:, N:].float()).all())


REPORT = {}


def _report(name, ratio):
    REPORT[name] = max(REPORT.get(name, 0.0), ratio)
    print(f'FP8-REPORT {name} worst error / gate = {REPORT[name]:.4f}')


SHAPES = [(12552, 2304, 768), (12552, 3072, 768), (12552, 768, 3072), (1000, 288, 96), (136, 384, 1536), (12544, 768, 768)]


@pytest.mark.parametrize('M,N,K', SHAPES)
@pytest.mark.parametrize('epi', ['bf16', 'f32', 'gelu_h'])
def test_gemm_e4m3_elementwise(M, N, K, epi):
    k = _k()
    a, b, A, B, acc, mag = _operands(M, N, K, seed=M + N + K)
    gen = torch.Generator().manual_seed(7)
    bias = torch.randn(N, generator=gen, dtype=torch.float64) * 4
    rs = torch.rand(M, generator=gen, dtype=torch.float64) + 0.5
    kw = dict(bias=bias.float().cuda(), row_scale=rs.float().cuda())
    bias, rs = bias.float().double(), rs.float().double()
    z = rs[:, None] * (acc + bias)
    zb = rs[:, None] * (mag + bias.abs())                  # magnitude of the exact sum (for the accumulation gate)
    full, out = _guarded_out(M, N, torch.float32 if epi == 'f32' else torch.bfloat16)
    if epi == 'f32':
        aux = torch.randn(M, N, generator=gen, dtype=torch.float64) * 16
        bias2 = torch.randn(N, generator=gen, dtype=torch.float64)
        kw.update(aux=aux.float().cuda(), bias2=bias2.float().cuda())
        ref = z + bias2.float().double() + aux.float().double()
        tol = GATE * rs[:, None] * mag + 2.0 ** -22 * (zb + aux.abs() + bias2.abs()) + 1e-30
    elif epi == 'bf16':
        ref = z
        tol = GATE * rs[:, None] * mag + U_BF16 * (z.abs() + GATE * rs[:, None] * mag) + 1e-30
    else:
        zr = z
        ref = 0.5 * zr * (1 + torch.erf(zr / 2 ** 0.5))
        # the kernel rounds z to bf16 before GELU (|gelu'| <= 1.13), then rounds h; 2e-7 |z|: its erf approximation
        ez = GATE * rs[:, None] * mag + U_BF16 * z.abs()
        tol = 1.13 * ez + U_BF16 * ref.abs() + 2e-7 * z.abs() + 1e-30
    k.gemm_e4m3(a, b, M, N, K, epi=epi, out=out, **kw)
    torch.cuda.synchronize()
    got = out.double().cpu()
    assert _guards_intact(full, M, N), 'rows or columns past M / N were written'
    assert not bool(torch.isnan(got).any()), 'NaN from the guard bytes / scales was read'
    err = (got - ref).abs()
    ratio = float((err / tol).max())
    _report(f'e4m3 {epi} vs fp64', ratio)
    assert ratio <= 1.0, (ratio, M, N, K, epi)


@pytest.mark.parametrize('M,N,K', [(12552, 2304, 768), (12552, 768, 3072), (1000, 288, 96)])
def test_gemm_e4m3_accumulation_vs_fp64_and_bf16_gemm(M, N, K):
    """Plain fp32 output (no epilogue arithmetic): the e4m3 GEMM against fp64 and against the bf16 GEMM on the same values."""
    k = _k()
    a, b, A, B, acc, mag = _operands(M, N, K, seed=3 * M + N + K)
    c8 = k.gemm_e4m3(a, b, M, N, K, epi='f32').double().cpu()
    c16 = k.gemm(A.to(torch.bfloat16).cuda(), B.to(torch.bfloat16).cuda(), M, N, K, epi='f32').double().cpu()
    assert torch.equal(A.to(torch.bfloat16).double(), A)                 # e4m3 x 2^k is exact in bf16
    r8 = float(((c8 - acc).abs() / (GATE * mag + 1e-30)).max())
    r16 = float(((c16 - acc).abs() / (GATE_BF16 * mag + 1e-30)).max())
    r816 = float(((c8 - c16).abs() / (GATE * mag + 1e-30)).max())
    print(f'FP8-REPORT accumulation M={M} N={N} K={K}: |e4m3 - fp64| / (2^-9 sum|ab|) = {r8:.4f}; bf16 GEMM / (2^-12 sum|ab|) '
          f'{r16:.4f}; |e4m3 - bf16 GEMM| / (2^-9 sum|ab|) {r816:.4f}')
    _report('e4m3 f32 plain vs fp64', r8)
    _report('bf16 GEMM on the e4m3 values vs fp64', r16)
    assert r8 <= 1.0 and r16 <= 1.0


def test_gemm_e4m3_affine_row_map_and_row_maps():
    """The residual-scatter epilogues of the divided space-time blocks: affine maps (temporal, spatial with the cls side
    rows) and out_row / aux_row arrays."""
    from videotransformer_pytorch_b200 import ops
    k = _k()
    B, T, P, D = 2, 4, 16, 768
    S = 1 + P * T
    maps = ops.token_maps(B, T, P, 'cuda')
    amaps = ops.affine_row_maps(B, T, P, D)
    gen = torch.Generator().manual_seed(1)
    for name, M, out_key, aux_key in (('temporal', B * P * T, 'temporal', 'temporal'), ('spatial', B * T * (P + 1), 'sp_out', 'sp_aux')):
        a, b, A, Bm, acc, mag = _operands(M, D, D, seed=M)
        x = torch.randn(B * S, D, generator=gen, dtype=torch.float64) * 8
        bias = torch.randn(D, generator=gen, dtype=torch.float64)
        bias2 = torch.randn(D, generator=gen, dtype=torch.float64) if name == 'temporal' else None
        rs = torch.rand(M, generator=gen, dtype=torch.float64) + 0.5
        orow, arow = maps[out_key].cpu().long(), maps[aux_key].cpu().long()
        for use_map in (True, False):
            out = torch.full((B * S + (B * T if name == 'spatial' else 0), D), float('nan'), device='cuda')
            kw = dict(bias=bias.float().cuda(), aux=x.float().cuda(), out=out, out_row=maps[out_key], aux_row=maps[aux_key],
                      row_scale=rs.float().cuda())
            if bias2 is not None:
                kw['bias2'] = bias2.float().cuda()
            if use_map:
                kw['row_map'] = amaps[name]
            k.gemm_e4m3(a, b, M, D, D, epi='f32', **kw)
            got = out.double().cpu()
            add = torch.where((arow >= 0)[:, None], x.float().double()[arow.clamp(min=0)], torch.zeros(M, D, dtype=torch.float64))
            b2 = bias2.float().double() if bias2 is not None else 0.0
            ref = rs.float().double()[:, None] * (acc + bias.float().double()) + b2 + add
            tol = GATE * rs[:, None] * mag + 2.0 ** -22 * (ref.abs() + add.abs() + rs[:, None] * mag) + 1e-30
            ratio = float(((got[orow] - ref).abs() / tol).max())
            _report(f'e4m3 f32 {name} row maps vs fp64', ratio)
            assert ratio <= 1.0, (name, use_map, ratio)
            written = torch.zeros(out.shape[0], dtype=torch.bool)
            written[orow] = True
            assert bool(torch.isnan(got[~written]).all())


def test_gemm_e4m3_rejects():
    k = _k()
    a, b, *_ = _operands(256, 128, 128, seed=5)
    with pytest.raises(RuntimeError):
        k.gemm_e4m3(a, b, 256, 128, 128, epi='gelu')
    from videotransformer_pytorch_b200._lib import E4M3
    a96 = E4M3(a.q[:, :104], a.scale)                     # K = 104: not a multiple of 16
    with pytest.raises(RuntimeError, match='multiples of 16'):
        k.gemm_e4m3(a96, E4M3(b.q[:, :104], b.scale), 256, 128, 104, epi='bf16')


@pytest.mark.parametrize('dtype', [torch.bfloat16, torch.float32])
@pytest.mark.parametrize('K', [96, 768, 3072])
def test_quant_rows_bitwise_against_twin(dtype, K):
    k = _k()
    gen = torch.Generator().manual_seed(K + (dtype == torch.float32))
    M = 777
    x = torch.randn(M, K, generator=gen) * torch.ldexp(torch.ones(M, 1), torch.randint(-30, 30, (M, 1), generator=gen))
    x[0] = 0.0
    x[1] = 0.5
    x[1, 3] = 448.0 * 2.0 ** 3                                   # amax exactly 448 * 2^k
    x[2, :] = torch.ldexp(torch.ones(K), torch.randint(-12, 0, (K,), generator=gen))    # powers of two
    x[3, ::2] = 1e-38                                           # tiny values next to normal ones
    pad = torch.zeros(M, K + 32)
    pad[:, :K] = x
    xs = pad.to(dtype)[:, :K]                                   # ld > K
    got = k.quant_rows_e4m3(xs.cuda())
    want = quant_rows_twin(xs)
    assert torch.equal(got.scale.cpu(), want.scale)
    assert torch.equal(got.q.cpu().view(torch.uint8), want.q.view(torch.uint8))
    assert float(got.q.cpu().float().abs().max()) <= E4M3_MAX


def test_quant_rows_rejects_misaligned_rows():
    k = _k()
    x = torch.randn(64, 776, device='cuda')
    with pytest.raises(RuntimeError, match='16-byte aligned'):
        k.quant_rows_e4m3(x[:, 2:770])                           # base 8 bytes off
    xb = torch.randn(64, 780, device='cuda').to(torch.bfloat16)
    with pytest.raises(RuntimeError, match='16-byte aligned'):
        k.quant_rows_e4m3(xb[:, :768])                           # row pitch 1560 bytes
    with pytest.raises(RuntimeError, match='multiple of 16'):
        k.quant_rows_e4m3(torch.randn(8, 104, device='cuda'))


# ------------------------------------------------------------------------------------------------ models
def _ts(g, attention_type):
    from videotransformer_pytorch_b200 import TimeSformer
    c = g.cfg
    m = TimeSformer(num_frames=c['num_frames'], img_size=c['img_size'], patch_size=c['patch_size'], embed_dims=c['embed_dims'],
                    num_heads=c['num_heads'], num_transformer_layers=c['num_transformer_layers'], attention_type=attention_type)
    m.load_state_dict(g.sd, strict=True)
    return m


def _vv(g, attention_type):
    from videotransformer_pytorch_b200 import ViViT
    c = g.cfg
    m = ViViT(num_frames=c['num_frames_in'], img_size=c['img_size'], patch_size=c['patch_size'], embed_dims=c['embed_dims'],
              num_heads=c['num_heads'], num_transformer_layers=c['num_transformer_layers'], attention_type=attention_type)
    m.load_state_dict(g.sd, strict=True)
    return m


# the goldens whose head dim (64) and width the GPU kernels take
CONFIGS = [('timesformer_hd64', _ts, 'divided_space_time'), ('timesformer_joint_n289', _ts, 'joint_space_time'),
           ('vivit_joint_hd64', _vv, 'joint_space_time'), ('vivit_divided_hd64', _vv, 'divided_space_time')]


def _emu_forward(build_model, x, fn=None):
    """The fp8 forward on the quantising fp64 emulation: same quantised operands, everything else in fp64."""
    from videotransformer_pytorch_b200 import _lib, ops
    old = _lib.K
    _lib.K = EmuKernels(exact=True, dtype=torch.float64, inference_forms=True, fp8_forms=True)
    ops.token_maps.cache_clear()
    ops.frame_maps.cache_clear()
    try:
        m = build_model().eval().set_inference_precision('fp8')
        with torch.no_grad():
            return (fn(m, x) if fn else m(x)).double()
    finally:
        _lib.K = old
        ops.token_maps.cache_clear()
        ops.frame_maps.cache_clear()


def _gpu_forward(build_model, x, precision, fn=None):
    m = build_model().cuda().eval().set_inference_precision(precision)
    with torch.no_grad():
        return (fn(m, x.cuda()) if fn else m(x.cuda())).double().cpu()


def _check_model(name, build_model, x, ref, fn=None):
    y16 = _gpu_forward(build_model, x, 'bf16', fn)
    y8 = _gpu_forward(build_model, x, 'fp8', fn)
    e16, e8 = rel_err(y16, ref), rel_err(y8, ref)
    e_emu = rel_err(_emu_forward(build_model, x, fn), ref)
    print(f'FP8-REPORT model {name}: rel-L2 vs fp64 oracle: bf16 {e16:.2e}, fp8 {e8:.2e}, fp8 emulation {e_emu:.2e}; '
          f'fp8 vs bf16 {rel_err(y8, y16):.2e}')
    assert e8 <= 1.5 * e_emu + e16, (name, e8, e_emu, e16)


@pytest.mark.parametrize('name,build,attention_type', CONFIGS, ids=[c[0] for c in CONFIGS])
def test_models_fp8_against_emulation_and_oracle(golden, name, build, attention_type):
    g = golden(name)
    _check_model(name, lambda: build(g, attention_type), g.x.float(), g.out['y_eval'].double())


@pytest.mark.parametrize('name', ['maskfeat_s32', 'maskfeat_s64'])
def test_maskfeat_fp8_against_emulation_and_oracle(maskfeat_golden, name):
    from videotransformer_pytorch_b200 import MaskFeat
    g = maskfeat_golden(name)
    sd = g.state(torch.float32)

    def build_model():
        m = MaskFeat(**g.kwargs)
        m.load_state_dict(sd, strict=True)
        return m
    fwd = lambda m, x: m.forward_features(x, g.mask.to(x.device))
    _check_model(name, build_model, g.x.float(), g.feats.double(), fwd)


def test_fp8_top1_agreement_synthetic():
    """TimeSformer-B (8 x 224) with trunc-normal weights and a 400-class head: top-1 agreement of fp8 with bf16 logits on
    random clips.  Random weights, not a trained checkpoint: this says nothing about accuracy on Kinetics."""
    from videotransformer_pytorch_b200 import ClassificationHead, TimeSformer
    torch.manual_seed(0)
    m = TimeSformer(num_frames=8, img_size=224, patch_size=16).cuda().eval()
    with torch.no_grad():
        for n, p in m.named_parameters():
            if 'temporal_fc' in n:
                p.normal_(std=0.02)
    head = ClassificationHead(400, 768).cuda()
    x = torch.randn(16, 8, 3, 224, 224, device='cuda')
    with torch.no_grad():
        l16 = head(m(x))
        m.set_inference_precision('fp8')
        l8 = head(m(x))
    agree = float((l16.argmax(1) == l8.argmax(1)).float().mean())
    print(f'FP8-REPORT synthetic TimeSformer-B batch 16: logits rel-L2 fp8 vs bf16 {rel_err(l8, l16):.2e}, '
          f'top-1 agreement {agree:.3f}')
    assert rel_err(l8, l16) < 0.2


# ------------------------------------------------------------------------------------------------ GraphedForward
def _tiny_ts(seed=0):
    from videotransformer_pytorch_b200 import TimeSformer
    torch.manual_seed(seed)
    m = TimeSformer(num_frames=4, img_size=48, patch_size=16, embed_dims=128, num_heads=2, num_transformer_layers=2)
    with torch.no_grad():
        for n, p in m.named_parameters():
            if 'temporal_fc' in n:
                p.normal_(std=0.05)
    return m.cuda()


def _train_step(m, x, lr=0.05, seed=11):
    m.train()
    torch.manual_seed(seed)
    loss = m(x).square().sum()
    loss.backward()
    grads = [p.grad.clone() for p in m.parameters()]
    with torch.no_grad():
        for p in m.parameters():
            p.sub_(lr * p.grad)
            p.grad = None
    m.eval()
    return loss.detach().clone(), grads


def test_graphed_forward_fp8_follows_training():
    from videotransformer_pytorch_b200.graph import GraphedForward
    m = _tiny_ts().eval().set_inference_precision('fp8')
    x = torch.randn(2, 4, 3, 48, 48, device='cuda')
    g = GraphedForward(lambda xx: m(xx), (x,))
    r1 = g(x).clone()
    with torch.no_grad():
        assert torch.equal(r1, m(x))
    _train_step(m, x)
    r2 = g(x).clone()
    with torch.no_grad():
        e2 = m(x)
    assert torch.equal(r2, e2), 'the replay did not re-quantise the updated weights'
    assert not torch.equal(r1, r2)


def test_fp8_inference_between_training_steps_leaves_training_unchanged():
    x = torch.randn(2, 4, 3, 48, 48, device='cuda')
    runs = []
    for prec in ('bf16', 'fp8'):
        m = _tiny_ts().eval().set_inference_precision(prec)
        out = []
        for step in range(2):
            with torch.inference_mode():
                m(x)
            out.append(_train_step(m, x, seed=20 + step))
        runs.append(out)
    for (l_a, g_a), (l_b, g_b) in zip(*runs):
        assert torch.equal(l_a, l_b)
        assert all(torch.equal(a, b) for a, b in zip(g_a, g_b))
