"""FP8 inference forms, host side, on the CPU: the quantiser twin against an exact fp64 restatement of e4m3 rounding, and
the fp8 forward-only forms of the models on the emulated kernel table (which launches they issue, that grad-enabled calls
never take them, shadow re-quantisation, and the errors)."""
import math

import pytest
import torch

from tests.conftest import rel_err
from tests.emu_fp8 import e4m3_cast, e4m3_round_fp64, quant_rows_twin
from tests.emu_kernels import EmuKernels


def _e4m3_grid():
    """Every finite non-negative e4m3 value, ascending."""
    v = torch.arange(256, dtype=torch.uint8).view(torch.float8_e4m3fn).double()
    return torch.unique(v[torch.isfinite(v) & (v >= 0)])


def test_restatement_is_the_e4m3_grid():
    g = _e4m3_grid()
    assert g.numel() == 127 and float(g[-1]) == 448.0 and float(g[1]) == 2.0 ** -9
    assert torch.equal(e4m3_round_fp64(g), g) and torch.equal(e4m3_round_fp64(-g), -g)
    mids = (g[1:] + g[:-1]) / 2                                    # ties: the neighbour with an even mantissa wins
    r = e4m3_round_fp64(mids)
    codes = r.float().to(torch.float8_e4m3fn).view(torch.uint8)
    assert bool(((codes & 1) == 0).all())
    assert bool(((r == g[1:]) | (r == g[:-1])).all())


def test_cast_twin_matches_restatement():
    g = _e4m3_grid()
    mids = (g[1:] + g[:-1]) / 2
    gen = torch.Generator().manual_seed(0)
    rnd = torch.ldexp(torch.rand(20000, generator=gen, dtype=torch.float64) + 0.5,
                      torch.randint(-14, 10, (20000,), generator=gen))
    vals = torch.cat([g, mids, mids + 2.0 ** -40, mids - 2.0 ** -40, rnd,
                      torch.tensor([448.0, 449.0, 464.0, 480.0, 500.0, 1e6, 2.0 ** -10, 2.0 ** -10 + 2.0 ** -30, 2.0 ** -11])])
    vals = torch.cat([vals, -vals]).float().double()               # fp32 inputs, as the kernel sees them
    twin = e4m3_cast(vals).double()
    assert torch.equal(twin, e4m3_round_fp64(vals))
    assert float(e4m3_cast(torch.tensor([1e6])).float()) == 448.0   # saturates, no NaN


@pytest.mark.parametrize('dtype', [torch.float32, torch.bfloat16])
@pytest.mark.parametrize('K', [96, 768, 3072])
def test_quant_rows_twin(dtype, K):
    gen = torch.Generator().manual_seed(K)
    M = 37
    x = torch.randn(M, K, generator=gen) * torch.ldexp(torch.ones(M, 1), torch.randint(-20, 20, (M, 1), generator=gen))
    x[3] = 0.0                                                      # zero row -> scale 1, q zero
    x[5, :] = 0.25
    x[5, 7] = -448.0 * 2.0 ** -6                                    # amax exactly 448 * 2^k
    x[6, :] = 0.5
    x[6, 1] = 2.0 ** 5                                              # amax exactly a power of two
    x = x.to(dtype)
    q = quant_rows_twin(x)
    xs = x.double()
    amax = xs.abs().amax(1)
    want = torch.tensor([1.0 if a == 0 else 2.0 ** math.ceil(math.log2(a / 448.0)) for a in amax.tolist()], dtype=torch.float64)
    assert torch.equal(q.scale.double(), want)
    assert float(q.scale[3]) == 1.0 and not bool(q.q[3].float().any())
    assert float(q.scale[5]) == 2.0 ** -6 and float(q.q[5, 7].float()) == -448.0
    assert float(q.scale[6]) == 2.0 ** -3
    assert torch.equal(q.q.double(), e4m3_round_fp64(xs / q.scale.double()[:, None]))
    ratio = (q.q.double().abs().amax(1) / 448.0)[amax > 0]
    assert bool((ratio >= 0.5).all() & (ratio <= 1.0).all())         # the scale uses the top binade of e4m3


# ------------------------------------------------------------------------------------------------ host logic
@pytest.fixture
def table():
    from videotransformer_pytorch_b200 import _lib, ops
    old = _lib.K
    _lib.K = EmuKernels(exact=True, inference_forms=True, fp8_forms=True)
    ops.token_maps.cache_clear()
    ops.frame_maps.cache_clear()
    yield _lib.K
    _lib.K = old


def _tiny(kind='timesformer', attention_type=None):
    from videotransformer_pytorch_b200 import TimeSformer, ViViT
    torch.manual_seed(0)
    if kind == 'timesformer':
        m = TimeSformer(num_frames=4, img_size=32, patch_size=16, embed_dims=64, num_heads=2, num_transformer_layers=2,
                        attention_type=attention_type or 'divided_space_time')
    else:
        m = ViViT(num_frames=4, img_size=32, patch_size=16, embed_dims=64, num_heads=2, num_transformer_layers=2,
                  attention_type=attention_type or 'fact_encoder')
    with torch.no_grad():
        for n, p in m.named_parameters():
            if 'temporal_fc' in n:
                p.normal_(std=0.05)
    return m.eval()


def _gemms(calls):
    return [c for c in calls if c[0] in ('gemm', 'gemm_e4m3')]


MODELS = [('timesformer', 'divided_space_time'), ('timesformer', 'space_only'), ('timesformer', 'joint_space_time'),
          ('vivit', 'fact_encoder'), ('vivit', 'joint_space_time'), ('vivit', 'divided_space_time')]


@pytest.mark.parametrize('kind,attention_type', MODELS, ids=[f'{a}-{b}' for a, b in MODELS])
def test_fp8_forward_only_launches(table, kind, attention_type):
    """Every block linear of the forward-only form runs as quantise-A + e4m3 GEMM with the bf16 form's shape and epilogue;
    the patch embedding stays bf16; weights are quantised once and then served from the shadow cache."""
    m = _tiny(kind, attention_type)
    x = torch.randn(2, 4, 3, 32, 32)
    with torch.no_grad():
        y16 = m(x)
    bf16 = [c for c in _gemms(table.calls) if not (c[4] is False and c[5] is True)]   # minus the W_f W_p product
    m.set_inference_precision('fp8')
    with torch.no_grad():
        m(x)                                                       # first call quantises the weights
    table.calls.clear()
    with torch.no_grad():
        y8 = m(x)
    calls = list(table.calls)
    g8 = _gemms(calls)
    assert [c[1:] for c in g8] == [c[1:] for c in bf16]
    assert g8[0][0] == 'gemm' and all(c[0] == 'gemm_e4m3' for c in g8[1:])          # patch embed bf16, the rest e4m3
    for i, c in enumerate(calls):
        if c[0] == 'gemm_e4m3':                                    # A quantised per token right before, M x K rows
            assert calls[i - 1][0] == 'quant_rows_e4m3' and calls[i - 1][1:] == (c[1], c[3]), (calls[i - 1], c)
    n_quant = sum(c[0] == 'quant_rows_e4m3' for c in calls)
    assert n_quant == len(g8) - 1                                  # cached shadows: no weight is re-quantised
    assert 0 < rel_err(y8, y16) < 0.1
    with torch.inference_mode():
        assert torch.equal(m(x), y8)


def test_fp8_grad_enabled_calls_are_untouched(table):
    """A grad-enabled forward ignores the precision: same launches, loss and gradients as a model without fp8 set."""
    x = torch.randn(2, 4, 3, 32, 32)
    runs = []
    for prec in ('bf16', 'fp8'):
        m = _tiny().train()
        m.set_inference_precision(prec)
        table.calls.clear()
        torch.manual_seed(3)
        y = m(x)
        y.square().sum().backward()
        assert not any(c[0] in ('quant_rows_e4m3', 'gemm_e4m3') for c in table.calls)
        runs.append((y.detach(), [p.grad.clone() for p in m.parameters()], list(table.calls)))
    assert torch.equal(runs[0][0], runs[1][0]) and runs[0][2] == runs[1][2]
    assert all(torch.equal(a, b) for a, b in zip(runs[0][1], runs[1][1]))
    # eval mode with parameters requiring grad and grad mode on: autograd records, so still the bf16 saving form
    m = _tiny().set_inference_precision('fp8')
    table.calls.clear()
    m(x)
    assert not any(c[0] in ('quant_rows_e4m3', 'gemm_e4m3') for c in table.calls)


def test_fp8_shadows_requantise_on_parameter_change(table):
    m = _tiny().set_inference_precision('fp8')
    x = torch.randn(1, 4, 3, 32, 32)
    ffn = m.transformer_layers.layers[0].ffns[0]
    tmp = m.transformer_layers.layers[0].attentions[0]
    with torch.no_grad():
        y0 = m(x)
        w1, wc = ffn._shadow._cache['w1:e4m3'], tmp.attn._shadow._cache['wc:e4m3']
        m(x)
        assert ffn._shadow._cache['w1:e4m3'] is w1 and tmp.attn._shadow._cache['wc:e4m3'] is wc
        ffn.layers[0][0].weight.mul_(2.0)                         # version bump: an optimizer step or load_state_dict
        tmp.attn.proj.weight.add_(0.01)
        y1 = m(x)
    w1b, wcb = ffn._shadow._cache['w1:e4m3'][1], tmp.attn._shadow._cache['wc:e4m3'][1]
    assert torch.equal(w1b.scale, 2 * w1[1].scale) and torch.equal(w1b.q.float(), w1[1].q.float())
    assert not torch.equal(wcb.q.float(), wc[1].q.float())
    assert not torch.equal(y0, y1)
    # the product weight is W_f W_p of the bf16 shadows, quantised per output channel
    D = 64
    prod = table.gemm(tmp.attn._shadow.get('temporal_fc', tmp.temporal_fc.weight), tmp.attn._shadow.get('proj', tmp.attn.proj.weight),
                      D, D, D, b_mn=True, epi='f32')
    assert torch.allclose(prod.double(), tmp.temporal_fc.weight.double() @ tmp.attn.proj.weight.double(), rtol=1e-5, atol=1e-7)
    want = quant_rows_twin(prod)
    assert prod.shape == (D, D) and torch.equal(wcb.q.float(), want.q.float()) and torch.equal(wcb.scale, want.scale)


def test_fp8_maskfeat_forward_only(table, maskfeat_golden):
    from tests.test_host_logic_mvit import build
    g = maskfeat_golden('maskfeat_s32')
    m = build(g).eval()
    with torch.no_grad():
        f16 = m.forward_features(g.x, g.mask)
    bf16 = _gemms(table.calls)
    m.set_inference_precision('fp8')
    with torch.no_grad():
        m.forward_features(g.x, g.mask)
    table.calls.clear()
    with torch.no_grad():
        f8 = m.forward_features(g.x, g.mask)
    g8 = _gemms(table.calls)
    assert [c[1:] for c in g8] == [c[1:] for c in bf16]
    assert g8[0][0] == 'gemm' and all(c[0] == 'gemm_e4m3' for c in g8[1:])
    n_blocks = len(m.mvit.blocks)
    n_proj = sum(b.dim != b.dim_out for b in m.mvit.blocks)
    assert len(g8) - 1 == 4 * n_blocks + n_proj
    # FC1 and the width-changing proj share one quantisation of norm2(x)
    assert sum(c[0] == 'quant_rows_e4m3' for c in table.calls) == 4 * n_blocks
    # each e4m3 operand carries ~2.7 % rel-L2 rounding error; over the 16 random-weight blocks of this MViT it grows to
    # ~21 % of the features (the exact emulation of the same quantisation against the fp64 oracle shows the same)
    assert 0 < rel_err(f8, f16) < 0.3


def test_fp8_errors(table, monkeypatch):
    from videotransformer_pytorch_b200 import MaskFeat, _lib
    m = _tiny()
    with pytest.raises(ValueError):
        m.set_inference_precision('fp16')
    with pytest.raises(ValueError):
        m.set_inference_precision('FP8')
    assert m.transformer_layers.layers[0].ffns[0].inference_precision == 'bf16'
    assert hasattr(MaskFeat, 'set_inference_precision')
    # non-sm_90 CUDA device
    monkeypatch.setattr(torch.cuda, 'get_device_capability', lambda d=None: (8, 0))
    with pytest.raises(RuntimeError, match='sm_90'):
        _lib.check_fp8_device('cuda:0')
    monkeypatch.setattr(torch.cuda, 'get_device_capability', lambda d=None: (9, 0))
    _lib.check_fp8_device('cuda:0')
    # a kernel table without the e4m3 forms: no fallback to bf16
    m.set_inference_precision('fp8')
    _lib.K = EmuKernels(exact=True, inference_forms=True, fp8_forms=False)
    with pytest.raises(RuntimeError, match='no fp8 forms'), torch.no_grad():
        m(torch.randn(1, 4, 3, 32, 32))
    m.set_inference_precision('bf16')
    with torch.no_grad():
        m(torch.randn(1, 4, 3, 32, 32))
