"""Host-side logic (row maps, cls handling, DropPath draws, backward formulas, state-dict surface) checked
on CPU against the reference-generated goldens, with the kernel table replaced by tests/emu_kernels.py."""
import pytest
import torch

from tests.conftest import check_grads, rel_err


def build_ts(g):
    from videotransformer_pytorch_b200 import TimeSformer
    c = g.cfg
    m = TimeSformer(num_frames=c['num_frames'], img_size=c['img_size'], patch_size=c['patch_size'],
                    embed_dims=c['embed_dims'], num_heads=c['num_heads'],
                    num_transformer_layers=c['num_transformer_layers'], attention_type='divided_space_time')
    missing = m.load_state_dict(g.sd, strict=True)
    return m


def build_vv(g):
    from videotransformer_pytorch_b200 import ViViT
    c = g.cfg
    m = ViViT(num_frames=c['num_frames_in'], img_size=c['img_size'], patch_size=c['patch_size'],
              embed_dims=c['embed_dims'], num_heads=c['num_heads'],
              num_transformer_layers=c['num_transformer_layers'], attention_type='fact_encoder')
    m.load_state_dict(g.sd, strict=True)
    return m


@pytest.mark.parametrize('name', ['timesformer_tiny', 'timesformer_hd64'])
def test_timesformer_state_dict_keys_match_reference(golden, name):
    g = golden(name)
    m = build_ts(g)
    assert list(m.state_dict().keys()) == list(g.sd.keys())
    for k, v in m.state_dict().items():
        assert tuple(v.shape) == tuple(g.sd[k].shape), k


@pytest.mark.parametrize('name', ['timesformer_tiny', 'timesformer_hd64'])
def test_timesformer_eval_tokens_attention(golden, emu, name):
    g = golden(name)
    m = build_ts(g).eval()
    with torch.no_grad():
        y = m(g.x)
        tok, b = m.prepare_tokens(g.x)
        attn = m.get_last_selfattention(g.x)
    assert rel_err(tok, g.out['tokens']) < 1e-5
    assert rel_err(y, g.out['y_eval']) < 2e-5
    assert attn.shape == g.out['last_attn'].shape
    assert rel_err(attn, g.out['last_attn']) < 2e-5


@pytest.mark.parametrize('name', ['timesformer_tiny', 'timesformer_hd64'])
def test_timesformer_train_forward_backward(golden, emu, name):
    g = golden(name)
    m = build_ts(g).train()
    x = g.x.clone().requires_grad_(True)
    torch.manual_seed(g.train_seed)
    y = m(x)
    assert rel_err(y, g.out['y_train']) < 2e-5
    (y.double() * g.out['loss_w']).sum().backward()
    assert rel_err(x.grad, g.out['dx']) < 1e-4
    grads = {n: p.grad for n, p in m.named_parameters()}
    assert all(v is not None for v in grads.values())
    check_grads(grads, g, 2e-4)


@pytest.mark.parametrize('name', ['vivit_tiny_b1', 'vivit_tiny_b3'])
def test_vivit_forward_backward(golden, emu, name):
    g = golden(name)
    m = build_vv(g)
    assert list(m.state_dict().keys()) == list(g.sd.keys())
    m.eval()
    with torch.no_grad():
        assert rel_err(m(g.x), g.out['y_eval']) < 2e-5
    m.train()
    x = g.x.clone().requires_grad_(True)
    torch.manual_seed(g.train_seed)
    y = m(x)
    assert rel_err(y, g.out['y_train']) < 2e-5
    (y.double() * g.out['loss_w']).sum().backward()
    assert rel_err(x.grad, g.out['dx']) < 1e-4
    check_grads({n: p.grad for n, p in m.named_parameters()}, g, 2e-4)


def test_standalone_modules_shapes(emu):
    from videotransformer_pytorch_b200 import Attention, FFNWithPreNorm, PatchEmbed
    torch.manual_seed(0)
    a = Attention(64, num_heads=4, qkv_bias=True)
    out, attn = a(torch.randn(3, 5, 64))
    assert out.shape == (3, 5, 64) and attn.shape == (3, 4, 5, 5)
    assert torch.allclose(attn.sum(-1), torch.ones(3, 4, 5), atol=1e-5)
    f = FFNWithPreNorm(embed_dims=64, hidden_channels=256)
    assert f(torch.randn(2, 7, 64)).shape == (2, 7, 64)
    pe = PatchEmbed(img_size=32, patch_size=16, embed_dims=64, conv_type='Conv2d')
    x = torch.randn(2, 3, 3, 32, 32)
    y = pe(x)
    ref = torch.nn.functional.conv2d(x.reshape(6, 3, 32, 32), pe.projection.weight, pe.projection.bias, stride=16)
    ref = ref.flatten(2).transpose(1, 2)
    assert rel_err(y, ref) < 1e-5


def test_timesformer_space_only(golden, emu):
    from videotransformer_pytorch_b200 import TimeSformer
    g = golden('timesformer_space_only_tiny')
    c = g.cfg
    m = TimeSformer(num_frames=c['num_frames'], img_size=c['img_size'], patch_size=c['patch_size'],
                    embed_dims=c['embed_dims'], num_heads=c['num_heads'],
                    num_transformer_layers=c['num_transformer_layers'], attention_type='space_only')
    assert list(m.state_dict().keys()) == list(g.sd.keys())          # no time_embed in space_only
    m.load_state_dict(g.sd, strict=True)
    m.eval()
    with torch.no_grad():
        assert rel_err(m(g.x), g.out['y_eval']) < 2e-5
    m.train()
    torch.manual_seed(g.train_seed)
    y = m(g.x)
    assert rel_err(y, g.out['y_train']) < 2e-5
    (y.double() * g.out['loss_w']).sum().backward()
    check_grads({n: p.grad for n, p in m.named_parameters()}, g, 2e-4)


@pytest.mark.parametrize('name', ['timesformer_joint_tiny', 'timesformer_joint_n289'])
def test_timesformer_joint_space_time_through_vt_attn(golden, emu, name):
    """joint_space_time (video_transformer.py:104-116): the packed-qkv attention vt_attn_* takes every sequence length,
    17 tokens and 289 tokens (past the 256 of the single-pass kernels) alike; the pooling attention vt_xattn_* never runs."""
    from videotransformer_pytorch_b200 import TimeSformer
    g = golden(name)
    c = g.cfg
    m = TimeSformer(num_frames=c['num_frames'], img_size=c['img_size'], patch_size=c['patch_size'],
                    embed_dims=c['embed_dims'], num_heads=c['num_heads'],
                    num_transformer_layers=c['num_transformer_layers'], attention_type='joint_space_time')
    assert list(m.state_dict().keys()) == list(g.sd.keys())
    m.load_state_dict(g.sd, strict=True)
    m.eval()
    with torch.no_grad():
        assert rel_err(m(g.x), g.out['y_eval']) < 2e-5
    m.train()
    torch.manual_seed(g.train_seed)
    y = m(g.x)
    assert rel_err(y, g.out['y_train']) < 2e-5
    (y.double() * g.out['loss_w']).sum().backward()
    check_grads({n: p.grad for n, p in m.named_parameters()}, g, 2e-4)
    n = 1 + c['num_frames'] * (c['img_size'] // c['patch_size']) ** 2
    assert n == (289 if name == 'timesformer_joint_n289' else 17)
    assert ('attn_fwd', True, n) in emu.calls and ('attn_bwd', n) in emu.calls
    assert not any(c_[0].startswith('xattn') for c_ in emu.calls)


def test_timesformer_accepts_uint8_clip(golden, emu):
    """SURVEY §8f rank 2: the decoder's uint8 clip [B,T,H,W,3] with ToTensor + Normalize folded into the patch operand
    gives what the reference computes from the CPU-normalised float clip."""
    from videotransformer_pytorch_b200 import TimeSformer
    g = golden('timesformer_tiny')
    c = g.cfg
    m = TimeSformer(num_frames=c['num_frames'], img_size=c['img_size'], patch_size=c['patch_size'],
                    embed_dims=c['embed_dims'], num_heads=c['num_heads'],
                    num_transformer_layers=c['num_transformer_layers'], attention_type='divided_space_time')
    m.load_state_dict(g.sd, strict=True)
    m.eval()
    mean, std = (0.485, 0.456, 0.406), (0.229, 0.224, 0.225)
    m.set_input_normalization(mean, std)
    u8 = torch.randint(0, 256, (2, c['num_frames'], c['img_size'], c['img_size'], 3), dtype=torch.uint8,
                       generator=torch.Generator().manual_seed(0))
    xf = (u8.float() / 255.0 - torch.tensor(mean)) / torch.tensor(std)          # ToTensor + Normalize
    with torch.no_grad():
        y8 = m(u8)
        yf = m(xf.permute(0, 1, 4, 2, 3).contiguous())
    assert rel_err(y8, yf) < 1e-5
    m.train()
    m(u8).sum().backward()                        # parameters still get gradients; the byte clip has none
    assert all(p.grad is not None for p in m.parameters())


@pytest.mark.parametrize('name,attention_type', [('vivit_joint_tiny', 'joint_space_time'),
                                                 ('vivit_divided_tiny', 'divided_space_time')])
def test_vivit_joint_and_divided_variants(golden, emu, name, attention_type):
    """ViViT models 1 and 3 (reference video_transformer.py:349-373): state-dict surface, eval and train-mode forward and
    all gradients against goldens generated by the real reference class."""
    from videotransformer_pytorch_b200 import ViViT
    g = golden(name)
    c = g.cfg
    m = ViViT(num_frames=c['num_frames_in'], img_size=c['img_size'], patch_size=c['patch_size'],
              embed_dims=c['embed_dims'], num_heads=c['num_heads'],
              num_transformer_layers=c['num_transformer_layers'], attention_type=attention_type)
    assert list(m.state_dict().keys()) == list(g.sd.keys())
    m.load_state_dict(g.sd, strict=True)
    m.eval()
    with torch.no_grad():
        assert rel_err(m(g.x), g.out['y_eval']) < 2e-5
    m.train()
    torch.manual_seed(g.train_seed)
    y = m(g.x)
    assert rel_err(y, g.out['y_train']) < 2e-5
    (y.double() * g.out['loss_w']).sum().backward()
    check_grads({n: p.grad for n, p in m.named_parameters()}, g, 2e-4)
