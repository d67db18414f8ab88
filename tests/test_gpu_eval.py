"""Forward-only evaluation path on the GPU: the 'gelu_h' GEMM epilogue against bf16 GEMM + GELU kernel, the kernels with
their statistics outputs left NULL against the calls that write them, the no_grad / inference_mode model forwards
against the grad-enabled eval forward, GraphedForward, the top-k counter kernel against torch, a linear-probe step and
inference mode between captured training steps.  -m gpu"""
import pytest
import torch

pytestmark = pytest.mark.gpu
SENTINEL = -12345.0


def K():
    from videotransformer_pytorch_b200 import _lib
    return _lib.K


def mk(shape, seed, scale=1.0):
    g = torch.Generator(device='cpu').manual_seed(seed)
    return (torch.randn(shape, generator=g) * scale).cuda()


# ------------------------------------------------------------------------------------------------ gelu_h GEMM
@pytest.mark.parametrize('staged', ['1', '0'], ids=['staged', 'register'])
@pytest.mark.parametrize('bn', [128, 192, 256])
def test_gelu_h_equals_bf16_gemm_then_gelu(bn, staged, monkeypatch):
    monkeypatch.setenv('VT_GEMM_STAGED_EPI', staged)
    k = K()
    Kd = 200
    for M, N in ((1, 8), (129, 200), (300, 776), (12552, 3072)):
        a, b, bias = mk((M, Kd), M, 0.3).bfloat16(), mk((N, Kd), N, 0.3).bfloat16(), mk((N,), 7)
        h = k.gemm(a, b, M, N, Kd, epi='gelu_h', bias=bias, force_bn=bn)
        ref = k.gelu(k.gemm(a, b, M, N, Kd, epi='bf16', bias=bias, force_bn=bn))
        assert torch.equal(h, ref), (bn, M, N)
        # and against the planner's own tile for the bf16 form (what the saving forward runs)
        assert torch.equal(h, k.gelu(k.gemm(a, b, M, N, Kd, epi='bf16', bias=bias))), (bn, M, N)


@pytest.mark.parametrize('staged', ['1', '0'], ids=['staged', 'register'])
@pytest.mark.parametrize('bn', [128, 192, 256])
def test_gelu_h_strided_output_keeps_guard_regions(bn, staged, monkeypatch):
    monkeypatch.setenv('VT_GEMM_STAGED_EPI', staged)
    k = K()
    M, N, Kd, PAD_C, PAD_R = 200, 200, 72, 56, 9
    a, b, bias = mk((M, Kd), 1, 0.3).bfloat16(), mk((N, Kd), 2, 0.3).bfloat16(), mk((N,), 3)
    buf = torch.full((M + PAD_R, N + PAD_C), SENTINEL, device='cuda').bfloat16()
    k.gemm(a, b, M, N, Kd, epi='gelu_h', bias=bias, force_bn=bn, out=buf[:M, :N])
    assert torch.equal(buf[:M, :N], k.gelu(k.gemm(a, b, M, N, Kd, epi='bf16', bias=bias, force_bn=bn)))
    assert bool((buf[M:] == SENTINEL).all()) and bool((buf[:, N:] == SENTINEL).all())


def test_gelu_h_under_graph_replay():
    k = K()
    M, N, Kd = 1000, 3072, 768
    a, b, bias = mk((M, Kd), 4, 0.3).bfloat16(), mk((N, Kd), 5, 0.3).bfloat16(), mk((N,), 6)
    k.gemm(a, b, M, N, Kd, epi='gelu_h', bias=bias)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        with torch.cuda.graph(g, stream=s):
            h = k.gemm(a, b, M, N, Kd, epi='gelu_h', bias=bias)
    torch.cuda.current_stream().wait_stream(s)
    a.copy_(mk((M, Kd), 9, 0.3).bfloat16())
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(h, k.gelu(k.gemm(a, b, M, N, Kd, epi='bf16', bias=bias)))


# ------------------------------------------------------------------------------------------------ NULL statistics
@pytest.mark.parametrize('N', [8, 9, 197, 290, 1569])
def test_attention_without_lse_equals_with(N):
    k = K()
    Bp, H, hd = (6 if N < 1000 else 2), 4, 64
    qkv = mk((Bp * N, 3 * H * hd), N, 0.5).bfloat16()
    if N <= 256:
        impls = [0, 1] + ([3] if N == 8 else []) + ([2] if N > 32 else [])
        for impl in impls:
            c1, lse, _ = k.attn_fwd(qkv, Bp, N, H, hd, hd ** -0.5, impl=impl)
            c0, none, _ = k.attn_fwd(qkv, Bp, N, H, hd, hd ** -0.5, impl=impl, want_lse=False)
            assert none is None and torch.equal(c0, c1), (N, impl)
    else:
        v5 = qkv.view(Bp, N, 3, H, hd)
        q4, k4, v4 = (v5[:, :, s].permute(0, 2, 1, 3) for s in range(3))
        for impl in (0, 1):                   # auto (tensor cores) and the CUDA-core kernels
            o1, _ = k.xattn_fwd(q4, k4, v4, hd ** -0.5, impl=impl)
            o0, none = k.xattn_fwd(q4, k4, v4, hd ** -0.5, impl=impl, want_lse=False)
            assert none is None and torch.equal(o0, o1), (N, impl)


@pytest.mark.parametrize('D,rows_map', [(768, False), (768, True), (96, False), (192, False)])
def test_layernorm_without_stats_equals_with(D, rows_map):
    k = K()
    x = mk((500, D), D)
    w, b = mk((D,), 1), mk((D,), 2)
    in_row = torch.randperm(500, device='cuda')[:321].int() if rows_map else None
    rows = 321 if rows_map else None
    for fp32 in (False, True):
        y1, m, r = k.ln_fwd(x, w, b, 1e-6, in_row=in_row, rows=rows, out_fp32=fp32)
        y0, m0, r0 = k.ln_fwd(x, w, b, 1e-6, in_row=in_row, rows=rows, out_fp32=fp32, stats=False)
        assert m0 is None and r0 is None and torch.equal(y0, y1)


@pytest.mark.parametrize('thw,stride', [((8, 56, 56), (1, 4, 4)), ((8, 28, 28), (1, 2, 2)), ((8, 14, 14), (1, 1, 1)),
                                        ((8, 7, 7), (1, 1, 1))])
def test_mvit_stage_pooling_and_maxpool_without_stats(thw, stride):
    """MViT-B stage shapes: q/k/v pooling + LayerNorm and the skip max-pool with pooled / mean / rstd / idx left NULL"""
    k = K()
    B, H, hd = 2, 2, 96
    T, Hh, W = thw
    N1 = 1 + T * Hh * W
    qkv = mk((B * N1, 3 * H * hd), 11, 0.5).bfloat16().view(B, N1, 3 * H * hd)
    src = qkv[:, :, H * hd:2 * H * hd]
    w, gm, bt = mk((hd, 27), 1, 0.2), mk((hd,), 2), mk((hd,), 3)
    o1, *_ = k.pool_fwd(src, H, hd, thw, stride, w, gm, bt, 1e-6)
    o0, pooled, mean, rstd, _ = k.pool_fwd(src, H, hd, thw, stride, w, gm, bt, 1e-6, stats=False)
    assert pooled is None and mean is None and rstd is None and torch.equal(o0, o1)
    x = mk((B, N1, H * hd), 4)
    kern = tuple(s + 1 if s > 1 else s for s in stride)
    y1, _, _ = k.maxpool_fwd(x, thw, kern, stride)
    y0, idx, _ = k.maxpool_fwd(x, thw, kern, stride, want_idx=False)
    assert idx is None and torch.equal(y0, y1)


# ------------------------------------------------------------------------------------------------ models
def _live(m):
    with torch.no_grad():
        for n, p in m.named_parameters():
            if 'temporal_fc' in n:
                p.normal_(std=0.05)
    return m


def _forms_equal(m, x):
    m = m.cuda().eval()
    y_grad = m(x)                               # grad enabled: the saving forward
    with torch.no_grad():
        y_ng = m(x)
    with torch.inference_mode():
        y_inf = m(x)
    assert y_grad.requires_grad
    assert torch.equal(y_ng, y_grad.detach()) and torch.equal(y_inf, y_ng)


@pytest.mark.parametrize('attention_type', ['divided_space_time', 'space_only', 'joint_space_time'])
@pytest.mark.parametrize('side', [224, 320])
def test_timesformer_forward_only_equals_grad_forward(attention_type, side):
    from videotransformer_pytorch_b200 import TimeSformer
    torch.manual_seed(0)
    frames = 8 if attention_type != 'joint_space_time' else 4
    m = _live(TimeSformer(num_frames=frames, img_size=224, patch_size=16, embed_dims=256, num_heads=4,
                          num_transformer_layers=2, attention_type=attention_type))
    _forms_equal(m, torch.randn(2, frames, 3, side, side, device='cuda'))


@pytest.mark.parametrize('attention_type', ['fact_encoder', 'joint_space_time', 'divided_space_time'])
def test_vivit_forward_only_equals_grad_forward(attention_type):
    from videotransformer_pytorch_b200 import ViViT
    torch.manual_seed(0)
    m = _live(ViViT(num_frames=8, img_size=64, patch_size=16, embed_dims=256, num_heads=4, num_transformer_layers=2,
                    attention_type=attention_type))
    _forms_equal(m, torch.randn(2, 8, 3, 64, 64, device='cuda'))


def test_maskfeat_features_with_head_forward_only_equals_grad_forward():
    from videotransformer_pytorch_b200 import ClassificationHead, MaskFeat
    torch.manual_seed(0)
    mf = MaskFeat(pool_q_stride_size=[[1, 1, 2, 2], [3, 1, 2, 2]], feature_dim=2 * 2 * 2 * 3 * 9).cuda().eval()
    head = ClassificationHead(400, mf.mvit.norm_embed.normalized_shape[0]).cuda()
    x = torch.randn(2, 16, 3, 224, 224, device='cuda')
    y_grad = head(mf.forward_features(x)[:, 0])
    with torch.no_grad():
        y_ng = head(mf.forward_features(x)[:, 0])
    with torch.inference_mode():
        y_inf = head(mf.forward_features(x)[:, 0])
    assert torch.equal(y_ng, y_grad.detach()) and torch.equal(y_inf, y_ng)


# ------------------------------------------------------------------------------------------------ GraphedForward
class Net(torch.nn.Module):
    def __init__(self, layers=3):
        super().__init__()
        from videotransformer_pytorch_b200 import ClassificationHead, TimeSformer
        self.model = _live(TimeSformer(num_frames=4, img_size=48, patch_size=16, embed_dims=128, num_heads=2,
                                       num_transformer_layers=layers))
        self.head = ClassificationHead(10, 128)

    def forward(self, x):
        return self.head(self.model(x))


def test_graphed_forward_matches_eager_and_tracks_training():
    from videotransformer_pytorch_b200 import _lib
    from videotransformer_pytorch_b200.graph import GraphedForward
    torch.manual_seed(0)
    net = Net().cuda().eval()
    x = torch.randn(2, 4, 3, 48, 48, device='cuda')
    fwd = GraphedForward(net, (x,))
    for trial in range(2):
        x2 = torch.randn(2, 4, 3, 48, 48, device='cuda')
        got = fwd(x2).clone()
        with torch.no_grad():
            want = net(x2)
        assert torch.equal(got, want), trial
        with torch.no_grad():                  # an optimizer step between validations
            for p in net.parameters():
                p.add_(0.01 * torch.randn_like(p))
    # one launch per kernel of the training forward, minus the stand-alone GELU of every FFN
    torch.cuda.synchronize()
    l0 = _lib.launch_count()
    net(x)
    torch.cuda.synchronize()
    train_fwd = _lib.launch_count() - l0
    assert fwd.kernels_per_replay == train_fwd - 3, (fwd.kernels_per_replay, train_fwd)


def test_graphed_forward_refuses_training_mode():
    from videotransformer_pytorch_b200.graph import GraphedForward
    net = Net().cuda().train()
    with pytest.raises(RuntimeError, match='eval mode'):
        GraphedForward(net, (torch.randn(2, 4, 3, 48, 48, device='cuda'),))


# ------------------------------------------------------------------------------------------------ top-k counters
@pytest.mark.parametrize('views', [1, 3])
@pytest.mark.parametrize('C', [400, 600])
def test_topk_hits_counts_equal_torch(views, C):
    from videotransformer_pytorch_b200.metrics import TopKAccuracy
    acc = TopKAccuracy(top_k=(1, 5, 10, 50), views=views, device='cuda')
    want, seen = {1: 0, 5: 0, 10: 0, 50: 0}, 0
    gen = torch.Generator().manual_seed(C + views)
    for B in (1, 5, 33, 64):
        logits = torch.randn(B * views, C, generator=gen) * 3.0
        labels = torch.randint(0, C, (B,), generator=gen)
        logits[torch.arange(B) * views, labels] += 4.0
        probs = acc.update(logits.cuda(), labels.cuda(), want_probs=True)
        mean = logits.cuda().view(B, views, C).mean(1)
        ref_probs = mean.softmax(-1)
        assert (probs - ref_probs).abs().max() < 1e-6
        for k in want:
            want[k] += int((ref_probs.topk(k, dim=-1).indices == labels.cuda()[:, None]).any(-1).sum())
        seen += B
    assert acc.compute() == {k: want[k] / seen for k in want}
    acc.reset()
    acc.update(torch.zeros(2 * views, C, device='cuda'), torch.tensor([0, C - 1], device='cuda'))
    assert acc.compute() == {1: 1.0, 5: 1.0, 10: 1.0, 50: 1.0}        # all tied: rank 0


def test_topk_hits_inside_graphed_forward():
    from videotransformer_pytorch_b200.graph import GraphedForward
    from videotransformer_pytorch_b200.metrics import TopKAccuracy
    torch.manual_seed(1)
    net = Net(layers=1).cuda().eval()
    acc = TopKAccuracy(top_k=(1, 5), views=3, device='cuda')

    def step(x, y):
        logits = net(x)
        acc.update(logits, y)
        return logits

    x, y = torch.randn(6, 4, 3, 48, 48, device='cuda'), torch.tensor([1, 2], device='cuda')
    fwd = GraphedForward(step, (x, y))
    hits1 = hits5 = 0
    for _ in range(3):
        x2, y2 = torch.randn(6, 4, 3, 48, 48, device='cuda'), torch.randint(0, 10, (2,), device='cuda')
        logits = fwd(x2, y2)
        p = logits.view(2, 3, 10).mean(1).softmax(-1)
        hits1 += int((p.topk(1).indices == y2[:, None]).any(-1).sum())
        hits5 += int((p.topk(5).indices == y2[:, None]).any(-1).sum())
    assert acc.compute() == {1: hits1 / 6, 5: hits5 / 6}


def test_readme_eval_pattern_counts_only_the_replayed_batches():
    """The README's evaluation loop as written (no reset): the example batch GraphedForward warms up on is not counted,
    also when it is the loader's first batch."""
    from videotransformer_pytorch_b200 import TopKAccuracy
    from videotransformer_pytorch_b200.graph import GraphedForward
    torch.manual_seed(2)
    net = Net(layers=1).cuda().eval()
    model, head = net.model, net.head
    gen = torch.Generator().manual_seed(3)
    loader = [(torch.randn(6, 4, 3, 48, 48, generator=gen).cuda(), torch.randint(0, 10, (2,), generator=gen).cuda())
              for _ in range(3)]
    x, y = loader[0]

    acc = TopKAccuracy(top_k=(1, 5), views=3, device='cuda')
    def test_step(x, y):
        logits = head(model(x))
        acc.update(logits, y)
        return logits
    step = GraphedForward(test_step, (x, y))
    want = {1: 0, 5: 0}
    for x, y in loader:
        logits = step(x, y)
        p = logits.view(2, 3, 10).mean(1).softmax(-1)
        for k in want:
            want[k] += int((p.topk(k).indices == y[:, None]).any(-1).sum())
    assert acc.compute() == {k: want[k] / 6 for k in want}
    assert int(acc._counts[-1]) == 6                                    # samples: the three replayed batches only


# ------------------------------------------------------------------------------------------------ probe / inference mode
def test_linear_probe_graphed_step_matches_eager():
    """linear_prob: backbone under no_grad in eval mode, head trained; captured step == eager step."""
    from videotransformer_pytorch_b200 import ClassificationHead, TimeSformer, cross_entropy
    from videotransformer_pytorch_b200.graph import GraphedTrainStep
    torch.manual_seed(0)
    backbone = _live(TimeSformer(num_frames=4, img_size=48, patch_size=16, embed_dims=128, num_heads=2,
                                 num_transformer_layers=2)).cuda().eval()
    head = ClassificationHead(10, 128).cuda()

    def loss_fn(x, y):
        with torch.no_grad():
            f = backbone(x)
        return cross_entropy(head(f), y)

    x, y = torch.randn(2, 4, 3, 48, 48, device='cuda'), torch.tensor([3, 8], device='cuda')
    step = GraphedTrainStep(loss_fn, (x, y), params=list(head.parameters()))
    x2 = torch.randn(2, 4, 3, 48, 48, device='cuda')
    step(x2, y)
    got = [p.grad.clone() for p in head.parameters()]
    for p in head.parameters():
        p.grad = None
    loss_fn(x2, y).backward()
    assert all(torch.equal(a, p.grad) for a, p in zip(got, head.parameters()))
    assert all(p.grad is None for p in backbone.parameters())


def test_inference_mode_eval_then_captured_training_then_eval():
    from videotransformer_pytorch_b200 import ops
    from videotransformer_pytorch_b200.graph import GraphedTrainStep
    ops.token_maps.cache_clear()
    torch.manual_seed(0)
    net = Net(layers=2).cuda()
    x, y = torch.randn(2, 4, 3, 48, 48, device='cuda'), torch.tensor([1, 7], device='cuda')
    net.eval()
    with torch.inference_mode():
        e0 = net(x)
    net.train()
    step = GraphedTrainStep(lambda a, b: torch.nn.functional.cross_entropy(net(a), b), (x, y), params=list(net.parameters()))
    loss = float(step(x, y))
    assert loss == loss
    net.eval()
    with torch.inference_mode():
        e1 = net(x)
    assert e0.shape == e1.shape and bool(torch.isfinite(e1).all())
