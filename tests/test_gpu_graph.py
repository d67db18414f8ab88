"""CUDA-graph captured training step == eager step (same DropPath draws, same grads).  -m gpu"""
import pytest
import torch

pytestmark = pytest.mark.gpu


class Net(torch.nn.Module):
    def __init__(self):
        super().__init__()
        from videotransformer_pytorch_b200 import ClassificationHead, TimeSformer
        self.model = TimeSformer(num_frames=4, img_size=48, patch_size=16, embed_dims=128, num_heads=2,
                                 num_transformer_layers=3)
        self.head = ClassificationHead(10, 128)
        with torch.no_grad():
            for n, p in self.model.named_parameters():
                if 'temporal_fc' in n:
                    p.normal_(std=0.05)

    def forward(self, x, y):
        return torch.nn.functional.cross_entropy(self.head(self.model(x)), y)


def test_graphed_step_matches_eager_and_tracks_weight_updates():
    from videotransformer_pytorch_b200.graph import GraphedTrainStep
    torch.manual_seed(0)
    net = Net().cuda().train()
    x = torch.randn(2, 4, 3, 48, 48).cuda()
    y = torch.tensor([1, 7]).cuda()
    step = GraphedTrainStep(net, (x, y))
    for trial in range(2):
        x2 = torch.randn(2, 4, 3, 48, 48).cuda()
        for g in step.static_grads:              # no gradient may depend on what its storage held before the replay
            g.fill_(float('nan'))
        torch.manual_seed(123 + trial)
        loss_g = float(step(x2, y).detach())
        gg = {n: p.grad.clone() for n, p in net.named_parameters()}
        nonfinite = [n for n, g in gg.items() if not bool(torch.isfinite(g).all())]
        assert not nonfinite, nonfinite
        for p in net.parameters():
            p.grad = None
        torch.manual_seed(123 + trial)
        loss_e = net(x2, y)
        loss_e.backward()
        assert abs(loss_g - float(loss_e)) < 1e-5, (loss_g, float(loss_e))
        bad = [n for n, p in net.named_parameters() if not torch.allclose(gg[n], p.grad, rtol=1e-4, atol=1e-6)]
        assert not bad, (len(bad), bad[:10])
        # emulate an optimizer step: the next replay must see the new weights (shadows re-cast in-graph)
        with torch.no_grad():
            for p in net.parameters():
                p.add_(0.01 * torch.randn_like(p))
