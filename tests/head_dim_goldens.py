"""The TimeSformer / ViViT fixtures at head widths 32, 96 and 128 (oracle/make_golden_head_dims.py) and the model run the
GPU and host tests share.  State and input are regenerated from the fixture's seed by the generator's own functions."""
import torch

from oracle import make_golden_head_dims as MG
from tests.conftest import check_grads, load_golden, rel_err

NAMES = MG.case_names()


class HeadDimGolden:
    def __init__(self, name):
        z = load_golden(name)
        self.name = name
        self.model, self.attention_type, self.kw, self.attn_step, self.seed = MG.case_config(name)
        assert int(z['seed']) == self.seed
        self.B, self.train_seed = int(z['B']), int(z['train_seed'])
        self.out = {k[5:]: torch.from_numpy(z[k]) for k in z.files if k.startswith('out::')}
        self.grad = {k[6:]: torch.from_numpy(z[k]) for k in z.files if k.startswith('grad::')}
        self.gradsum = {k[9:]: z[k] for k in z.files if k.startswith('gradsum::')}
        self.attn_shape = tuple(int(v) for v in z['attn_shape'])
        self.x = MG.random_input(self.kw, self.B, self.seed)

    def build(self):
        import videotransformer_pytorch_b200 as vt
        m = getattr(vt, self.model)(**self.kw)
        m.load_state_dict(MG.random_state({k: tuple(v.shape) for k, v in m.state_dict().items()}, self.seed), strict=True)
        return m


def run(g, dev, grad_tol):
    """eval output, last-layer attention rows, train output, input gradient of frame 0 and the parameter gradients of the
    model on `dev` -> dict of relative L2 errors against the fixture (grads: the worst verbatim one; every gradient, checksums
    included, is asserted within grad_tol)"""
    m = g.build().to(dev).eval()
    x = g.x.to(dev)
    with torch.no_grad():
        y = m(x)
        attn = m.get_last_selfattention(x)
    assert tuple(attn.shape) == g.attn_shape, (tuple(attn.shape), g.attn_shape)
    err = {'y_eval': rel_err(y.cpu(), g.out['y_eval']),
           'last_attn': rel_err(attn[..., ::g.attn_step, :].cpu(), g.out['last_attn_rows'])}
    m.train()
    xg = x.clone().requires_grad_(True)
    torch.manual_seed(g.train_seed)
    yt = m(xg)
    err['y_train'] = rel_err(yt.detach().cpu(), g.out['y_train'])
    w = torch.linspace(-1, 1, yt.numel(), dtype=torch.float64).reshape(yt.shape).to(dev)
    (yt.double() * w).sum().backward()
    err['dx'] = rel_err(xg.grad[:, 0].cpu(), g.out['dx0'])
    grads = {n: p.grad for n, p in m.named_parameters()}
    assert all(v is not None for v in grads.values())
    err['grads'] = check_grads(grads, g, grad_tol)
    return err
