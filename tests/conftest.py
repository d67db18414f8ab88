import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
GOLD = os.path.join(ROOT, 'tests', 'golden')


class GoldenArrays(dict):
    """Arrays of one fixture: `<name>.npz` plus its continuation files `<name>.1.npz`, `<name>.2.npz`, ... (fixtures are
    split so that no file exceeds 1 MB)."""

    @property
    def files(self):
        return list(self)


def load_golden(name):
    z, i, path = GoldenArrays(), 0, os.path.join(GOLD, name + '.npz')
    while os.path.exists(path):
        with np.load(path) as part:
            z.update({k: part[k] for k in part.files})
        i += 1
        path = os.path.join(GOLD, f'{name}.{i}.npz')
    if not z:
        raise FileNotFoundError(os.path.join(GOLD, name + '.npz'))
    return z


def pytest_configure(config):
    config.addinivalue_line('markers', 'gpu: needs a CUDA device (an H100: pytest -m gpu)')
    config.addinivalue_line('markers', 'experimental: kernel paths that ship disabled until confirmed on hardware '
                                       '(run with VT_EXPERIMENTAL=1; the test switches the path on itself)')


def pytest_collection_modifyitems(config, items):
    if not os.environ.get('VT_EXPERIMENTAL'):
        skip_exp = pytest.mark.skip(reason='experimental kernel path (set VT_EXPERIMENTAL=1)')
        for it in items:
            if 'experimental' in it.keywords:
                it.add_marker(skip_exp)
    if torch.cuda.is_available():
        return
    skip = pytest.mark.skip(reason='no CUDA device')
    for it in items:
        if 'gpu' in it.keywords:
            it.add_marker(skip)


class Golden:
    """One reference-generated fixture (oracle/make_golden.py)."""

    def __init__(self, name):
        z = load_golden(name)
        self.raw = z
        self.x = torch.from_numpy(z['x'])
        self.sd = {k[4:]: torch.from_numpy(z[k]) for k in z.files if k.startswith('sd::')}
        self.out = {k[5:]: torch.from_numpy(z[k]) for k in z.files if k.startswith('out::')}
        self.grad = {k[6:]: torch.from_numpy(z[k]) for k in z.files if k.startswith('grad::')}
        self.gradsum = {k[9:]: z[k] for k in z.files if k.startswith('gradsum::')}
        self.cfg = {k[4:]: int(z[k]) for k in z.files if k.startswith('cfg_')}
        self.train_seed = int(z['train_seed'])
        self.B = int(z['B'])


class MaskFeatGolden:
    """MaskFeat fixture: inputs + reference outputs; the (large) state is regenerated from its seed with
    ``oracle.mvit_oracle.random_maskfeat_state`` exactly as oracle/make_golden.py did."""

    def __init__(self, name):
        import ast
        from oracle import mvit_oracle as mo
        z = load_golden(name)
        self.kwargs = ast.literal_eval(str(z['cfg_kwargs'][0]))
        self.cfg = mo.maskfeat_config(**self.kwargs)
        self.seed, self.B = int(z['seed']), int(z['B'])
        self.x = torch.from_numpy(z['x'])
        self.mask = torch.from_numpy(z['mask'])
        self.target = torch.from_numpy(z['target'])
        self.cube_marker = ast.literal_eval(str(z['cube_marker'][0]))
        self.feats = torch.from_numpy(z['feats'])
        self.feats_nomask_cls = torch.from_numpy(z['feats_nomask_cls'])
        self.pred = torch.from_numpy(z['pred'])
        self.loss = float(z['loss'])
        self.grad = {k[6:]: torch.from_numpy(z[k]) for k in z.files if k.startswith('grad::')}
        self.gradsum = {k[9:]: z[k] for k in z.files if k.startswith('gradsum::')}

    def state(self, dtype=torch.float64):
        from oracle import mvit_oracle as mo
        return mo.random_maskfeat_state(self.cfg, seed=self.seed, dtype=dtype)


@pytest.fixture(scope='session')
def maskfeat_golden():
    cache = {}

    def get(name):
        if name not in cache:
            cache[name] = MaskFeatGolden(name)
        return cache[name]
    return get


@pytest.fixture(scope='session')
def golden():
    cache = {}

    def get(name):
        if name not in cache:
            cache[name] = Golden(name)
        return cache[name]
    return get


def rel_err(a, b):
    a, b = a.double(), b.double()
    return float((a - b).norm() / (b.norm() + 1e-30))


def check_grads(named_grads, g, tol):
    """named_grads: dict name -> tensor; compares against verbatim grads and checksum triples."""
    worst = 0.0
    for n, ref in g.grad.items():
        e = rel_err(named_grads[n].cpu(), ref)
        worst = max(worst, e)
        assert e < tol, (n, e)
    for n, ref in g.gradsum.items():
        t = named_grads[n].detach().cpu().double()
        lin = torch.linspace(-1, 1, t.numel(), dtype=torch.float64)
        mine = np.array([t.sum().item(), t.norm().item(), (t.reshape(-1) * lin).sum().item()])
        # l2 norm is the scale; sums are compared relative to it
        scale = ref[1] + 1e-30
        assert abs(mine[1] - ref[1]) / scale < tol, (n, mine, ref)
        assert abs(mine[0] - ref[0]) / (scale * np.sqrt(t.numel())) < tol, (n, mine, ref)
        assert abs(mine[2] - ref[2]) / (scale * np.sqrt(t.numel())) < tol, (n, mine, ref)
    return worst


@pytest.fixture
def emu():
    """Swap the kernel table for the CPU emulation (host-logic tests only)."""
    from tests.emu_kernels import EmuKernels
    from videotransformer_pytorch_b200 import _lib
    old = _lib.K
    _lib.K = EmuKernels(exact=True)
    yield _lib.K
    _lib.K = old
