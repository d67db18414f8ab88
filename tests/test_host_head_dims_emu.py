"""TimeSformer / ViViT at head widths 32, 96 and 128 on the CPU kernel table (tests/emu_kernels.py) against the fixtures
from the reference classes: the host side (head split, scale, row maps, the probability output) at every width."""
import pytest

from tests import head_dim_goldens as HG


@pytest.mark.parametrize('name', HG.NAMES)
def test_head_dim_golden_on_emulated_kernels(emu, name):
    err = HG.run(HG.HeadDimGolden(name), 'cpu', 2e-4)
    assert err['y_eval'] < 2e-5 and err['last_attn'] < 2e-5 and err['y_train'] < 2e-5, err
    assert err['dx'] < 1e-4, err
