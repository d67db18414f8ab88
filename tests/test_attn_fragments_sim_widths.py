"""The ldmatrix / mma.sync fragment walk of tests/test_attn_fragments_sim.py at the packed-qkv head widths 32 and 128:
the [64][HD + 8] tile pitch (80 and 272 bytes) puts the 8 rows of every ldmatrix phase in distinct banks, and every
(row block, k chunk, n block) fragment the kernels load is the one the MMA layout asks for."""
import pytest

from tests import test_attn_fragments_sim as F


@pytest.mark.parametrize('HD', [32, 128])
def test_ldmatrix_a_fragments_at_head_width(HD):
    F.test_ldmatrix_a_fragments(HD)


@pytest.mark.parametrize('HD', [32, 128])
def test_ldmatrix_b_fragments_row_operand_at_head_width(HD):
    F.test_ldmatrix_b_fragments_row_operand(HD)


@pytest.mark.parametrize('HD', [32, 128])
def test_ldmatrix_b_fragments_trans_at_head_width(HD):
    F.test_ldmatrix_b_fragments_trans(HD)
