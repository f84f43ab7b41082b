"""The PReLU backward's row groups (the summation order at B2G_LAYER_PRELU in include/b200gan.h): the group count of a pass is not monotone in
its row count, so the slope partials of a net are sized for min(max_batch, 64, 1024 / ceil(M / 2048)) groups.  That bound must hold for every
pass of 1 ... max_batch rows."""
import pytest

from gan_deeplearning4j_b200 import engine


def allocated_groups(max_rows, row_elems):
    return max(1, min(max_rows, 64, max(1, 1024 // -(-row_elems // 2048))))


def test_group_count_is_not_monotone():
    assert engine.prelu_groups(65, 32) == 33 and engine.prelu_groups(64, 32) == 64


@pytest.mark.parametrize("row_elems", [1, 32, 128, 2048, 2049, 40960, 65536, 1 << 20, 1 << 22])
def test_allocation_bounds_every_batch(row_elems):
    for max_rows in list(range(1, 200)) + [256, 1000, 1024]:
        cap = allocated_groups(max_rows, row_elems)
        assert max(engine.prelu_groups(r, row_elems) for r in range(1, max_rows + 1)) <= cap, (row_elems, max_rows)
