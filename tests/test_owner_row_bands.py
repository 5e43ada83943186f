"""The row bands of the owner-rows reduction (vpca_owner_row_bands, host-only): they cover [0, N) in order, end on
multiples of 32, hold at least 32 rows each, and split the lower triangle into equal shares wherever the minimum-width
clamps leave the rounding alone.  Band-only contexts allocate exactly these bands."""
import math

import pytest


def _bands(n, world):
    from spark_examples_b200 import native
    return native.ownerRowBands(n, world)


def _sizes(world):
    ns = list(range(64 * world, 3001, 29))                     # every residue mod 32 over the range
    ns += [64 * world + d for d in (1, 2, 3, 31, 32, 33)]       # ragged N just past the minimum
    ns += [1092, 1093, 1094, 2504, 4099, 65_537, 100_000]
    return sorted({n for n in ns if n >= 64 * world})


@pytest.mark.parametrize("world", range(1, 17))
def test_bands_cover_the_rows_in_equal_triangle_shares(world):
    for n in _sizes(world):
        bands = _bands(n, world)
        assert len(bands) == world
        prev = 0
        for q, (row0, rows) in enumerate(bands):
            end = row0 + rows
            assert row0 == prev, (n, world, q)                 # in order, no gap, no overlap
            assert rows >= 32, (n, world, q)
            if q + 1 < world:
                assert end % 32 == 0, (n, world, q)
                ideal = n * math.sqrt((q + 1) / world)          # rows [0, R) hold R^2 / 2 cells of the triangle
                # the clamps: 32 rows for this band and for each after it, on multiples of 32
                lo, hi = prev + 32, (n // 32) * 32 - 32 * (world - 1 - q)
                if lo <= ideal - 16 and ideal + 16 <= hi:
                    assert abs(end - ideal) <= 16, (n, world, q, end, ideal)
                else:
                    assert lo <= end <= hi, (n, world, q, end)
            prev = end
        assert prev == n, (n, world)


@pytest.mark.parametrize("world", [1, 2, 5, 16])
def test_fewer_than_64_rows_per_rank_is_refused(world):
    from spark_examples_b200 import native
    with pytest.raises(native.VpcaError) as ei:
        _bands(64 * world - 1, world)
    assert ei.value.code == native.VPCA_ERR_BAD_ARG
    assert len(_bands(64 * world, world)) == world


@pytest.mark.parametrize("world", [0, 17])
def test_world_outside_1_to_16_is_refused(world):
    from spark_examples_b200 import native
    with pytest.raises(native.VpcaError):
        native.ownerRowBands(4096, world)
