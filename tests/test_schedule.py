"""Host-side checks of the Gram kernel's work decomposition (no GPU needed): the tile list and the per-worker pieces
are computed by the same code the kernel's two roles replay (plan_segments in csrc/gram_sm90.cu), exposed through
vpca_debug_tiles / vpca_debug_plan.

What must hold for S = sum_v x_v x_v^T (VariantsPca.scala:186-188) to come out exact:
  * exact block cover: every 128 x 128 block (col block c <= row block r) of the lower triangle is produced by exactly
    one (A block, B block) product -- directly, or as the mirror image (c > r, written transposed);
  * the pieces of all workers partition every (tile, k-block) unit of a window: nothing twice, nothing missing;
  * the accumulators of one worker fit its budget -- one tile of up to 256 B rows, held in the registers of its two
    consumer warpgroups -- whenever the schedule is declared resident.
"""
import numpy as np
import pytest

from spark_examples_b200 import native


@pytest.fixture(scope="module", autouse=True)
def _lib():
    import __graft_entry__ as entry
    if not native.library_path().exists():
        entry.build()
    native.load_library()


def _cover(tiles, n, cg):
    nb = (n + 127) // 128
    cover = np.zeros((nb, nb), int)            # [row block][col block]
    mma_rows = 0
    for a0, a1, rb, ne, ws, fl, _, _ in tiles:
        assert a0 % 128 == 0 and a1 % 128 == 0 and rb % 128 == 0 and ne % 16 == 0 and 0 < ne <= 256
        assert rb + ne <= ((n + 15) // 16) * 16
        b_blocks = [rb // 128] + ([rb // 128 + 1] if ne > 128 else [])
        a_blocks = [a0 // 128] + ([a1 // 128] if cg == 2 and not (fl & 2) else [])
        mma_rows += cg * ne
        for ca in a_blocks:
            for r in b_blocks:
                if r >= ca:
                    cover[r, ca] += 1
                else:
                    assert fl & 1, "a block above the diagonal needs the transposed-write flag"
                    cover[ca, r] += 1
    return cover, mma_rows


@pytest.mark.parametrize("cg", [1, 2])
@pytest.mark.parametrize("n", [2, 70, 128, 129, 257, 385, 513, 600, 641, 769, 1092, 2504, 2560, 5000, 10000])
def test_exact_block_cover(n, cg):
    tiles = native.debugTiles(n, cg, True)
    nb = (n + 127) // 128
    cover, mma_rows = _cover(tiles, n, cg)
    assert np.array_equal(cover, np.tril(np.ones((nb, nb), int)))
    assert np.array_equal(tiles[:, 4], np.concatenate([[0], np.cumsum(tiles[:-1, 3] // 16)]))     # weight prefix
    # no filler unless the number of blocks of a row is odd and there is no partner row to trade a block with
    fillers = int(((tiles[:, 5] & 2) != 0).sum())
    assert fillers <= (1 if cg == 2 else 0) * ((nb + 3) // 4 + 1)


def test_exact_cover_saves_the_redundant_quarter_of_diagonal_tiles():
    """2560 samples = 20 blocks: 210 needed blocks; the square 256 x 256 tiling issues 55 tiles x 4 = 220."""
    tiles = native.debugTiles(2560, 2, True)
    _, mma_rows = _cover(tiles, 2560, 2)
    assert mma_rows == 210 * 128
    assert len(tiles) == 60 and int((tiles[:, 3] == 256).sum()) == 45


@pytest.mark.parametrize("cg,workers", [(2, 74), (1, 148), (2, 66), (1, 132)])   # H100: 66 CTA pairs / 132 CTAs
@pytest.mark.parametrize("n,kbw", [(2504, 64), (2504, 32), (2504, 7), (1092, 64), (600, 16), (130, 64), (2000, 128)])
def test_pieces_partition_every_window_and_fit_tmem(n, kbw, cg, workers):
    tiles = native.debugTiles(n, cg, True)
    pieces = native.debugPlan(tiles, workers, kbw)
    seen = np.zeros((len(tiles), kbw), int)
    for w, t, lo, hi, col, cols in pieces:
        assert 0 <= lo < hi <= kbw
        seen[t, lo:hi] += 1
        assert col % 32 == 0 and col + tiles[t, 3] <= cols <= 256
    assert (seen == 1).all()
    # accumulators of one worker never overlap
    for w in np.unique(pieces[:, 0]):
        mine = pieces[pieces[:, 0] == w]
        spans = sorted((c, c + ((tiles[t, 3] + 31) // 32) * 32) for _, t, _, _, c, _ in mine)
        assert all(spans[i][1] <= spans[i + 1][0] for i in range(len(spans) - 1))
    # one accumulator per worker: a worker owns a piece of one tile per window
    assert np.bincount(pieces[:, 0], minlength=workers).max() == 1
    # balance: no worker is given more than the mean share plus what the repair moves to it from a cut tile, and never
    # more than one whole tile
    work = np.zeros(workers)
    for w, t, lo, hi, _, _ in pieces:
        work[w] += (hi - lo) * (tiles[t, 3] // 16)
    mean = work.sum() / workers
    assert work.max() <= (tiles[:, 3] // 16).max() * kbw
    assert work.max() <= 2 * mean + 16


def test_large_cohorts_leave_the_resident_schedule():
    """N = 5000: more accumulators per worker than its budget holds -> the host must pick the wave schedule (debugPlan reports
    the overflow instead of a plan)."""
    tiles = native.debugTiles(5000, 2, True)
    with pytest.raises(native.VpcaError):
        native.debugPlan(tiles, 66, 64)
    # whole-tile waves deal out only full-weight two-row tiles, in compact patches of S
    full = tiles[tiles[:, 3] == 256]
    lead = 0
    while lead < len(tiles) and tiles[lead, 3] == 256:
        lead += 1
    assert lead == len(full)
    wave = tiles[:66]
    rows_of_x = set(wave[:, 0] // 128) | set(wave[:, 1] // 128) | set(wave[:, 2] // 128) | set(wave[:, 2] // 128 + 1)
    assert len(rows_of_x) <= 40              # ~34 row blocks of X per wave instead of ~150 for a row-major tile order


def test_rectangles_cover_the_triangle():
    """The default tiling, 256 x (<= 256) rectangles: every cell with row >= col lies in exactly one of them, and the B
    strips have nearly equal widths (so that tiles have nearly equal weights)."""
    n = 2504
    tiles = native.debugTiles(n, 2, False)
    hit = np.zeros((n, n), np.int8)
    for a0, a1, rb, ne, ws, fl, _, _ in tiles:
        assert fl & ~4 == 0 and a1 == a0 + 128 and rb % 16 == 0 and ne % 16 == 0 and ne <= 256
        hit[rb:min(n, rb + ne), a0:min(n, a0 + 256)] += 1
    assert (np.tril(hit) == np.tril(np.ones((n, n), np.int8))).all()
    assert set(tiles[:, 3]) == {240, 256}


# col_limit is the budget handed to the repair (256: the kernel's one 256-row register accumulator; the larger budgets
# check the same repair when a worker may hold two accumulators)
@pytest.mark.parametrize("n,exact,col_limit", [(2504, True, 512), (2504, False, 480), (1092, True, 512), (2000, True, 512),
                                               (2504, False, 256), (1500, False, 256), (1092, True, 256)])
@pytest.mark.parametrize("seed", [0, 1, 2, 3])
def test_rebalanced_splits_are_repaired_to_fit_tmem(n, exact, col_limit, seed):
    """The speed-weighted split the device publishes (rebalance_kernel -> repair_split) must keep every worker inside its
    accumulator budget whatever speeds were measured: skew the shares by up to +-35 % (the clamp of the rebalancer) and check that
    the repaired split still partitions every (tile, k-block) unit and fits `col_limit` columns."""
    workers, kbw = 74, 104
    tiles = native.debugTiles(n, 2, exact)
    rng = np.random.default_rng(seed)
    share = rng.uniform(0.65, 1.35, workers)
    cum = np.concatenate([[0.0], np.cumsum(share / share.sum())])
    cum[-1] = 1.0
    try:
        native.debugPlan(tiles, workers, kbw)
    except native.VpcaError:
        pytest.skip("equal split is not resident for this shape")
    cum2, pieces = native.debugRebalance(tiles, workers, kbw, cum, col_limit)
    assert cum2[0] == 0.0 and cum2[-1] == 1.0 and (np.diff(cum2) >= 0).all()
    seen = np.zeros((len(tiles), kbw), int)
    for w, t, lo, hi, col, cols in pieces:
        seen[t, lo:hi] += 1
        assert col + tiles[t, 6] <= cols <= col_limit
    assert (seen == 1).all()
    assert np.bincount(pieces[:, 0], minlength=workers).max() <= 4
    # the repair only trims: no worker gets more than the candidate gave it plus what its predecessors gave up
    want = np.diff(cum)
    got = np.diff(cum2)
    assert got.max() <= want.max() + (want - got).clip(0).sum() + 1e-9


@pytest.mark.parametrize("n,world", [(2504, 8), (1092, 4), (100_000, 8), (777, 2), (10_000, 3)])
def test_owner_computes_bands_tile_the_triangle_exactly_once(n, world):
    """Biobank form without a reduction (SURVEY 8e): context q stores rows [lo_q, hi_q) of S and enumerates only the
    products of those rows.  Over all bands every cell with row >= col must be produced exactly once, no tile may reach
    past its band (the band is all the memory the context has), and the bands carry equal shares of the MMA work."""
    bands = native.ownerRowBands(n, world)
    work = []
    blocks = {}                                          # (row block of 16, col block of 128) -> times produced
    for row0, rows in bands:
        t = native.debugBandTiles(n, 2, row0, rows)
        assert (t[:, 2] >= row0).all() and (t[:, 2] % 16 == 0).all() and (t[:, 3] % 16 == 0).all()
        assert (np.minimum(t[:, 2] + t[:, 3], n) <= row0 + rows).all()          # never beyond the band (ragged last band: n)
        work.append(int((256 * t[:, 3]).sum()))
        for a0, a1, rb, ne, *_ in t:
            assert a1 == a0 + 128
            for r16 in range(rb // 16, (min(rb + ne, n) + 15) // 16):
                for cb in (a0 // 128, a1 // 128):
                    if cb * 128 <= min(r16 * 16 + 15, n - 1) and cb * 128 < n:      # the block touches row >= col
                        blocks[(r16, cb)] = blocks.get((r16, cb), 0) + 1
    assert set(blocks.values()) == {1}
    need = sum(1 for r16 in range((n + 15) // 16) for cb in range((n + 127) // 128) if cb * 128 <= min(r16 * 16 + 15, n - 1))
    assert len(blocks) == need
    assert max(work) <= 1.25 * (sum(work) / world) + 256 * 256 * 4     # equal shares of the triangle, up to tile granularity


def test_repair_is_safe_for_any_split_hypothesis():
    """Property test of repair_split (the last line of defence before a launch: overlapping accumulators would corrupt
    S silently): for ANY monotone split of a window -- far outside the +-35 % the rebalancer proposes, including empty and
    huge shares -- the repaired split either fits every worker into its accumulator budget and still partitions the window, or is
    rejected."""
    from hypothesis import given, settings, strategies as st

    tiles_by = {(n, ex): native.debugTiles(n, 2, ex) for n, ex in [(2504, True), (2504, False), (1092, True), (1500, False)]}

    @settings(max_examples=120, deadline=None)
    @given(st.sampled_from(sorted(tiles_by)), st.integers(8, 74), st.integers(4, 128),
           st.lists(st.floats(0.0, 4.0, allow_nan=False), min_size=74, max_size=74))
    def check(which, workers, kbw, raw):
        tiles = tiles_by[which]
        col_limit = 256
        share = np.asarray(raw[:workers]) + 1e-9
        cum = np.concatenate([[0.0], np.cumsum(share / share.sum())])
        cum[-1] = 1.0
        try:
            cum2, pieces = native.debugRebalance(tiles, workers, kbw, cum, col_limit)
        except native.VpcaError:
            return                                            # rejected: the device keeps its previous split
        seen = np.zeros((len(tiles), kbw), int)
        for w, t, lo, hi, col, cols in pieces:
            assert 0 <= lo < hi <= kbw and col + tiles[t, 6] <= cols <= col_limit
            seen[t, lo:hi] += 1
        assert (seen == 1).all()
        assert len(pieces) == 0 or np.bincount(pieces[:, 0], minlength=workers).max() <= 4
        assert (np.diff(cum2) >= 0).all() and cum2[0] == 0.0 and cum2[-1] == 1.0

    check()
