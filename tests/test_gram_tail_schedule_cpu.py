"""Host-side checks of the Gram kernel's front/tail schedule (no GPU needed), through vpca_debug_schedule, which replays
the per-worker schedule the kernel's roles run (Sched in csrc/gram_sm90.cu) for a whole launch.

When the tiles T number more than half the workers W but fewer than W, front worker t < T owns tile t for k-blocks
[0, s) and the W - T tail workers split T tiles x [s, K) into contiguous tile-major shares, flushing every piece.
For every schedule (whole-tile waves, the within-window resident split, front/tail) this file checks that:
  * every (tile, k-block) unit of the launch is multiplied exactly once;
  * a worker holds one accumulator at a time: a piece that does not start from zero continues the tile of the open
    accumulator, and every accumulator is flushed before the next one starts and by the end of the launch;
  * the front/tail schedule is taken exactly when W / 2 < T < W -- never at T = W, where a resident worker holds a whole
    tile for the whole launch (N = 2696 with single CTAs on 132 SMs);
  * under it, at the initial split point s = K T / W, every worker's k-blocks plus flushes stay within
    2 ceil(T / (W - T)) + 3 of K T / W; the pieces stay exact for any s.
"""
import math

import numpy as np
import pytest

from spark_examples_b200 import native


@pytest.fixture(scope="module", autouse=True)
def _lib():
    import __graft_entry__ as entry
    if not native.library_path().exists():
        entry.build()
    native.load_library()


KBW = 64                                   # one 8192-variant int8 panel per window
WORKERS = ((66, 2), (57, 2), (132, 1), (114, 1))   # H100 SXM / PCIe: CTA pairs, single CTAs
TILINGS = (("rect", False), ("exact", True))


def _kb_totals():
    return (1, KBW - 1, KBW, KBW + 1, 3 * KBW + 5, 7813)


def _edge_ns(cg, exact, workers):
    """N where the tile count crosses W / 2 and W (last below, first at or above), N = 2504 and a stride over 2 .. 6000."""
    ns = set(range(2, 6001, 97)) | {2504}
    prev = None
    for n in range(2, 6001):
        t = len(native.debugTiles(n, cg, exact))
        if prev is not None:
            for edge in (workers // 2 + 1, workers):
                if prev < edge <= t:
                    ns |= {n - 1, n}
        prev = t
    return sorted(ns)


def _check(pieces, kind, s, n_tiles, workers, kb_total, bounded=True):
    assert kind in (0, 1, 2)
    cover = np.zeros((n_tiles, kb_total), np.int64)
    held = {}                              # worker -> tile of its open accumulator
    work = np.zeros(workers, np.int64)     # k-blocks + flushes per worker
    for w, t, k0, k1, first, flush in pieces:
        assert 0 <= w < workers and 0 <= t < n_tiles and 0 <= k0 <= k1 <= kb_total
        cover[t, k0:k1] += 1
        if first:
            assert w not in held, f"worker {w} starts tile {t} while tile {held[w]} is not flushed"
            held[w] = t
        else:
            assert held.get(w) == t, f"worker {w} continues tile {t} without holding it"
        work[w] += (k1 - k0) + (1 if flush else 0)
        if flush:
            del held[w]
    assert not held, f"accumulators never flushed: {held}"
    assert cover.min() == 1 and cover.max() == 1
    if kind == 2:
        T, W, K = n_tiles, workers, kb_total
        bound = K * T / W + 2 * math.ceil(T / (W - T)) + 3
        assert not bounded or work.max() <= bound, (work.max(), bound)
        front = pieces[pieces[:, 0] < T]
        assert np.all(front[:, 1] == front[:, 0]) and np.all(front[:, 3] <= s)
        tail = pieces[pieces[:, 0] >= T]
        assert np.all(tail[:, 2] >= s) and np.all(tail[:, 4] == 1) and np.all(tail[:, 5] == 1)
    return work


@pytest.mark.parametrize("workers,cg", WORKERS)
@pytest.mark.parametrize("tiling,exact", TILINGS)
def test_every_unit_once_one_accumulator_and_bounded_work(workers, cg, tiling, exact):
    for n in _edge_ns(cg, exact, workers):
        T = len(native.debugTiles(n, cg, exact))
        for K in _kb_totals():
            if K == 7813 and not (workers < 2 * T and T <= workers):
                continue                   # long launches only where the front/tail choice is made
            pieces, kind, s = native.debugSchedule(n, cg, exact, workers, KBW, K)
            assert (kind == 2) == (workers < 2 * T < 2 * workers), (n, T, kind)
            if kind == 2:
                assert s == int(K * (T / workers))
            else:
                assert s == K
            _check(pieces, kind, s, T, workers, K)


@pytest.mark.parametrize("workers,cg", WORKERS)
@pytest.mark.parametrize("tiling,exact", TILINGS)
def test_split_point_anywhere(workers, cg, tiling, exact):
    """s at 0 (no front), K (no tail), a window edge, just off it and inside a window, for a few K."""
    n = 2504
    T = len(native.debugTiles(n, cg, exact))
    if not workers < 2 * T < 2 * workers:
        n = next(m for m in range(2, 6001) if workers < 2 * len(native.debugTiles(m, cg, exact)) < 2 * workers)
        T = len(native.debugTiles(n, cg, exact))
    for K in (1, 5, KBW, 3 * KBW + 5, 7813):
        for s_want in sorted({0, K, min(K, KBW), max(0, min(K, KBW) - 1), K // 2, (K * 5) // 6}):
            frac = (s_want + 0.5) / K if s_want < K else 1.0
            pieces, kind, s = native.debugSchedule(n, cg, exact, workers, KBW, K, frac)
            assert kind == 2 and s == s_want
            _check(pieces, kind, s, T, workers, K, bounded=False)


def test_flagship_shape():
    """2504 samples on 66 CTA pairs: 55 tiles, the 11 tail pairs take 5 tiles each over [5K/6, K), in lockstep."""
    K = 7813
    pieces, kind, s = native.debugSchedule(2504, 2, False, 66, KBW, K)
    assert kind == 2 and s == int(K * 55 / 66)
    work = _check(pieces, kind, s, 55, 66, K)
    tail = pieces[pieces[:, 0] >= 55]
    for w in range(55, 66):
        mine = tail[tail[:, 0] == w]
        assert list(mine[:, 1]) == [5 * (w - 55) + i for i in range(5)]
        assert np.all(mine[:, 2] == s) and np.all(mine[:, 3] == K)
    # the critical path: 6510 k-blocks + 1 flush (front) against 5 x 1303 + 5 flushes (tail), not 7813
    assert work.max() <= s + 1 + 10 and work.max() < 0.84 * K


def test_no_front_tail_at_as_many_tiles_as_workers():
    """N = 2696 with single CTAs: T = W = 132, one whole tile per worker for the whole launch (the bf16 whole-launch
    accumulator test relies on it)."""
    assert len(native.debugTiles(2696, 1, False)) == 132
    for K in (1, KBW, 7813):
        pieces, kind, s = native.debugSchedule(2696, 1, False, 132, KBW, K)
        assert kind == 1 and s == K
        for w in range(132):
            mine = pieces[pieces[:, 0] == w]
            assert len(set(mine[:, 1])) == 1 and mine[0, 4] == 1 and mine[-1, 5] == 1 and mine[:-1, 5].sum() == 0
        _check(pieces, kind, s, 132, 132, K)


def test_bad_arguments():
    with pytest.raises(native.VpcaError):
        native.debugSchedule(1, 2, False, 66, KBW, 10)
    with pytest.raises(native.VpcaError):
        native.debugSchedule(2504, 2, False, 0, KBW, 10)
    with pytest.raises(native.VpcaError):
        native.debugSchedule(2504, 2, False, 66, 0, 10)
    with pytest.raises(native.VpcaError):
        native.debugSchedule(2504, 2, False, 66, KBW, 0)
    with pytest.raises(native.VpcaError):
        native.debugSchedule(2504, 2, False, 66, KBW, 10, 1.5)
