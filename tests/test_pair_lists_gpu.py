"""The pair lists of KING kinship (vpca_kinship_pairs) and LD pruning (vpca_ld_prune_bed[_masked]) past their device pair
scratch, and LD pruning at its widest windows over several sample pieces, bit for bit against exact references.

Both lists are emitted in rounds of whole 32-row tiles, each round no larger than a fixed device scratch: the host turns
the per-row totals of a count pass into output positions, then copies each round's pairs to their place.  The tests
mirror that round rule and the LD chunk geometry in a few lines of Python, only to choose shapes and max_pairs values that
land on round, chunk and piece edges, and each test asserts that its shapes really reach several rounds, chunks or
pieces, so that a change of scratch size or geometry fails here instead of moving the test off its edge.  The oracle is
always the reference list: the sums of every pair are FP64 products on the device (sums of small integers below 2^53,
exact in any order), with the semantics of kinship_ref.py and ld_ref.py."""
import ctypes

import numpy as np
import pytest
import torch

import ld_ref
from kinship_ref import king_pairs, kinship_value, pair_counts
from spark_examples_b200 import native

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
KIN_SCRATCH_MIN = 1 << 21       # kinship pair scratch: max(2^21, 32 N) pairs (kinship.cu, kin_pair_alloc)
LD_SCRATCH_MIN = 1 << 20        # LD pair scratch: max(2^20, 1024 T) pairs (vpca.cu, ld_buffers)


@pytest.fixture(autouse=True)
def _free_torch_cache():
    yield
    torch.cuda.empty_cache()     # the device is shared with the library's own buffers and other tests


def _bits(a):
    return np.ascontiguousarray(a, np.float64).view(np.int64)


# ---- data: seeded genotypes made on the device, packed into .bed rows ------------------------------------------------

def _codes(seed, v, n, block=6, copy=0.85, missing=0.02):
    """(v, n) uint8 .bed codes on the device: blocks of `block` variants copy their founder on a `copy` share of the
    samples (LD), A1 frequencies in [0.05, 0.5], about `missing` missing calls."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    to_code = torch.tensor([3, 2, 0], dtype=torch.uint8, device=DEV)      # A1 count 0 / 1 / 2 -> 11 / 10 / 00
    out = torch.empty((v, n), dtype=torch.uint8, device=DEV)
    step = max(block, (1 << 26) // max(n, 1) // block * block)
    for v0 in range(0, v, step):
        m = min(step, v - v0)
        nb = -(-m // block)
        dose = lambda p, rows: ((torch.rand((rows, n), generator=g, device=DEV) < p).to(torch.uint8) +
                                (torch.rand((rows, n), generator=g, device=DEV) < p).to(torch.uint8))
        founder = dose(0.05 + 0.45 * torch.rand((nb, 1), generator=g, device=DEV), nb)
        own = dose(0.05 + 0.45 * torch.rand((m, 1), generator=g, device=DEV), m)
        fj = founder.repeat_interleave(block, dim=0)[:m]
        d = torch.where(torch.rand((m, n), generator=g, device=DEV) < copy, fj, own)
        c = to_code[d.long()]
        c[torch.rand((m, n), generator=g, device=DEV) < missing] = 1
        out[v0:v0 + m] = c
    return out


def _pack(codes):
    """(v, n) codes -> (v, ceil(n / 4)) .bed rows on the device, padding samples 00 like PLINK."""
    v, n = codes.shape
    c = torch.nn.functional.pad(codes, (0, (-n) % 4)).view(v, -1, 4)
    return c[:, :, 0] | (c[:, :, 1] << 2) | (c[:, :, 2] << 4) | (c[:, :, 3] << 6)


def _unpack(rows, n):
    """(v, stride) .bed rows -> (v, n) codes (low bits first), as the library reads them."""
    return torch.stack([(rows >> s) & 3 for s in (0, 2, 4, 6)], dim=-1).reshape(rows.shape[0], -1)[:, :n]


# ---- references on the device ---------------------------------------------------------------------------------------

def _king_ref(rows, n):
    """Every pair at -inf, as kinship_ref.king_pairs: ids (P, 2) int32 by b then a, counts (P, 5) int32, kinship (P,)."""
    c = _unpack(rows, n).T
    het, p1, p2 = (c == 2).double(), (c == 0).double(), (c == 3).double()
    called = het + p1 + p2
    mm = lambda x, y: torch.round(x @ y.T).long()
    nsnp, hethet, ibs0, h1 = mm(called, called), mm(het, het), mm(p1, p2) + mm(p2, p1), mm(het, p1 + p2)
    b, a = torch.tril_indices(n, n, -1, device=DEV)                     # row-major lower triangle: by b, then a
    counts = torch.stack([nsnp[a, b], hethet[a, b], ibs0[a, b], h1[a, b], h1[b, a]], dim=1).int().cpu().numpy()
    ids = torch.stack([a, b], dim=1).int().cpu().numpy()
    kin = kinship_value(counts[:, 1], counts[:, 2], counts[:, 3], counts[:, 4])
    return ids, counts, kin


def _select(full, thr):
    ids, counts, kin = full
    keep = kin >= thr                                                    # NaN never passes
    return ids[keep], counts[keep], kin[keep]


def _ld_ref(rows, n, window_lo, r2_max, eligible=None, block=512):
    """Every in-LD pair (i, j), window_lo[j] <= i < j, both eligible, in order of j then i, as ld_ref.ld_pairs ->
    (pairs (P, 2) int64, r2 (P,)); r2 with ld_ref.r2_of's three rounded double operations."""
    v = rows.shape[0]
    lut = torch.tensor([2.0, 0.0, 1.0, 0.0], dtype=torch.float64, device=DEV)
    lo_t = torch.from_numpy(np.asarray(window_lo, np.int64)).to(DEV)
    el = None if eligible is None else torch.from_numpy(np.asarray(eligible, bool)).to(DEV)
    mm = lambda x, y: torch.round(x @ y.T).long()
    out_p, out_r = [], []
    for j0 in range(0, v, block):
        j1 = min(v, j0 + block)
        i0 = int(window_lo[j0])                                          # window_lo is non-decreasing
        c = _unpack(rows[i0:j1], n)
        D, M = lut[c.long()], (c != 1).double()
        Dj, Mj = D[j0 - i0:], M[j0 - i0:]
        cnt, sx, sy, sxy = mm(M, Mj), mm(D, Mj), mm(M, Dj), mm(D, Dj)
        sxx, syy = mm(D * D, Mj), mm(M, Dj * Dj)
        del D, M, c
        cov, vx, vy = cnt * sxy - sx * sy, cnt * sxx - sx * sx, cnt * syy - sy * sy
        ok = (vx > 0) & (vy > 0)
        cf = cov.double()
        r2 = torch.where(ok, (cf * cf) / (vx.double() * vy.double()), torch.zeros((), dtype=torch.float64, device=DEV))
        ii = torch.arange(i0, j1, device=DEV)[:, None]
        jj = torch.arange(j0, j1, device=DEV)[None, :]
        sel = ok & (r2 > r2_max) & (ii < jj) & (ii >= lo_t[j0:j1][None, :])
        if el is not None:
            sel &= el[i0:j1][:, None] & el[j0:j1][None, :]
        js, is_ = torch.nonzero(sel.T, as_tuple=True)                    # by j, then i
        out_p.append(torch.stack([is_ + i0, js + j0], dim=1).cpu())
        out_r.append(r2.T[js, is_].cpu())
    return torch.cat(out_p).numpy().astype(np.int64), torch.cat(out_r).numpy()


def _sweep(v, pairs, eligible=None):
    """ld_ref.sweep over a list sorted by j: one step per variant instead of per pair."""
    ptr = np.searchsorted(pairs[:, 1], np.arange(v + 1))
    part = pairs[:, 0]
    keep = np.zeros(v, bool)
    for j in range(v):
        keep[j] = (eligible is None or eligible[j]) and not keep[part[ptr[j]:ptr[j + 1]]].any()
    return keep


def _ld_prune_ref(rows, n, window_lo, r2_max, eligible=None):
    pairs, r2 = _ld_ref(rows, n, window_lo, r2_max, eligible)
    return _sweep(rows.shape[0], pairs, eligible), pairs, r2


# ---- mirrors of the host's round rule and LD geometry (vpca.cu), used only to choose where to probe ----------------

def _kin_rounds(row_total, cap, limit):
    """vpca_kinship_pairs' rounds for a listing of `limit` pairs -> [(tile lo, tile hi, base, end)]."""
    n = len(row_total)
    start = np.concatenate([[0], np.cumsum(row_total, dtype=np.int64)])
    row_end = lambda bt: int(start[min(n, 32 * bt)])
    tiles, rounds, lo = -(-n // 32), [], 0
    while lo < tiles and row_end(lo) < limit:
        hi = lo + 1
        while hi < tiles and row_end(hi + 1) - row_end(lo) <= cap and row_end(hi) < limit:
            hi += 1
        rounds.append((lo, hi, row_end(lo), min(row_end(hi), limit)))
        lo = hi
    return rounds


def _ld_geometry(n, nv, H):
    """vpca_ld_prune_bed's chunk rows c, bit words T, plane panel width P and sample piece."""
    c = -(-max(2 * H, 1024) // 32) * 32
    if nv <= c:
        c = -(-nv // 32) * 32
    T = (H + 31) // 32 + 1
    R = 3 * c
    P = min(-(-n // 128) * 128, max(128, min(8192, (16 << 20) // R // 128 * 128)))
    piece = max(P, min(32768, (256 << 20) // R) // P * P)
    piece = min(piece, -(-n // P) * P)
    return c, T, P, piece


def _ld_chunks(nv, H, c):
    """-> [(s, nc, own_lo)]: chunks of c rows overlapping by H; a chunk decides rows [s + own_lo, s + nc)."""
    out, s = [], 0
    while True:
        e = min(s + c, nv)
        out.append((s, e - s, 0 if s == 0 else H))
        if e == nv:
            return out
        s = e - H


def _ld_rounds(row_total, n, H, max_pairs, cap=LD_SCRATCH_MIN):
    """vpca_ld_prune_bed's emit rounds -> [(chunk, tile lo, tile hi, base, end)] and each chunk's first position."""
    nv = len(row_total)
    c = _ld_geometry(n, nv, H)[0]
    rounds, firsts, listed = [], [], 0
    for k, (s, nc, lo) in enumerate(_ld_chunks(nv, H, c)):
        if listed >= max_pairs:
            break
        start = listed + np.concatenate([[0], np.cumsum(row_total[s + lo:s + nc], dtype=np.int64)])
        firsts.append(listed)
        limit = min(int(start[-1]), max_pairs)
        row_end = lambda bt: int(start[min(nc, max(lo, 32 * bt)) - lo])
        tiles, tlo = -(-nc // 32), lo // 32
        while tlo < tiles and row_end(tlo) < limit:
            thi = tlo + 1
            while thi < tiles and row_end(thi + 1) - row_end(tlo) <= cap and row_end(thi) < limit:
                thi += 1
            if min(row_end(thi), limit) > row_end(tlo):
                rounds.append((k, tlo, thi, row_end(tlo), min(row_end(thi), limit)))
            tlo = thi
        listed = int(start[-1])
    return rounds, firsts


# ---- calls through the ABI: the total each listing reports, and nothing written past the listed prefix --------------

def _kin_call(nat, thr, m):
    """vpca_kinship_pairs(thr, max_pairs = m) -> (ids, counts, kinship, *n_pairs); m = 0 counts with NULL outputs."""
    L, total = native.load_library(), ctypes.c_int64(-1)
    if m == 0:
        assert L.vpca_kinship_pairs(nat._h, float(thr), 0, None, None, None, ctypes.byref(total)) == native.VPCA_OK
        return None, None, None, total.value
    ids, counts, kin = np.full((m + 4, 2), -3, np.int32), np.full((m + 4, 5), -3, np.int32), np.full(m + 4, -2.0)
    assert L.vpca_kinship_pairs(nat._h, float(thr), m, ids.ctypes.data, counts.ctypes.data, kin.ctypes.data,
                                ctypes.byref(total)) == native.VPCA_OK
    got = min(m, total.value)
    assert (ids[got:] == -3).all() and (counts[got:] == -3).all() and (kin[got:] == -2.0).all()
    return ids[:got], counts[:got], kin[:got], total.value


def _ld_call(nat, rows, lo, r2_max, m, eligible=None):
    """vpca_ld_prune_bed[_masked](max_pairs = m) -> (keep, pairs, r2, *n_pairs); m = 0 counts with NULL outputs."""
    L, total = native.load_library(), ctypes.c_int64(-1)
    nv, stride = rows.shape
    lo = np.ascontiguousarray(lo, np.int64)
    keep = np.full(nv, 7, np.uint8)
    pairs, r2 = np.full((m + 4, 2), -3, np.int64), np.full(m + 4, -2.0)
    op, orr = (pairs.ctypes.data, r2.ctypes.data) if m else (None, None)
    if eligible is None:
        rc = L.vpca_ld_prune_bed(nat._h, rows.ctypes.data, nv, stride, lo.ctypes.data, float(r2_max), keep.ctypes.data,
                                 m, op, orr, ctypes.byref(total))
    else:
        el = np.ascontiguousarray(eligible, bool).view(np.uint8)
        rc = L.vpca_ld_prune_bed_masked(nat._h, rows.ctypes.data, nv, stride, lo.ctypes.data, el.ctypes.data,
                                        float(r2_max), keep.ctypes.data, m, op, orr, ctypes.byref(total))
    assert rc == native.VPCA_OK, nat._lib.vpca_last_error(nat._h)
    assert set(np.unique(keep).tolist()) <= {0, 1}
    got = min(m, total.value)
    assert (pairs[got:] == -3).all() and (r2[got:] == -2.0).all()
    return keep != 0, pairs[:got], r2[:got], total.value


def _ld_list(nat, rows, lo, r2_max, eligible=None):
    """The whole list: a count-only call, then a listing of exactly its total; both report the same total and keep."""
    keep0, _, _, total = _ld_call(nat, rows, lo, r2_max, 0, eligible)
    keep, pairs, r2, total1 = _ld_call(nat, rows, lo, r2_max, max(total, 1), eligible)
    assert total1 == total and len(pairs) == total
    np.testing.assert_array_equal(keep, keep0)
    return keep, pairs, r2


def _same_kin(got, want):
    np.testing.assert_array_equal(got[0], want[0])
    np.testing.assert_array_equal(got[1], want[1])
    np.testing.assert_array_equal(_bits(got[2]), _bits(want[2]))


def _same_ld(got, want):
    np.testing.assert_array_equal(got[0], want[0])
    np.testing.assert_array_equal(got[1], want[1])
    np.testing.assert_array_equal(_bits(got[2]), _bits(want[2]))


def _probes(edges, total, extra=()):
    """max_pairs values at every edge -1, 0, +1 and the given extras, within [1, total + 5]."""
    ms = {e + d for e in edges for d in (-1, 0, 1)} | set(extra) | {total - 1, total, total + 5}
    return sorted(m for m in ms if 1 <= m <= total + 5)


# ---- 1. kinship lists over several rounds ----------------------------------------------------------------------------

def test_kinship_all_pairs_and_truncation_over_four_rounds():
    """N = 4000 at -inf: about 8 M pairs in four rounds of the 2^21-pair scratch; then max_pairs at every round end -1 / 0
    / +1, inside a tile row, inside a round and at the total, in a mixed order on the same counts: each a prefix of the
    whole list, with *n_pairs the total every time."""
    n, nv = 4000, 1500
    rows = _pack(_codes(41, nv, n, block=1, copy=0.0))
    full = _king_ref(rows, n)
    total = len(full[0])
    assert total == n * (n - 1) // 2
    cap = max(KIN_SCRATCH_MIN, 32 * n)
    rounds = _kin_rounds(np.bincount(full[0][:, 1], minlength=n), cap, total)
    assert len(rounds) >= 4 and all(e - b <= cap for _, _, b, e in rounds)
    ends = [e for _, _, _, e in rounds[:-1]]
    b = 32 * 90 + 17
    inside_tile_row = b * (b - 1) // 2 + 5                                # the sixth pair of row b, inside tile row 90
    mid = (rounds[1][2] + rounds[1][3]) // 2
    ms = _probes(ends, total, [inside_tile_row, mid])
    order = np.random.default_rng(4000).permutation(len(ms))
    with native.NativePca(n) as nat:
        nat.kinshipBed(rows.cpu().numpy())
        assert _kin_call(nat, float("-inf"), 0)[3] == total
        ids, counts, kin, t = _kin_call(nat, float("-inf"), total)
        assert t == total
        _same_kin((ids, counts, kin), full)
        del ids, counts, kin
        for i in list(order) + list(order[:3]):
            m = ms[i]
            ids, counts, kin, t = _kin_call(nat, float("-inf"), m)
            assert t == total, m
            _same_kin((ids, counts, kin), tuple(x[:m] for x in full))


def _clustered(seed, n, nv, runs):
    """Random samples, then runs of tile rows [t0, t1) whose samples copy one base sample except on a share q of the
    variants: pairs inside the runs are related, every other pair is not."""
    codes = _codes(seed, nv, n, block=1, copy=0.0)
    g = torch.Generator(device=DEV).manual_seed(seed + 1)
    base = codes[:, 32 * runs[0][0]].clone()
    for t0, t1, q in runs:
        cols = slice(32 * t0, min(n, 32 * t1))
        width = codes[:, cols].shape[1]
        own = torch.rand((nv, width), generator=g, device=DEV) < q
        codes[:, cols] = torch.where(own, codes[:, cols], base[:, None])
    return _pack(codes)


def _gap_inside(per_tile):
    """an empty tile row followed by a non-empty one"""
    empty, full = np.flatnonzero(per_tile == 0), np.flatnonzero(per_tile)
    return empty.size > 0 and full.size > 0 and empty.min() < full.max()


def test_kinship_clustered_selection_jumps_empty_tile_rows():
    """Related samples in runs of tile rows separated by unrelated ones: at each threshold the selected pairs sit in
    dense runs of rows with empty tile rows between them, rounds span the empty rows, and the list is truncated at every
    round end and inside a run."""
    n, nv = 4000, 3000
    runs = [(3, 20, 0.0), (31, 52, 0.05), (60, 61, 0.0), (75, 100, 0.15), (108, 125, 0.02)]
    rows = _clustered(43, n, nv, runs)
    full = _king_ref(rows, n)
    tiles = -(-n // 32)
    in_run = np.zeros(tiles, bool)
    for t0, t1, _ in runs:
        in_run[t0:t1] = True
    cap = max(KIN_SCRATCH_MIN, 32 * n)
    with native.NativePca(n) as nat:
        nat.kinshipBed(rows.cpu().numpy())
        multi = 0
        for thr in (0.2, 0.4, 0.46):
            want = _select(full, thr)
            total = len(want[0])
            per_row = np.bincount(want[0][:, 1], minlength=n)
            per_tile = np.add.reduceat(per_row, np.arange(0, n, 32))
            full_tiles = np.flatnonzero(per_tile)
            assert (per_tile[~in_run] == 0).all() and (np.diff(full_tiles) > 1).sum() >= 2, thr
            rounds = _kin_rounds(per_row, cap, total)
            assert any(_gap_inside(per_tile[lo:hi]) for lo, hi, _, _ in rounds), thr
            multi += len(rounds) >= 2
            got = _kin_call(nat, thr, max(total, 1))
            assert got[3] == total
            _same_kin(got[:3], want)
            first_tile = int(np.flatnonzero(per_tile)[0])
            inside = int(np.cumsum(per_row)[32 * first_tile + 20]) - 3
            for m in _probes([e for _, _, _, e in rounds[:-1]], total, [inside]):
                got = _kin_call(nat, thr, m)
                assert got[3] == total, (thr, m)
                _same_kin(got[:3], tuple(x[:m] for x in want))
        assert multi >= 2


def test_kinship_at_the_sample_limit_lists_a_planted_block_over_two_rounds():
    """N = 21 845: 2100 identical samples give 2 203 950 pairs of kinship exactly 0.5, more than the 2^21-pair scratch;
    kinshipPairs(0.3) lists exactly their combinatorial id set in (b, a) order, with the counts of an identical pair."""
    n, nv, k = native.KINSHIP_MAX_SAMPLES, 2048, 2100
    rng = np.random.default_rng(21845)
    members = np.sort(rng.choice(n, size=k, replace=False))
    codes = _codes(45, nv, n, block=1, copy=0.0)
    mt = torch.from_numpy(members).to(DEV)
    codes[:, mt] = codes[:, mt[:1]]
    host_codes = codes.cpu().numpy()
    rows = _pack(codes).cpu().numpy()
    del codes, mt
    torch.cuda.empty_cache()
    bi, ai = np.tril_indices(k, -1)
    want_ids = np.stack([members[ai], members[bi]], axis=1).astype(np.int32)
    total = len(want_ids)
    cap = max(KIN_SCRATCH_MIN, 32 * n)
    assert total == k * (k - 1) // 2 > cap
    rounds = _kin_rounds(np.bincount(want_ids[:, 1], minlength=n), cap, total)
    assert len(rounds) >= 2
    c0 = host_codes[:, members[0]]
    same = (int((c0 != 1).sum()), int((c0 == 2).sum()), 0, 0, 0)
    with native.NativePca(n) as nat:
        nat.kinshipBed(rows)
        ids, counts, kin, t = _kin_call(nat, 0.3, total)
        assert t == total
        np.testing.assert_array_equal(ids, want_ids)
        assert (counts == np.asarray(same, np.int32)).all() and (kin == 0.5).all()
        for i in rng.choice(total, size=200, replace=False):
            a, b = int(ids[i, 0]), int(ids[i, 1])
            assert pair_counts(host_codes, a, b) == same, (a, b)
        for m in _probes([rounds[0][3]], total):
            got = _kin_call(nat, 0.3, m)
            assert got[3] == total
            np.testing.assert_array_equal(got[0], want_ids[:m])
        # a sample of the unrelated pairs, counted directly
        far = _kin_call(nat, float("-inf"), 5000)[:3]
        for i in rng.choice(5000, size=100, replace=False):
            a, b = int(far[0][i, 0]), int(far[0][i, 1])
            want = pair_counts(host_codes, a, b)
            assert tuple(far[1][i]) == want
            assert _bits(far[2][i]) == _bits(kinship_value(want[1], want[2], want[3], want[4]))


# ---- 2. LD lists over several rounds and chunks ----------------------------------------------------------------------

def _ld_case(seed, n, v, H, far=(), **kw):
    """Planted LD blocks, windows of H variants, and a copy of row i at row i + H for each i in `far`: pairs in LD
    across the whole window."""
    codes = _codes(seed, v, n, **kw)
    for i in far:
        codes[i + H] = codes[i]
    lo = np.maximum(0, np.arange(v, dtype=np.int64) - H)
    return _pack(codes), lo


@pytest.mark.parametrize("n", [1000, 1531])
def test_ld_dense_listing_over_rounds_and_chunks(n):
    """r2_max = 0 with H = 1500 over 7000 variants: five chunks, each owning 2-3.5 M pairs listed in three or four rounds
    of the 2^20-pair scratch."""
    H, v = 1500, 7000
    rows, lo = _ld_case(60 + n, n, v, H)
    want = _ld_prune_ref(rows, n, lo, 0.0)
    rounds, firsts = _ld_rounds(np.bincount(want[1][:, 1], minlength=v), n, H, len(want[1]))
    per_chunk = np.bincount([r[0] for r in rounds])
    assert len(firsts) >= 4 and (per_chunk >= 3).sum() >= 3 and per_chunk.max() >= 4
    assert 0 < want[0].sum() < v
    with native.NativePca(n) as nat:
        _same_ld(_ld_list(nat, rows.cpu().numpy(), lo, 0.0), want)


def test_ld_truncation_at_round_and_chunk_edges():
    """max_pairs at every round end -1 / 0 / +1, each chunk's first and last listed pair -1 / 0 / +1, inside a tile row,
    and at the total: the listed pairs are a prefix, the keep mask and the total do not change."""
    n, H, v = 1531, 1500, 6200
    rows, lo = _ld_case(71, n, v, H)
    keep, pairs, r2 = _ld_prune_ref(rows, n, lo, 0.0)
    total = len(pairs)
    rounds, firsts = _ld_rounds(np.bincount(pairs[:, 1], minlength=v), n, H, total)
    assert len(firsts) >= 4 and len(rounds) >= 2 * len(firsts)
    edges = [r[4] for r in rounds] + firsts + [f + 1 for f in firsts[1:]]
    inside = int(np.searchsorted(pairs[:, 1], 3100)) + 7                  # row 3100 (second chunk): inside a tile row
    ms = _probes(edges, total, [inside])
    host = rows.cpu().numpy()
    with native.NativePca(n) as nat:
        for m in ms:
            got = _ld_call(nat, host, lo, 0.0, m)
            assert got[3] == total, m
            np.testing.assert_array_equal(got[0], keep)
            np.testing.assert_array_equal(got[1], pairs[:m])
            np.testing.assert_array_equal(_bits(got[2]), _bits(r2[:m]))


def test_ld_masked_dense_listing_equals_the_eligible_rows_alone():
    """About 70 % of the variants eligible, r2_max = 0: keep and the pairs equal vpca_ld_prune_bed on the eligible rows
    alone with their windows recomputed, indices mapped back, at a density that crosses rounds."""
    n, H, v = 1203, 1500, 6000
    rows, lo = _ld_case(83, n, v, H)
    el = np.random.default_rng(83).random(v) < 0.7
    want = _ld_prune_ref(rows, n, lo, 0.0, el)
    rounds, firsts = _ld_rounds(np.bincount(want[1][:, 1], minlength=v), n, H, len(want[1]))
    assert len(firsts) >= 3 and np.bincount([r[0] for r in rounds]).max() >= 2
    idx = np.flatnonzero(el)
    lo_c = np.searchsorted(idx, lo[idx])                                 # first eligible variant at or after window_lo[j]
    host = rows.cpu().numpy()
    with native.NativePca(n) as nat:
        got = _ld_list(nat, host, lo, 0.0, el)
        _same_ld(got, want)
        ck, cp, cr = _ld_list(nat, np.ascontiguousarray(host[idx]), lo_c, 0.0)
    keep_c = np.zeros(v, bool)
    keep_c[idx] = ck
    _same_ld(got, (keep_c, idx[cp], cr))


# ---- 3. LD at the widest windows over several sample pieces ----------------------------------------------------------

@pytest.mark.parametrize("H, n, v, pieces, missing", [
    (4096, 10881, 9700, 2, 0.02),            # the last piece is one sample and one staged byte wide
    (4096, 2 * 10880 + 3001, 9000, 3, 0.05),
    (1500, 28672 + 37, 4000, 2, 0.02),
])
def test_ld_widest_windows_over_sample_pieces(H, n, v, pieces, missing):
    c, _, P, piece = _ld_geometry(n, v, H)
    assert -(-n // piece) == pieces and len(_ld_chunks(v, H, c)) >= 2
    if pieces == 2 and H == 4096:
        assert n - piece == 1 and -(-n // 4) - piece // 4 == 1
    rows, lo = _ld_case(90 + n, n, v, H, far=(0, 7, c - H - 3, c - H + 40, v - H - 1), missing=missing)
    want = _ld_prune_ref(rows, n, lo, 0.2)
    assert len(want[1]) > 1000 and 0 < want[0].sum() < v
    assert (want[1][:, 1] - want[1][:, 0] == H).sum() >= 5
    with native.NativePca(n) as nat:
        _same_ld(_ld_list(nat, rows.cpu().numpy(), lo, 0.2), want)


# ---- 4. one context across window geometries ------------------------------------------------------------------------

def test_one_context_across_window_geometries():
    """H = 1500 (dense) -> 40 -> 4096 -> 200 masked -> 1500 on one context, kinship calls between them: every result
    equals a fresh context and the reference, though later calls run on buffers sized by earlier, larger ones."""
    n, v = 517, 9000
    rows_d = _pack(_codes(97, v, n))
    rows = rows_d.cpu().numpy()
    ar = np.arange(v, dtype=np.int64)
    el = np.random.default_rng(97).random(v) < 0.8
    steps = [(4500, 1500, 0.0, None), (v, 40, 0.1, None), (v, 4096, 0.2, None), (v, 200, 0.1, el), (4500, 1500, 0.0, None)]
    assert len({_ld_geometry(n, nv, H)[0] for nv, H, _, _ in steps}) >= 3
    kin_want = king_pairs(_unpack(rows_d[:3000], n).cpu().numpy(), -np.inf)
    _same_kin(_king_ref(rows_d[:3000], n), kin_want)
    first = None
    with native.NativePca(n) as nat:
        nat.kinshipBed(rows[:3000])
        _same_kin(nat.kinshipPairs(), kin_want)
        for k, (nv, H, r2_max, elig) in enumerate(steps):
            lo = np.maximum(0, ar[:nv] - H)
            sub = rows[:nv]
            mask = None if elig is None else elig[:nv]
            got = _ld_list(nat, sub, lo, r2_max, mask)
            with native.NativePca(n) as fresh:
                _same_ld(got, _ld_list(fresh, sub, lo, r2_max, mask))
            _same_ld(got, _ld_prune_ref(rows_d[:nv], n, lo, r2_max, mask))
            if H == 40:
                _same_ld(got, ld_ref.prune(sub, n, lo, r2_max))                # the numpy restatement itself
            if k == 0:
                first = got
                assert len(_ld_rounds(np.bincount(got[1][:, 1], minlength=nv), n, H, len(got[1]))[0]) >= 4
            if k == len(steps) - 1:
                _same_ld(got, first)
            _same_kin(nat.kinshipPairs(), kin_want)
            _same_kin(nat.kinshipPairs(0.05), _select(kin_want, 0.05))
