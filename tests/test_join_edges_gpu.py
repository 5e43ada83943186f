"""The device join / merge of several variant sets (csrc/join.cu, VariantsPca.scala:115-148) past a million rows and at its
edges, against a sort-based reference written here on integer key ids.

What these tests pin that tests/test_join_gpu.py does not reach:
  - the scan's carry loop (`scan_blocks_kernel` walks the block totals in steps of 1024 blocks, so its carry matters only
    past 2^20 rows): JOIN and MERGE at 1, 1023, 1024, 1025, 2^20, 2^20 + 1 and 3 * 2^20 + 517 rows, full CSR compared;
  - input whose key offsets and call offsets start above zero (the library shifts its base pointers instead of rebasing);
  - heavy fan-out (300 x 300 rows of one key, 1 x 4096, merge groups of 499 / 500 / 501) and the long probe clusters it
    makes; the call time of these cases is printed (the cluster walk is O(G^2) in a key's multiplicity G);
  - edge inputs: no left rows, no right rows, no rows, rows without calls, empty keys, keys that are prefixes of one
    another, byte-identical keys of different variants, variant_set_count = 1, groups from a single dataset;
  - one context reused for joins of different sizes, vpca_reset, and refused calls (which keep the previous result);
  - the Gram of a 3.15 M-row join over several chunks, and the driver from VCF files with 2 (join) and 4 (merge) sets.

The reference builds every key from an int64 id through a fixed layout whose inverse is checked on every case, so equal
ids mean equal key bytes and, through murmur3, equal device keys.  The output is compared as a full CSR: the device emits
one row per (left, right) pair or per kept group, empty rows included."""
import ctypes
import functools
import time

import numpy as np
import pytest

import spark_examples_b200 as pkg
from spark_examples_b200 import native, variants_pca, vcf
from spark_examples_b200.variants_pca import VariantsPcaDriver, variantKeyBytes

pytestmark = pytest.mark.gpu

JOIN, MERGE = native.JOIN, native.MERGE
N = 97                         # a prime: (base + k * step) % N lists distinct samples for k < N and step != 0
SCAN_ROWS = [1, 1023, 1024, 1025, 1 << 20, (1 << 20) + 1, 3 * (1 << 20) + 517]
BIG = 3 * (1 << 20) + 517


def _log(msg):
    print(f"[join-edges] {msg}")


# ---- reference 2: MurmurHash3_x64_128 (seed 0) of equal-length keys, column-wise in wrapping uint64 arithmetic ----------
_C1, _C2 = np.uint64(0x87C37B91114253D5), np.uint64(0x4CF5AD432745937F)


def _rotl(x, r):
    return (x << np.uint64(r)) | (x >> np.uint64(64 - r))


def _fmix(k):
    k = k ^ (k >> np.uint64(33))
    k = k * np.uint64(0xFF51AFD7ED558CCD)
    k = k ^ (k >> np.uint64(33))
    k = k * np.uint64(0xC4CEB9FE1A85EC53)
    return k ^ (k >> np.uint64(33))


def murmur3_fixed(keys: np.ndarray) -> np.ndarray:
    """(nkeys, L) uint8 -> (nkeys, 2) uint64 (h1, h2), what vpca_hash_keys returns for those keys."""
    n, L = keys.shape
    buf = np.zeros((n, (L + 15) // 16 * 16), np.uint8)
    buf[:, :L] = keys
    w = buf.view("<u8")                                          # zero-padded little-endian words, two per 16-byte block
    h1, h2 = np.zeros(n, np.uint64), np.zeros(n, np.uint64)
    with np.errstate(over="ignore"):
        for b in range(L // 16):
            h1 ^= _rotl(w[:, 2 * b] * _C1, 31) * _C2
            h1 = _rotl(h1, 27) + h2
            h1 = h1 * np.uint64(5) + np.uint64(0x52DCE729)
            h2 ^= _rotl(w[:, 2 * b + 1] * _C2, 33) * _C1
            h2 = _rotl(h2, 31) + h1
            h2 = h2 * np.uint64(5) + np.uint64(0x38495AB5)
        t, b = L & 15, L // 16
        if t > 8:
            h2 ^= _rotl(w[:, 2 * b + 1] * _C2, 33) * _C1
        if t > 0:
            h1 ^= _rotl(w[:, 2 * b] * _C1, 31) * _C2
        h1 ^= np.uint64(L)
        h2 ^= np.uint64(L)
        h1 = h1 + h2
        h2 = h2 + h1
        h1, h2 = _fmix(h1), _fmix(h2)
        h1 = h1 + h2
        h2 = h2 + h1
    return np.stack([h1, h2], axis=1)


# ---- keys from integer ids ------------------------------------------------------------------------------------------
KEY_LEN = 23
_BASES = np.frombuffer(b"ACGT", np.uint8)


def id_keys(ids) -> np.ndarray:
    """The key of variant id i, laid out like variantKeyBytes (one KEY_LEN-byte row per id): contig b"chrNN" with
    NN = i % 23, start = i // 23 and end = start + 1 + i % 5 as little-endian int64, one reference and one alternate
    base.  (contig, start) gives i back, so the layout is one-to-one: every call checks that id_of_key inverts it."""
    ids = np.asarray(ids, np.int64)
    k = np.empty((len(ids), KEY_LEN), np.uint8)
    c, start = ids % 23, ids // 23
    k[:, 0:3] = np.frombuffer(b"chr", np.uint8)
    k[:, 3] = 48 + c // 10
    k[:, 4] = 48 + c % 10
    k[:, 5:13] = start.astype("<i8").view(np.uint8).reshape(-1, 8)
    k[:, 13:21] = (start + 1 + ids % 5).astype("<i8").view(np.uint8).reshape(-1, 8)
    k[:, 21] = _BASES[ids % 4]
    k[:, 22] = _BASES[(ids // 4) % 4]
    assert np.array_equal(id_of_key(k), ids)
    return k


def id_of_key(k: np.ndarray) -> np.ndarray:
    start = np.ascontiguousarray(k[:, 5:13]).view("<i8").ravel()
    return start * 23 + (k[:, 3].astype(np.int64) - 48) * 10 + (k[:, 4].astype(np.int64) - 48)


def ids_of_bytes(keys) -> np.ndarray:
    """Ids of arbitrary key bytes: equal bytes, equal id."""
    seen = {}
    return np.asarray([seen.setdefault(bytes(k), len(seen)) for k in keys], np.int64)


def random_calls(rng, nrows, max_len=6):
    """CSR of `nrows` rows of 0..max_len distinct samples each (about 1 in 7 rows empty)."""
    lens = rng.integers(0, max_len + 1, nrows).astype(np.int64)
    off = np.zeros(nrows + 1, np.int64)
    np.cumsum(lens, out=off[1:])
    k = np.arange(off[-1], dtype=np.int64) - np.repeat(off[:-1], lens)
    base = np.repeat(rng.integers(0, N, nrows), lens)
    step = np.repeat(rng.integers(1, N, nrows), lens)
    return off, ((base + k * step) % N).astype(np.int32)


# ---- reference 1: sort-based join / merge on ids ----------------------------------------------------------------------
def _segments(starts, lens):
    """Concatenation of arange(starts[j], starts[j] + lens[j]) over j."""
    starts, lens = np.asarray(starts, np.int64), np.asarray(lens, np.int64)
    ends = np.cumsum(lens)
    return np.repeat(starts - (ends - lens), lens) + np.arange(ends[-1] if len(ends) else 0, dtype=np.int64)


def _concat_rows(off, idx, members):
    """Output row r = the calls of input rows members[r, 0], members[r, 1], ... in that order."""
    lens = np.diff(off)
    flat = members.ravel()
    out_off = np.zeros(len(members) + 1, np.int64)
    np.cumsum(lens[members].sum(axis=1), out=out_off[1:])
    return out_off, idx[_segments(off[flat], lens[flat])]


def ref_join(ids, off, idx, n_left):
    """VariantsPca.scala:115-128: for each left row in row order, the right rows with its id in row order, each giving
    calls(left) ++ calls(right).  Returns (offsets, idx, first input row of each output row)."""
    left, right = ids[:n_left], ids[n_left:]
    order = np.argsort(right, kind="stable")
    sr = right[order]
    lo, hi = np.searchsorted(sr, left, "left"), np.searchsorted(sr, left, "right")
    cnt = hi - lo
    L = np.repeat(np.arange(n_left, dtype=np.int64), cnt)
    R = n_left + order[_segments(lo, cnt)]
    return (*_concat_rows(off, idx, np.stack([L, R], axis=1)), L)


def ref_merge(ids, off, idx, vsc):
    """VariantsPca.scala:136-148: groups of equal ids with exactly `vsc` rows, ordered by first row, members in row order."""
    _, first, counts = np.unique(ids, return_index=True, return_counts=True)
    order = np.argsort(ids, kind="stable")
    group_start = np.cumsum(counts) - counts
    keep = np.flatnonzero(counts == vsc)
    keep = keep[np.argsort(first[keep])]
    members = order[_segments(group_start[keep], counts[keep])].reshape(-1, vsc)
    return (*_concat_rows(off, idx, members), first[keep])


def reference(mode, ids, off, idx, n_left, vsc):
    return ref_join(ids, off, idx, n_left) if mode == JOIN else ref_merge(ids, off, idx, vsc)


def drop_empty(off, idx):
    return [idx[off[i]:off[i + 1]].tolist() for i in range(len(off) - 1) if off[i + 1] > off[i]]


def oracle_rows(oracle, mode, keys, off, idx, n_left, vsc):
    """The oracle's own restatement on (murmur3 hex, calls) records, empty rows dropped (:166)."""
    recs = [(oracle.np_murmur3_128(bytes(k)).hex(), idx[off[i]:off[i + 1]].tolist()) for i, k in enumerate(keys)]
    rows = (oracle.np_join_datasets(recs[:n_left], recs[n_left:]) if mode == JOIN
            else oracle.np_merge_datasets([recs], vsc))
    return [r for r in rows if r]


# ---- the raw ABI ------------------------------------------------------------------------------------------------------
def _ptr(a):
    """Host address of `a` for a C call: the caller keeps `a` bound to a name until that call returns, since the address
    alone does not keep a temporary array alive."""
    return None if a is None else a.ctypes.data


def raw_join(nat, mode, vsc, n_left, payload, koff, off, idx, nrows=None):
    """vpca_join_rows on numpy buffers -> (status, rows, calls)."""
    rows, nnz = ctypes.c_int64(-1), ctypes.c_int64(-1)
    nrows = len(koff) - 1 if nrows is None else nrows
    rc = nat._lib.vpca_join_rows(nat._h, int(mode), int(vsc), int(n_left), _ptr(payload), _ptr(koff), _ptr(off), _ptr(idx),
                                 int(nrows), ctypes.byref(rows), ctypes.byref(nnz))
    return rc, rows.value, nnz.value


def device_join(nat, mode, vsc, n_left, payload, koff, off, idx):
    """Join on the device and fetch the result: (offsets, idx, seconds of the vpca_join_rows call)."""
    t0 = time.perf_counter()
    rc, rows, nnz = raw_join(nat, mode, vsc, n_left, payload, koff, off, idx)
    dt = time.perf_counter() - t0
    assert rc == native.VPCA_OK, nat._lib.vpca_last_error(nat._h)
    assert nat.joinSize() == (rows, nnz)
    got_off, got_idx = nat.joinFetch(rows, nnz)
    assert got_off[0] == 0 and got_off[-1] == nnz == len(got_idx)
    return got_off, got_idx, dt


def check_small(nat, oracle, mode, keys, off, idx, n_left=0, vsc=2):
    """Device result == the id reference as a full CSR, and == the oracle's rows once empty rows are dropped."""
    off, idx = np.asarray(off, np.int64), np.asarray(idx, np.int32)
    ids = ids_of_bytes(keys)
    want_off, want_idx, _ = reference(mode, ids, off, idx, n_left, vsc)
    payload, koff = native.NativePca._keys(keys)
    got_off, got_idx, _ = device_join(nat, mode, vsc, n_left, payload, koff, off, idx)
    assert np.array_equal(got_off, want_off) and np.array_equal(got_idx, want_idx)
    assert drop_empty(got_off, got_idx) == oracle_rows(oracle, mode, keys, off, idx, n_left, vsc)
    return got_off, got_idx


# ---- reference 2 against the oracle, then against the device ------------------------------------------------------------
def test_vectorised_murmur3_equals_the_oracle(oracle):
    rng = np.random.default_rng(1)
    for L in list(range(0, 50)) + [63, 64, 65, 127]:
        keys = rng.integers(0, 256, (4, L), dtype=np.uint8)
        got = murmur3_fixed(keys)
        for k, h in zip(keys, got):
            assert h.astype("<u8").tobytes() == oracle.np_murmur3_128(k.tobytes())


@pytest.mark.parametrize("L", [1, 8, 9, 15, 16, 17, 31, 32, 33, 40])
def test_hash_keys_of_a_million_keys(L):
    rng = np.random.default_rng(100 + L)
    nkeys = 1_000_000
    keys = rng.integers(0, 256, (nkeys, L), dtype=np.uint8)
    koff = np.arange(nkeys + 1, dtype=np.int64) * L
    out = np.zeros((nkeys, 2), np.uint64)
    with native.NativePca(64) as nat:
        rc = nat._lib.vpca_hash_keys(nat._h, _ptr(keys), _ptr(koff), nkeys, _ptr(out))
        assert rc == native.VPCA_OK
    assert np.array_equal(out, murmur3_fixed(keys))


def test_key_layout_is_one_to_one():
    ids = np.concatenate([np.arange(100_000), np.random.default_rng(2).integers(0, 1 << 40, 100_000)])
    k = id_keys(ids)
    assert np.array_equal(id_of_key(k), ids)
    assert len(np.unique(k.view(np.dtype((np.void, KEY_LEN))))) == len(np.unique(ids))


# ---- scan edges -------------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=2)
def scan_case(mode, nrows):
    """JOIN: two thirds left rows, ids over a third of nrows (about one partner per left row, repeats on both sides).
    MERGE: rows of 3 datasets with variant_set_count = 3; ids repeat 1..4 times and the union order is shuffled, so kept
    groups start anywhere in the input.  Returns the input (fixed-length keys) and the reference CSR."""
    rng = np.random.default_rng(nrows * 2 + mode)
    if mode == JOIN:
        n_left = (2 * nrows + 2) // 3
        u = max(1, nrows // 3)
        ids = np.concatenate([rng.integers(0, u, n_left), rng.integers(0, u, nrows - n_left)])
    else:
        n_left = 0
        sizes = rng.choice([1, 2, 3, 3, 3, 4], size=nrows)
        ids = rng.permutation(np.repeat(np.arange(nrows, dtype=np.int64), sizes)[:nrows])
        if nrows >= 30:    # ten kept groups of fresh ids in the last 30 rows: the last, partial block of the scan counts
            ids[-30:] = rng.permutation(np.repeat(np.arange(nrows, nrows + 10), 3))
    ids = ids.astype(np.int64) * 7919 + 11                      # spread over contigs and positions
    keys = id_keys(ids)
    off, idx = random_calls(rng, nrows)
    want = reference(mode, ids, off, idx, n_left, 3)
    koff = np.arange(nrows + 1, dtype=np.int64) * KEY_LEN
    return keys, koff, off, idx, n_left, want


@pytest.mark.parametrize("nrows", SCAN_ROWS)
@pytest.mark.parametrize("mode", [JOIN, MERGE], ids=["join", "merge3"])
def test_scan_edges(mode, nrows, oracle):
    """Regression note: with the carry of scan_blocks_kernel dropped (block_tot[i] = ex), every output row produced by an
    input row past 2^20 gets a wrong CSR offset.  Both 3 * 2^20 + 517-row cases and the large Gram below fail on it, and
    tests/test_join_gpu.py does not notice.  At 2^20 + 1 rows the one row past 2^20 is the last one: a right row (join)
    or a row that cannot start a group of 3 (merge), so no output offset is read from its block."""
    keys, koff, off, idx, n_left, (want_off, want_idx, src) = scan_case(mode, nrows)
    with native.NativePca(N) as nat:
        got_off, got_idx, dt = device_join(nat, mode, 3, n_left, keys.ravel(), koff, off, idx)
    _log(f"scan {'join' if mode == JOIN else 'merge'} nrows={nrows}: {len(want_off) - 1} rows, {len(want_idx)} calls, "
         f"last producing input row {src.max() if len(src) else -1}, {dt * 1e3:.1f} ms")
    if nrows == BIG:       # the case reaches the carry: output rows come from input rows past the second step of 2^20
        assert src.max() >= (2 << 20) and (mode == JOIN or src.max() >= (3 << 20))
    assert np.array_equal(got_off, want_off)
    assert np.array_equal(got_idx, want_idx)
    if nrows <= 1025:
        assert drop_empty(got_off, got_idx) == oracle_rows(oracle, mode, keys, off, idx, n_left, 3)


def test_gram_of_the_large_join_over_several_chunks(oracle):
    keys, koff, off, idx, n_left, (want_off, want_idx, _) = scan_case(JOIN, BIG)
    chunk = 1 << 19
    assert len(want_off) - 1 > 3 * chunk
    with native.NativePca(N, max_multiplicity=2, chunk_variants=chunk) as nat:
        device_join(nat, JOIN, 2, n_left, keys.ravel(), koff, off, idx)
        h2d = nat.stats()["h2d_bytes"]
        nat.accumulateJoined(0)
        nat.commit(0)
        assert nat.stats()["h2d_bytes"] == h2d                 # the joined rows were encoded where they were
        nat.finalizeGram()
        S = nat.getGram()
    assert np.array_equal(S, oracle.c_similarity(N, want_off, want_idx, 4))


# ---- fan-out and long probe clusters ------------------------------------------------------------------------------------
def _fanout_join(rng, heavy, n_unique):
    """Left / right ids: `heavy` = [(left rows, right rows)] of keys 0.., then n_unique keys once on the left and, 70 %
    of them, once on the right; each side shuffled."""
    left = [np.full(a, g) for g, (a, _) in enumerate(heavy)]
    right = [np.full(b, g) for g, (_, b) in enumerate(heavy)]
    u = np.arange(len(heavy), len(heavy) + n_unique)
    left = rng.permutation(np.concatenate(left + [u]))
    right = rng.permutation(np.concatenate(right + [u[rng.random(n_unique) < 0.7]]))
    return np.concatenate([left, right]).astype(np.int64), len(left)


@pytest.mark.parametrize("name,heavy,n_unique", [("one key 300 x 300", [(300, 300)], 0),
                                                 ("four keys 300 x 300 among unique keys", [(300, 300)] * 4, 20_000),
                                                 ("one key 1 x 4096", [(1, 4096)], 100)])
def test_join_fanout(name, heavy, n_unique):
    rng = np.random.default_rng(len(heavy) * 1000 + n_unique)
    ids, n_left = _fanout_join(rng, heavy, n_unique)
    ids = ids * 104729 + 5
    off, idx = random_calls(rng, len(ids), 4)
    want_off, want_idx, _ = ref_join(ids, off, idx, n_left)
    assert len(want_off) - 1 >= sum(a * b for a, b in heavy)
    with native.NativePca(N) as nat:
        got_off, got_idx, dt = device_join(nat, JOIN, 2, n_left, id_keys(ids).ravel(),
                                           np.arange(len(ids) + 1, dtype=np.int64) * KEY_LEN, off, idx)
    _log(f"fan-out join, {name}: {len(ids)} rows in, {len(want_off) - 1} rows out, {dt * 1e3:.1f} ms")
    assert np.array_equal(got_off, want_off) and np.array_equal(got_idx, want_idx)


def test_merge_groups_at_and_around_variant_set_count():
    """variant_set_count = 500: two groups of exactly 500 rows are kept, groups of 499 and 501 and 2000 single rows are
    dropped."""
    rng = np.random.default_rng(500)
    sizes = [500, 499, 501, 500] + [1] * 2000
    ids = rng.permutation(np.repeat(np.arange(len(sizes)), sizes)).astype(np.int64) * 31 + 3
    off, idx = random_calls(rng, len(ids), 4)
    want_off, want_idx, first = ref_merge(ids, off, idx, 500)
    assert len(want_off) == 3 and sorted(ids[first]) == [3, 3 * 31 + 3]
    with native.NativePca(N) as nat:
        got_off, got_idx, dt = device_join(nat, MERGE, 500, 0, id_keys(ids).ravel(),
                                           np.arange(len(ids) + 1, dtype=np.int64) * KEY_LEN, off, idx)
    _log(f"fan-out merge, groups of 499 / 500 / 501: {len(ids)} rows in, {dt * 1e3:.1f} ms")
    assert np.array_equal(got_off, want_off) and np.array_equal(got_idx, want_idx)


# ---- edge inputs --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n_left", ["none", "all"])
def test_join_with_one_side_empty(n_left, oracle):
    rng = np.random.default_rng(7)
    keys = [b"k%d" % (i % 5) for i in range(40)]
    off, idx = random_calls(rng, 40, 5)
    with native.NativePca(N) as nat:
        got_off, _ = check_small(nat, oracle, JOIN, keys, off, idx, 0 if n_left == "none" else 40)
    assert len(got_off) == 1


@pytest.mark.parametrize("mode", [JOIN, MERGE], ids=["join", "merge"])
def test_no_rows(mode):
    with native.NativePca(N) as nat:
        assert nat.joinRows(mode, [], np.zeros(1, np.int64), np.zeros(0, np.int32), 0, 2) == (0, 0)
        assert nat.joinSize() == (0, 0)
        off, idx = nat.joinFetch(0, 0)
        nat.accumulateJoined(0)
        nat.commit(0)
        nat.finalizeGram()
        assert not nat.getGram().any()
    assert off.tolist() == [0] and len(idx) == 0


@pytest.mark.parametrize("mode", [JOIN, MERGE], ids=["join", "merge"])
def test_rows_without_calls(mode, oracle):
    keys = [b"a", b"b", b"a", b"c", b"a", b"b", b"c", b"c"]
    off = np.zeros(len(keys) + 1, np.int64)
    with native.NativePca(N) as nat:
        got_off, got_idx = check_small(nat, oracle, mode, keys, off, np.zeros(0, np.int32), 4, 3 if mode == MERGE else 2)
        assert len(got_off) > 1 and not got_off.any() and len(got_idx) == 0   # rows out, every one empty
        nat.accumulateJoined(0)
        nat.commit(0)
        nat.finalizeGram()
        assert not nat.getGram().any()


@pytest.mark.parametrize("mode", [JOIN, MERGE], ids=["join", "merge"])
def test_keys_of_length_zero(mode, oracle):
    keys = [b"", b"x", b"", b"", b"x", b"", b"y"]
    off, idx = random_calls(np.random.default_rng(8), len(keys), 5)
    with native.NativePca(N) as nat:
        got_off, _ = check_small(nat, oracle, mode, keys, off, idx, 3, 4)
    assert len(got_off) - 1 == (2 * 2 + 1 if mode == JOIN else 1)      # join: 2 x 2 empty keys + x; merge: 4 empty keys


@pytest.mark.parametrize("mode", [JOIN, MERGE], ids=["join", "merge"])
def test_keys_that_are_prefixes_of_one_another(mode, oracle):
    """Every prefix of a 40-byte key (lengths 0..40 cross the 8- and 16-byte steps of the hash) is its own key."""
    rng = np.random.default_rng(9)
    full = b"chr1" + (1234567).to_bytes(8, "little") + (1234568).to_bytes(8, "little") + b"ACGTTGCAACGTTGCAACGT"
    assert len(full) == 40
    pre = [full[:L] for L in range(41)] + [full + b"\0", b"chr1\0"]
    if mode == JOIN:
        keys = [pre[i] for i in rng.permutation(len(pre))] + [pre[i] for i in rng.permutation(len(pre))]
        n_left, vsc, want_rows = len(pre), 2, len(pre)
    else:
        keys = [pre[i] for i in rng.permutation(np.repeat(np.arange(len(pre)), 2 + np.arange(len(pre)) % 2))]
        n_left, vsc, want_rows = 0, 2, (len(pre) + 1) // 2
    off, idx = random_calls(rng, len(keys), 5)
    with native.NativePca(N) as nat:
        got_off, _ = check_small(nat, oracle, mode, keys, off, idx, n_left, vsc)
    assert len(got_off) - 1 == want_rows


@pytest.mark.parametrize("mode", [JOIN, MERGE], ids=["join", "merge"])
def test_byte_identical_keys_of_different_variants(mode, oracle):
    """getVariantKey concatenates without separators (:65-73): ref AC + alt G and ref A + alt CG, and alt [C, T] and alt
    [CT], hash the same bytes, so the reference joins them; so must the device."""
    V = pkg.Variant
    a1, a2 = V("7", start=100, end=102, referenceBases="AC", alternateBases=["G"]), V("7", start=100, end=102, referenceBases="A", alternateBases=["CG"])
    b1, b2 = V("7", start=200, end=201, referenceBases="A", alternateBases=["C", "T"]), V("7", start=200, end=201, referenceBases="A", alternateBases=["CT"])
    other = V("7", start=100, end=102, referenceBases="AC", alternateBases=["T"])
    for x, y in ((a1, a2), (b1, b2)):
        assert variantKeyBytes(x) == variantKeyBytes(y)
        assert oracle.np_variant_key(x.contig, x.start, x.end, x.referenceBases, x.alternateBases) == \
            oracle.np_variant_key(y.contig, y.start, y.end, y.referenceBases, y.alternateBases)
    keys = [variantKeyBytes(v) for v in (a1, b1, other, a2, b2, other)]
    off, idx = random_calls(np.random.default_rng(10), len(keys), 5)
    with native.NativePca(N) as nat:
        got_off, _ = check_small(nat, oracle, mode, keys, off, idx, 3, 2)
    assert len(got_off) - 1 == 3


def test_merge_with_variant_set_count_one(oracle):
    """One variant set: every key seen once is a row of its own, every repeated key is dropped."""
    rng = np.random.default_rng(11)
    ids = rng.permutation(np.repeat(np.arange(600), rng.choice([1, 1, 2, 3], 600)))
    keys = [bytes(k) for k in id_keys(ids)]
    off, idx = random_calls(rng, len(keys), 5)
    with native.NativePca(N) as nat:
        got_off, _ = check_small(nat, oracle, MERGE, keys, off, idx, 0, 1)
    assert len(got_off) - 1 == int((np.bincount(ids) == 1).sum())


def test_merge_groups_from_a_single_dataset(oracle):
    """The reference counts a key's records over the union (:144): three records in one dataset form a kept group just
    like one record in each of three datasets."""
    rng = np.random.default_rng(12)
    d0 = [b"all3", b"only0", b"only0", b"two0", b"only0", b"two0", b"dup"]
    d1 = [b"all3", b"dup", b"x1"]
    d2 = [b"all3", b"two0", b"dup", b"dup"]
    keys = d0 + d1 + d2
    off, idx = random_calls(rng, len(keys), 5)
    with native.NativePca(N) as nat:
        got_off, got_idx = check_small(nat, oracle, MERGE, keys, off, idx, 0, 3)
    recs = [(k, idx[off[i]:off[i + 1]].tolist()) for i, k in enumerate(keys)]
    want = [r for r in oracle.np_merge_datasets([recs[:7], recs[7:10], recs[10:]], 3) if r]   # per dataset, as :140
    assert drop_empty(got_off, got_idx) == want
    assert len(got_off) - 1 == 3                                  # all3, only0, two0; dup (4 records) is dropped


# ---- offsets that start above zero -------------------------------------------------------------------------------------
@pytest.mark.parametrize("kpad,cpad", [(1, 1), (37, 11), ((1 << 20) + 3, (1 << 18) + 1)])
@pytest.mark.parametrize("mode", [JOIN, MERGE], ids=["join", "merge"])
def test_offsets_that_start_above_zero(mode, kpad, cpad, oracle):
    """key_offsets[0] = kpad and offsets[0] = cpad over buffers that really hold that many leading bytes / calls (filled
    with values no row holds): same result as the rebased input, for vpca_join_rows and vpca_hash_keys."""
    rng = np.random.default_rng(kpad + cpad + mode)
    pool = list(dict.fromkeys(bytes(rng.integers(0, 256, int(rng.integers(0, 41)), dtype=np.uint8)) for _ in range(3000)))
    keys = [pool[i] for i in rng.integers(0, len(pool), 5000)]
    off, idx = random_calls(rng, len(keys), 5)
    payload, koff = native.NativePca._keys(keys)
    payload_s = np.concatenate([rng.integers(0, 256, kpad, dtype=np.uint8), payload])
    idx_s = np.concatenate([np.full(cpad, 12345, np.int32), idx])
    koff_s, off_s = koff + kpad, off + cpad
    ids = ids_of_bytes(keys)
    want_off, want_idx, _ = reference(mode, ids, off, idx, 2500, 2)
    with native.NativePca(N) as nat:
        base_off, base_idx, _ = device_join(nat, mode, 2, 2500, payload, koff, off, idx)
        got_off, got_idx, _ = device_join(nat, mode, 2, 2500, payload_s, koff_s, off_s, idx_s)
        h0, h1 = np.zeros((len(keys), 2), np.uint64), np.zeros((len(keys), 2), np.uint64)
        assert nat._lib.vpca_hash_keys(nat._h, _ptr(payload), _ptr(koff), len(keys), _ptr(h0)) == native.VPCA_OK
        assert nat._lib.vpca_hash_keys(nat._h, _ptr(payload_s), _ptr(koff_s), len(keys), _ptr(h1)) == native.VPCA_OK
    assert np.array_equal(base_off, want_off) and np.array_equal(base_idx, want_idx)
    assert np.array_equal(got_off, want_off) and np.array_equal(got_idx, want_idx)
    assert np.array_equal(h1, h0)
    for q in range(0, len(keys), 499):
        assert h0[q].astype("<u8").tobytes() == oracle.np_murmur3_128(keys[q])


# ---- one context, many calls -----------------------------------------------------------------------------------------
def _id_case(rng, mode, nrows, vsc):
    if mode == JOIN:
        n_left = nrows // 2
        ids = rng.integers(0, max(1, nrows // 2), nrows)
    else:
        n_left = 0
        ids = rng.permutation(np.repeat(np.arange(nrows), rng.choice([1, vsc, vsc, vsc + 1], nrows))[:nrows])
    ids = ids.astype(np.int64)
    off, idx = random_calls(rng, nrows)
    return id_keys(ids).ravel(), np.arange(nrows + 1, dtype=np.int64) * KEY_LEN, off, idx, n_left, \
        reference(mode, ids, off, idx, n_left, vsc)


def test_one_context_reused_for_joins_of_different_sizes(oracle):
    """Large, then small (the grow-only buffers are larger than needed), then larger than the first (they grow); every
    accumulateJoined uses the latest result.  vpca_reset drops the result."""
    rng = np.random.default_rng(13)
    S_want = np.zeros((N, N), np.int64)
    with native.NativePca(N, max_multiplicity=3) as nat:
        for pid, (mode, nrows) in enumerate([(JOIN, 300_000), (MERGE, 2_000), (JOIN, 700_000)]):
            payload, koff, off, idx, n_left, (want_off, want_idx, _) = _id_case(rng, mode, nrows, 3)
            got_off, got_idx, _ = device_join(nat, mode, 3, n_left, payload, koff, off, idx)
            assert np.array_equal(got_off, want_off) and np.array_equal(got_idx, want_idx)
            nat.accumulateJoined(pid)
            nat.commit(pid)
            S_want += oracle.c_similarity(N, want_off, want_idx, 1)
            assert np.array_equal(np.tril(nat.partialGram()), np.tril(S_want))
        nat.reset()
        for call in (nat.joinSize, lambda: nat.joinFetch(0, 0), lambda: nat.accumulateJoined(9)):
            with pytest.raises(native.VpcaError) as e:
                call()
            assert e.value.code == native.VPCA_ERR_STATE


def test_refused_calls_keep_the_previous_result(oracle):
    """Every argument check runs on the host before any copy or kernel: a refused call returns VPCA_ERR_BAD_ARG and the
    result of the last good call stays in place, usable by joinFetch and accumulateJoined."""
    rng = np.random.default_rng(14)
    payload, koff, off, idx, n_left, (want_off, want_idx, _) = _id_case(rng, JOIN, 5000, 2)
    z1, k3 = np.zeros(2, np.int64), np.array([0, 3], np.int64)
    i3 = np.zeros(3, np.int32)
    refused = {
        "mode 2": (2, 2, 0, payload, koff, off, idx, None),
        "mode -1": (-1, 2, 0, payload, koff, off, idx, None),
        "n_left -1": (JOIN, 2, -1, payload, koff, off, idx, None),
        "n_left past nrows": (JOIN, 2, 5001, payload, koff, off, idx, None),
        "variant_set_count 0": (MERGE, 0, 0, payload, koff, off, idx, None),
        "variant_set_count -3": (MERGE, -3, 0, payload, koff, off, idx, None),
        "decreasing key offsets": (JOIN, 2, 1, np.zeros(8, np.uint8), np.array([0, 5, 3], np.int64), np.zeros(3, np.int64), i3, None),
        "decreasing call offsets": (JOIN, 2, 1, np.zeros(8, np.uint8), np.array([0, 1, 2], np.int64), np.array([0, 2, 1], np.int64), i3, None),
        "negative first offset": (JOIN, 2, 0, np.zeros(8, np.uint8), np.array([-1, 2], np.int64), z1, i3, None),
        "NULL payload with key bytes": (JOIN, 2, 0, None, k3, z1, i3, None),
        "NULL calls with calls": (JOIN, 2, 0, np.zeros(3, np.uint8), k3, np.array([0, 3], np.int64), None, None),
        "nrows past 0x7ffffff0": (JOIN, 2, 0, np.zeros(3, np.uint8), k3, z1, i3, 0x7ffffff1),
    }
    with native.NativePca(N, max_multiplicity=2) as nat:
        device_join(nat, JOIN, 2, n_left, payload, koff, off, idx)
        for what, (mode, vsc, nl, p, ko, o, ix, nrows) in refused.items():
            rc, _, _ = raw_join(nat, mode, vsc, nl, p, ko, o, ix, nrows)
            assert rc == native.VPCA_ERR_BAD_ARG, what
            assert nat.joinSize() == (len(want_off) - 1, len(want_idx)), what
        got_off, got_idx = nat.joinFetch(len(want_off) - 1, len(want_idx))
        nat.accumulateJoined(0)
        nat.commit(0)
        nat.finalizeGram()
        S = nat.getGram()
    assert np.array_equal(got_off, want_off) and np.array_equal(got_idx, want_idx)
    assert np.array_equal(S, oracle.c_similarity(N, want_off, want_idx, 1))


# ---- the driver from VCF files ----------------------------------------------------------------------------------------
def _write_sets(tmp_path, oracle, n_sets):
    """n_sets VCF files over shared sites (each file keeps 85 % of them), plus: a site written with alt "C,T" in even
    files and "CT" in odd ones (byte-identical keys), a site written twice in the first file (a duplicate inside one
    set), and a site without carriers in every file."""
    rng = np.random.default_rng(40 + n_sets)
    per = [20, 15, 12, 10][:n_sets]
    n = sum(per)
    nv = 400
    d = oracle.c_synth_dense(20241017, n, 0, nv + 2, 1)         # dosage 0 / 1 / 2 with population structure
    gt = {0: "0/0", 1: "0/1", 2: "1/1"}
    paths, s0 = [], 0
    for f in range(n_sets):
        rows = slice(s0, s0 + per[f])
        s0 += per[f]
        keep = rng.random(nv) < 0.85
        recs = [dict(chrom="chr3", pos=10_000 + 7 * j, ref="G", alt=["A"], gts=[gt[int(x)] for x in d[rows, j]])
                for j in range(nv) if keep[j]]
        recs.append(dict(chrom="chr3", pos=50_000, ref="A", alt=["C", "T"] if f % 2 == 0 else ["CT"],
                         gts=[gt[int(x)] for x in d[rows, nv]]))
        if f == 0:
            recs.append(dict(chrom="chr3", pos=50_100, ref="T", alt=["G"], gts=[gt[int(x)] for x in d[rows, nv + 1]]))
            recs.append(dict(chrom="chr3", pos=50_100, ref="T", alt=["G"], gts=[gt[int(x)] for x in d[rows, nv]]))
        elif f < 3:
            recs.append(dict(chrom="chr3", pos=50_100, ref="T", alt=["G"], gts=[gt[int(x)] for x in d[rows, nv + 1]]))
        recs.append(dict(chrom="chr3", pos=50_200, ref="C", alt=["A"], gts=["0/0"] * per[f]))
        paths.append(str(tmp_path / f"set{chr(97 + f)}.vcf"))
        vcf.write_vcf(paths[-1], [f"S{f}_{i:02d}" for i in range(per[f])], recs)
    return paths, per


@pytest.mark.parametrize("n_sets", [2, 4], ids=["join2", "merge4"])
def test_driver_from_vcf_files(n_sets, tmp_path, monkeypatch, capsys, oracle):
    paths, per = _write_sets(tmp_path, oracle, n_sets)
    n = sum(per)
    recs, base = [], 0
    for f, path in enumerate(paths):
        recs.append([(oracle.np_variant_key(v.contig, v.start, v.end, v.referenceBases, v.alternateBases),
                      [base + i for i, c in enumerate(v.calls) if any(a > 0 for a in c.genotype)])
                     for v in vcf.read_variants(path)])
        base += per[f]
    rows = oracle.np_join_datasets(recs[0], recs[1]) if n_sets == 2 else oracle.np_merge_datasets(recs, n_sets)
    rows = [r for r in rows if r]
    off = np.concatenate([[0], np.cumsum([len(r) for r in rows])]).astype(np.int64)
    S_want = oracle.c_similarity(n, off, np.asarray([c for r in rows for c in r], np.int32), 1)
    U_want, _ = oracle.compute_pca(S_want, 2)

    got = {}
    real_join, real_sim, real_pca = native.NativePca.joinRows, VariantsPcaDriver.getSimilarityMatrix, VariantsPcaDriver.computePca

    def join_rows(self, mode, keys, offsets, sample_idx, n_left=0, variant_set_count=2):
        got["join"] = (mode, len(keys), n_left, variant_set_count)
        return real_join(self, mode, keys, offsets, sample_idx, n_left, variant_set_count)

    def sim(self, rdd):
        m = real_sim(self, rdd)
        got["S"] = m.toArray().copy()
        return m

    def pca(self, m):
        got["pcs"] = real_pca(self, m)
        return got["pcs"]
    monkeypatch.setattr(native.NativePca, "joinRows", join_rows)
    monkeypatch.setattr(VariantsPcaDriver, "getSimilarityMatrix", sim)
    monkeypatch.setattr(VariantsPcaDriver, "computePca", pca)
    variants_pca.main(["--vcf-path", ",".join(paths)])
    lines = [ln for ln in capsys.readouterr().out.splitlines() if ln.count("\t") == 3]

    mode, nrows, n_left, vsc = got["join"]
    assert nrows == sum(len(r) for r in recs)
    if n_sets == 2:
        assert (mode, n_left) == (JOIN, len(recs[0]))
    else:
        assert (mode, vsc) == (MERGE, n_sets)
    assert np.array_equal(got["S"], S_want)
    ids = [cid for cid, _, _ in got["pcs"]]
    assert ids == [f"{vcf.dataset_stem(p)}-{i}" for p, m in zip(paths, per) for i in range(m)]
    assert np.all(oracle.eigvec_rel_err(np.array([[a, b] for _, a, b in got["pcs"]]), U_want) <= 1e-6)
    assert len(lines) == n
