"""KING-robust kinship on the GPU (vpca_kinship_bed / vpca_kinship_pairs, DESIGN.md 7): counts and kinship bit for bit
against numpy integer products of the genotype planes (tests/kinship_ref.py), selection order and truncation, the PCA
Gram left alone, planted relatives in KING's degree intervals, the sample and overflow limits, and the driver flags."""
import numpy as np
import pytest

from kinship_ref import MISSING, dosage_codes, king_pairs, kinship_value, pack_codes, pair_counts
from spark_examples_b200 import native, plink, variants_pca

pytestmark = pytest.mark.gpu


def _codes(rng, n, nv, missing=0.01):
    """Random genotypes with per-variant allele frequencies and about `missing` missing calls."""
    p = rng.uniform(0.05, 0.95, size=nv)[:, None]
    d = (rng.random((nv, n)) < p).astype(np.int64) + (rng.random((nv, n)) < p)
    c = dosage_codes(d.T)
    c[rng.random((nv, n)) < missing] = MISSING
    return c


def _assert_same(got, want):
    ids, counts, kin = got
    wids, wcounts, wkin = want
    np.testing.assert_array_equal(ids, wids)
    np.testing.assert_array_equal(counts, wcounts)
    assert kin.dtype == np.float64
    np.testing.assert_array_equal(kin.view(np.int64), wkin.view(np.int64))    # same bits, NaN included


@pytest.mark.parametrize("n", [2, 3, 5, 127, 128, 129, 1000, 2504])
def test_counts_and_kinship_bit_exact(n):
    """Every pair at -inf against numpy; small staging chunks (chunk_nnz: 96 rows or more) push the rows through many
    chunks, and N % 4 != 0 leaves padding bits in the last byte of a row."""
    rng = np.random.default_rng(1000 + n)
    nv = 3000 if n > 1000 else 5000
    codes = _codes(rng, n, nv)
    rows = pack_codes(codes)
    with native.NativePca(n, chunk_nnz=max(1024, 24 * rows.shape[1])) as nat:
        nat.kinshipBed(rows)
        _assert_same(nat.kinshipPairs(), king_pairs(codes))


def test_n_one_cannot_make_a_context():
    """A single sample has no pair; vpca_create needs n_samples >= 2 for every path, kinship included."""
    with pytest.raises(native.VpcaError) as e:
        native.NativePca(1)
    assert e.value.code == native.VPCA_ERR_BAD_ARG


def test_rows_past_one_chunk_and_wide_stride():
    """Rows past one default staging chunk, with rows padded beyond ceil(N / 4) bytes."""
    rng = np.random.default_rng(7)
    n, nv = 301, 70000
    codes = _codes(rng, n, nv)
    rows = pack_codes(codes)
    wide = np.concatenate([rows, np.full((nv, 5), 0xFF, np.uint8)], axis=1)     # junk after the row is never read
    with native.NativePca(n) as nat:
        nat.kinshipBed(wide)
        _assert_same(nat.kinshipPairs(), king_pairs(codes))


def test_split_calls_equal_one_call():
    rng = np.random.default_rng(11)
    n, nv = 133, 9001
    codes = _codes(rng, n, nv)
    rows = pack_codes(codes)
    with native.NativePca(n) as one, native.NativePca(n, chunk_nnz=1024) as many:
        one.kinshipBed(rows)
        for lo, hi in [(0, 1), (1, 33), (33, 4000), (4000, 4000), (4000, 9001)]:
            many.kinshipBed(rows[lo:hi])
        _assert_same(many.kinshipPairs(), one.kinshipPairs())
        _assert_same(one.kinshipPairs(), king_pairs(codes))


def test_all_missing_sample_gives_nan_pairs():
    rng = np.random.default_rng(5)
    n, nv = 40, 2000
    codes = _codes(rng, n, nv)
    codes[:, 17] = MISSING
    with native.NativePca(n) as nat:
        nat.kinshipBed(pack_codes(codes))
        ids, counts, kin = nat.kinshipPairs()
        with17 = (ids == 17).any(axis=1)
        assert with17.sum() == n - 1 and np.isnan(kin[with17]).all() and (counts[with17] == 0).all()
        assert not np.isnan(kin[~with17]).any()
        _assert_same((ids, counts, kin), king_pairs(codes))
        fids, _, fkin = nat.kinshipPairs(-1e300)                       # any finite threshold drops NaN pairs
        assert len(fids) == len(ids) - (n - 1) and not (fids == 17).any() and np.isfinite(fkin).all()


def test_threshold_order_and_truncation():
    rng = np.random.default_rng(3)
    n, nv = 300, 4000
    codes = _codes(rng, n, nv)
    for a, b in [(3, 250), (10, 11), (0, 299)]:                         # a few duplicates so that some pairs pass
        codes[:, b] = codes[:, a]
    with native.NativePca(n) as nat:
        nat.kinshipBed(pack_codes(codes))
        for thr in [0.3, 0.0, -0.05, 0.5, 0.6]:
            want = king_pairs(codes, thr)
            got = nat.kinshipPairs(thr)
            _assert_same(got, want)
            assert (got[2] >= thr).all()
            order = got[0][:, 1].astype(np.int64) * n + got[0][:, 0]
            assert (np.diff(order) > 0).all() and (got[0][:, 0] < got[0][:, 1]).all()
        ids, _, _ = nat.kinshipPairs(0.3)
        assert {tuple(p) for p in ids.tolist()} == {(3, 250), (10, 11), (0, 299)}
        full = king_pairs(codes, 0.0)
        for m in [0, 1, 7, len(full[0]) - 1, len(full[0]), len(full[0]) + 5]:
            got = nat.kinshipPairs(0.0, max_pairs=m)
            _assert_same(got, tuple(x[:m] for x in full))
        # the raw ABI: a count-only call with NULL outputs, and the total reported past max_pairs
        L, total = native.load_library(), native.ctypes.c_int64(-1)
        assert L.vpca_kinship_pairs(nat._h, 0.0, 0, None, None, None, native.ctypes.byref(total)) == native.VPCA_OK
        assert total.value == len(full[0])
        ids3, cnt3, kin3 = np.zeros((3, 2), np.int32), np.zeros((3, 5), np.int32), np.zeros(3)
        total.value = -1
        assert L.vpca_kinship_pairs(nat._h, 0.0, 3, ids3.ctypes.data, cnt3.ctypes.data, kin3.ctypes.data,
                                    native.ctypes.byref(total)) == native.VPCA_OK
        assert total.value == len(full[0])
        _assert_same((ids3, cnt3, kin3), tuple(x[:3] for x in full))


def test_dtypes_give_identical_output():
    rng = np.random.default_rng(9)
    n, nv = 257, 6000
    rows = pack_codes(_codes(rng, n, nv))
    outs = []
    for dt in [native.DTYPE_I8, native.DTYPE_BF16, native.DTYPE_E2M1]:
        with native.NativePca(n, dtype=dt) as nat:
            nat.kinshipBed(rows)
            outs.append(nat.kinshipPairs())
    _assert_same(outs[1], outs[0])
    _assert_same(outs[2], outs[0])


def test_pca_gram_untouched_and_reset_zeroes_counts():
    rng = np.random.default_rng(13)
    n, nv = 200, 5000
    codes = _codes(rng, n, nv)
    rows = pack_codes(codes)
    with native.NativePca(n) as plain:
        plain.accumulateBed(0, rows[:2500])
        plain.accumulateBed(1, rows[2500:])
        plain.commit(0)
        plain.commit(1)
        plain.finalizeGram()
        S_plain = plain.getGram()
    with native.NativePca(n) as nat:
        with pytest.raises(native.VpcaError) as e:
            nat.kinshipPairs()
        assert e.value.code == native.VPCA_ERR_STATE                     # nothing added since creation
        nat.kinshipBed(rows[:1000])
        nat.accumulateBed(0, rows[:2500])
        nat.kinshipBed(rows[1000:])
        nat.accumulateBed(1, rows[2500:])
        nat.commit(0)
        nat.commit(1)
        nat.finalizeGram()
        before = nat.kinshipPairs()
        nat.computePca(2)
        nat.kinshipBed(rows[:0])                                          # an empty call changes nothing
        np.testing.assert_array_equal(nat.getGram(), S_plain)
        _assert_same(nat.kinshipPairs(), before)
        _assert_same(before, king_pairs(codes))
        nat.setGram(S_plain)                                             # the PCA Gram's calls leave the counts alone
        _assert_same(nat.kinshipPairs(), before)
        nat.reset()
        with pytest.raises(native.VpcaError) as e:
            nat.kinshipPairs()
        assert e.value.code == native.VPCA_ERR_STATE
        nat.kinshipBed(rows[:100])                                       # counts start from zero again
        _assert_same(nat.kinshipPairs(), king_pairs(codes[:100]))


def _pedigree(rng, nv):
    """Seeded haplotypes of a pedigree: founders, then children made of one random haplotype of each parent per variant."""
    p = rng.uniform(0.1, 0.9, size=nv)
    hap = {}

    def founder(name):
        hap[name] = (rng.random(nv) < p, rng.random(nv) < p)

    def child(name, mother, father):
        pick = lambda who: np.where(rng.random(nv) < 0.5, hap[who][0], hap[who][1])
        hap[name] = (pick(mother), pick(father))

    for f in ["F1", "F2", "F3", "F4", "F5", "F6", "F7", "U1", "U2", "U3", "U4"]:
        founder(f)
    child("C1", "F1", "F2")          # full sibs, children of F1 x F2
    child("C2", "F1", "F2")
    child("C3", "F1", "F3")          # half sib of C1 / C2 through F1
    child("G1", "C1", "F4")          # first cousins: children of the full sibs C1 and C2
    child("G2", "C2", "F5")
    hap["D1"] = hap["U1"]            # duplicate of U1
    names = list(hap)
    dosage = np.stack([hap[s][0].astype(np.int64) + hap[s][1] for s in names])   # A1 counts
    return names, dosage


def test_planted_relatives_fall_in_king_degree_intervals():
    rng = np.random.default_rng(20240901)
    nv = 50000
    names, dosage = _pedigree(rng, nv)
    codes = dosage_codes(dosage)
    codes[rng.random(codes.shape) < 0.01] = MISSING
    n = len(names)
    at = {s: i for i, s in enumerate(names)}
    with native.NativePca(n) as nat:
        nat.kinshipBed(pack_codes(codes))
        ids, counts, kin = nat.kinshipPairs()
    _assert_same((ids, counts, kin), king_pairs(codes))
    k = {(names[a], names[b]): float(v) for (a, b), v in zip(ids.tolist(), kin)}
    get = lambda x, y: k[(x, y)] if (x, y) in k else k[(y, x)]
    related = {("U1", "D1"): (0.354, 1.0),                                   # duplicate
               ("F1", "C1"): (0.177, 0.354), ("F2", "C2"): (0.177, 0.354),   # parent-offspring
               ("C1", "G1"): (0.177, 0.354),
               ("C1", "C2"): (0.177, 0.354),                                 # full sibs
               ("C1", "C3"): (0.0884, 0.177), ("C2", "C3"): (0.0884, 0.177),  # half sibs
               ("F1", "G1"): (0.0884, 0.177),                                # grandparent
               ("G1", "G2"): (0.0442, 0.0884)}                               # first cousins
    for (x, y), (lo, hi) in related.items():
        assert lo < get(x, y) <= hi, (x, y, get(x, y))
    expected_related = {frozenset(p) for p in related} | {frozenset(p) for p in [
        ("F2", "C1"), ("F1", "C2"), ("F1", "C3"), ("F3", "C3"), ("C2", "G2"), ("F4", "G1"), ("F5", "G2"), ("C1", "G2"),
        ("C2", "G1"), ("F2", "G1"), ("F1", "G2"), ("F2", "G2"), ("C3", "G1"), ("C3", "G2")]}
    for (x, y), v in k.items():
        if frozenset((x, y)) not in expected_related:
            assert v < 0.0442, (x, y, v)                                     # unrelated


def test_sample_limit_pairs_and_refusals():
    """N = 21 845 (3N = 65 535): sampled pairs against direct numpy counts, the first pairs in order, a duplicate planted at
    samples 0 and 21 844, the total at -inf; N = 21 846 and band-only contexts are refused."""
    n, nv = native.KINSHIP_MAX_SAMPLES, 2048
    rng = np.random.default_rng(21845)
    codes = _codes(rng, n, nv)
    codes[:, n - 1] = codes[:, 0]
    with native.NativePca(n) as nat:
        nat.kinshipBed(pack_codes(codes))
        ids, counts, kin = nat.kinshipPairs(0.09)
        dup = np.flatnonzero((ids[:, 0] == 0) & (ids[:, 1] == n - 1))
        assert len(dup) == 1 and kin[dup[0]] == 0.5
        order = ids[:, 1].astype(np.int64) * n + ids[:, 0]
        assert (np.diff(order) > 0).all() and (kin >= 0.09).all()
        first = nat.kinshipPairs(max_pairs=3000)
        sample = np.concatenate([np.arange(len(ids)), np.arange(len(ids), len(ids) + 3000)])
        all_ids = np.concatenate([ids, first[0]])
        all_counts = np.concatenate([counts, first[1]])
        all_kin = np.concatenate([kin, first[2]])
        pick = rng.choice(len(sample), size=min(len(sample), 600), replace=False)
        for i in pick:
            a, b = all_ids[i]
            want = pair_counts(codes, int(a), int(b))
            assert tuple(all_counts[i]) == want, (a, b)
            w = kinship_value(want[1], want[2], want[3], want[4])
            assert np.float64(all_kin[i]).view(np.int64) == np.float64(w).view(np.int64)
        b3, a3 = np.tril_indices(80, -1)
        np.testing.assert_array_equal(first[0], np.stack([a3, b3], axis=1)[:3000])
        total = native.ctypes.c_int64(0)
        assert native.load_library().vpca_kinship_pairs(nat._h, float("-inf"), 0, None, None, None,
                                                        native.ctypes.byref(total)) == native.VPCA_OK
        assert total.value == n * (n - 1) // 2
    with native.NativePca(n + 1) as big:
        with pytest.raises(native.VpcaError) as e:
            big.kinshipBed(pack_codes(codes[:10, :1].repeat(n + 1, axis=1)))
        assert e.value.code == native.VPCA_ERR_UNSUPPORTED
        with pytest.raises(native.VpcaError) as e:
            big.kinshipPairs()
        assert e.value.code == native.VPCA_ERR_UNSUPPORTED
    with native.NativePca(64, gram_band=(0, 32)) as band:
        with pytest.raises(native.VpcaError) as e:
            band.kinshipBed(pack_codes(codes[:10, :64]))
        assert e.value.code == native.VPCA_ERR_UNSUPPORTED


def test_bad_arguments():
    with native.NativePca(10) as nat:
        L = native.load_library()
        rows = np.zeros((4, 3), np.uint8)
        assert L.vpca_kinship_bed(nat._h, rows.ctypes.data, 4, 2) == native.VPCA_ERR_BAD_ARG     # stride < ceil(10 / 4)
        assert L.vpca_kinship_bed(nat._h, None, 4, 3) == native.VPCA_ERR_BAD_ARG
        nat.kinshipBed(rows)
        total = native.ctypes.c_int64(0)
        assert L.vpca_kinship_pairs(nat._h, 0.0, 5, None, None, None, native.ctypes.byref(total)) == native.VPCA_ERR_BAD_ARG
        assert L.vpca_kinship_pairs(nat._h, 0.0, 0, None, None, None, None) == native.VPCA_ERR_BAD_ARG


def test_overflow_bound_at_two_to_the_31():
    """N <= 4 puts one byte in a row: 2^30 rows of homozygous-A1 calls count exactly 2^30 in every pair, and a further 2^30
    rows would pass 2^31 - 1 and are refused before any of them is read."""
    n = 4
    rows = np.zeros((1 << 30, 1), np.uint8)                                # code 00 everywhere: hom A1
    with native.NativePca(n) as nat:
        nat.kinshipBed(rows)
        ids, counts, kin = nat.kinshipPairs()
        assert len(ids) == 6 and (counts[:, 0] == 1 << 30).all() and (counts[:, 1:] == 0).all() and np.isnan(kin).all()
        with pytest.raises(native.VpcaError) as e:
            nat.kinshipBed(rows)
        assert e.value.code == native.VPCA_ERR_OVERFLOW
        _assert_same(nat.kinshipPairs(), (ids, counts, kin))
        nat.kinshipBed(rows[:(1 << 30) - 1])                                  # up to 2^31 - 1 in all is allowed
        assert (nat.kinshipPairs()[1][:, 0] == (1 << 31) - 1).all()


def test_driver_writes_the_king_table_and_the_same_pcs(tmp_path, capsys):
    rng = np.random.default_rng(2024)
    names, dosage = _pedigree(rng, 6000)
    extra = (rng.random((40, 6000)) < 0.4).astype(np.int64) + (rng.random((40, 6000)) < 0.4)
    dosage = np.concatenate([dosage, extra])
    dosage[rng.random(dosage.shape) < 0.01] = -1
    n = dosage.shape[0]
    fam = [(f"fam{i % 3}", f"I{i:03d}") for i in range(n)]
    prefix = str(tmp_path / "cohort")
    plink.write_fileset(prefix, dosage, fam=fam)
    base = ["--bed-path", prefix, "--variants-per-partition", "2500"]
    variants_pca.main(base)
    plain = capsys.readouterr().out.splitlines()
    table = str(tmp_path / "cohort.kin0")
    variants_pca.main(base + ["--make-king-table", table, "--king-table-filter", "0.0442"])
    king = capsys.readouterr().out.splitlines()
    stats = lambda lines: [ln for ln in lines if not ln.startswith("GPU stats:")]
    assert stats(king) == stats(plain) and any(ln.count("\t") == 3 for ln in plain)
    codes = dosage_codes(dosage)
    ids, counts, kin = king_pairs(codes, 0.0442)
    want = [variants_pca.KING_HEADER.rstrip("\n")] + [
        f"{fam[a][0]}\t{fam[a][1]}\t{fam[b][0]}\t{fam[b][1]}\t{c[0]}\t{c[1]}\t{c[2]}\t{float(k)!r}"
        for (a, b), c, k in zip(ids.tolist(), counts.tolist(), kin)]
    lines = open(table, encoding="utf-8").read().splitlines()
    assert lines == want and len(lines) > 10
    for ln, k in zip(lines[1:], kin):
        assert float(ln.split("\t")[7]) == k
