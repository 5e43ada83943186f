"""LD pruning on the GPU (vpca_ld_prune_bed, DESIGN.md 9): the keep mask, the pair list and the r2 bits against the numpy
restatement (tests/ld_ref.py) -- sample counts from 2 to 100 000 (the sample-axis split), missing data, several contigs
and chunks, the window limit, thresholds, truncation, the counted allele, repeated calls, the state it must leave alone,
and the driver end to end against a plain run on the fileset of the kept variants."""
import ctypes

import numpy as np
import pytest

import ld_ref
from kinship_ref import dosage_codes, king_pairs
from spark_examples_b200 import native, plink, variants_pca
from spark_examples_b200.conf import PcaConf
from spark_examples_b200.variants_pca import VariantsPcaDriver, check_ld_flags

pytestmark = pytest.mark.gpu


def _bits(a):
    return np.ascontiguousarray(a, np.float64).view(np.int64)


def _planted(rng, n, v, block=6, copy=0.85, missing=0.02):
    """(n, v) A1 counts with LD blocks: each variant copies its block's founder on a `copy` share of the samples."""
    d = np.empty((n, v), np.int64)
    for b0 in range(0, v, block):
        p = rng.uniform(0.05, 0.5)
        founder = rng.binomial(2, p, size=n)
        for j in range(b0, min(v, b0 + block)):
            own = rng.binomial(2, rng.uniform(0.05, 0.5), size=n)
            d[:, j] = np.where(rng.random(n) < copy, founder, own)
    d[rng.random((n, v)) < missing] = -1
    return d


def _layout(rng, v, contigs=3, step_bp=(200, 3000)):
    """Sorted contigs and positions: `contigs` runs, random steps (ties included)."""
    names = np.repeat([str(c + 1) for c in range(contigs)], -(-v // contigs))[:v].tolist()
    pos = np.cumsum(rng.integers(step_bp[0], step_bp[1], size=v))
    pos[rng.random(v) < 0.05] = 0
    pos = np.maximum.accumulate(pos) + 1
    return names, pos


def _rows(dosage):
    """(n, v) A1 counts, -1 missing -> (v, ceil(n / 4)) .bed rows."""
    codes = dosage_codes(dosage)
    pad = (-codes.shape[1]) % 4
    codes = np.concatenate([codes, np.zeros((codes.shape[0], pad), np.uint8)], axis=1)
    c4 = codes.reshape(codes.shape[0], -1, 4)
    return (c4[:, :, 0] | (c4[:, :, 1] << 2) | (c4[:, :, 2] << 4) | (c4[:, :, 3] << 6)).astype(np.uint8)


def _run(nat, rows, lo, r2_max, max_pairs=None):
    """keep, all listed pairs (or the first max_pairs), their r2, and the total the count-only call reports."""
    keep0, _, _ = nat.ldPruneBed(rows, lo, r2_max)
    total = ctypes.c_int64(0)
    L = native.load_library()
    k = np.zeros(max(len(lo), 1), np.uint8)
    assert L.vpca_ld_prune_bed(nat._h, rows.ctypes.data, rows.shape[0], rows.shape[1], np.ascontiguousarray(lo).ctypes.data,
                               float(r2_max), k.ctypes.data, 0, None, None, ctypes.byref(total)) == native.VPCA_OK
    p = int(total.value) if max_pairs is None else max_pairs
    keep, pairs, r2 = nat.ldPruneBed(rows, lo, r2_max, max_pairs=p)
    assert np.array_equal(keep, keep0) and np.array_equal(keep, k[:len(lo)] != 0)
    return keep, pairs, r2, int(total.value)


def _check(nat, rows, n, lo, r2_max):
    keep, pairs, r2, total = _run(nat, rows, lo, r2_max)
    want_keep, want_pairs, want_r2 = ld_ref.prune(rows, n, lo, r2_max)
    assert total == len(want_pairs)
    np.testing.assert_array_equal(pairs, want_pairs)
    np.testing.assert_array_equal(_bits(r2), _bits(want_r2))
    np.testing.assert_array_equal(keep, want_keep)
    return keep, pairs, r2


@pytest.mark.parametrize("n", [2, 3, 129, 1000, 2504])
def test_matches_reference(n):
    rng = np.random.default_rng(100 + n)
    v = 2600
    d = _planted(rng, n, v)
    contigs, pos = _layout(rng, v)
    lo = plink.window_starts([plink.BimRecord(c, "x", int(p), "A", "G") for c, p in zip(contigs, pos)], 150)
    h = int(np.max(np.arange(v) - lo))
    assert 40 < h < 200 and v > 1024 + h                                # several chunks: windows cross chunk boundaries
    rows = _rows(d)
    with native.NativePca(n) as nat:
        keep, pairs, _ = _check(nat, rows, n, lo, 0.2)
        if n >= 129:
            assert len(pairs) > 0 and 0 < keep.sum() < v
        assert not any(contigs[i] != contigs[j] for i, j in pairs.tolist())


def test_hundred_thousand_samples_split_the_sample_axis():
    rng = np.random.default_rng(7)
    n, v = 100000, 1300
    d = _planted(rng, n, v, block=4, copy=0.6, missing=0.01)
    pos = np.arange(v) * 1000 + 1
    lo = plink.window_starts([plink.BimRecord("1", "x", int(p), "A", "G") for p in pos], 50)
    rows = _rows(d)
    with native.NativePca(n) as nat:
        keep, pairs, _ = _check(nat, rows, n, lo, 0.1)
    assert len(pairs) > 0 and 0 < keep.sum() < v


def test_missing_monomorphic_and_duplicates():
    rng = np.random.default_rng(8)
    n, v = 157, 400
    d = _planted(rng, n, v, missing=0.1)
    d[:, 5] = -1                                      # all-missing variant
    d[11, :] = -1                                     # all-missing sample
    d[:, 9] = 1                                       # monomorphic
    d[:, 10] = 2
    d[:, 20] = d[:, 17]                               # exact duplicates: r2 = 1
    d[:, 300] = d[:, 299]
    lo = np.maximum(0, np.arange(v) - 40)
    rows = _rows(d)
    with native.NativePca(n) as nat:
        keep, pairs, r2 = _check(nat, rows, n, lo, 0.3)
        listed = {tuple(p): r for p, r in zip(pairs.tolist(), r2.tolist())}
        assert listed[(17, 20)] == 1.0 and listed[(299, 300)] == 1.0
        assert not any(5 in p or 9 in p or 10 in p for p in listed)
        assert keep[5] and keep[9] and keep[10] and not keep[20] and not keep[300]
        assert np.all(r2 <= 1.0)
        _check(nat, rows, n, lo, 0.0)                 # R2 = 0: every pair with a nonzero covariance


def test_threshold_equal_to_an_attained_r2_is_strict():
    rng = np.random.default_rng(9)
    n, v = 300, 500
    d = _planted(rng, n, v)
    lo = np.maximum(0, np.arange(v) - 25)
    rows = _rows(d)
    with native.NativePca(n) as nat:
        _, pairs, r2, _ = _run(nat, rows, lo, 0.0)
        t = float(np.sort(r2)[len(r2) // 2])
        keep_t, pairs_t, r2_t = _check(nat, rows, n, lo, t)
        assert np.all(r2_t > t) and (r2 == t).any()
        assert len(pairs_t) == int(np.sum(r2 > t))
        for thr in (0.05, 0.5, 0.8, 0.999):
            _check(nat, rows, n, lo, thr)


def test_windows_with_no_partner_and_one_variant():
    rng = np.random.default_rng(10)
    n = 64
    with native.NativePca(n) as nat:
        d = _planted(rng, n, 300)
        lo = np.arange(300)                           # every window holds only the variant itself
        keep, pairs, r2, total = _run(nat, _rows(d), lo, 0.0)
        assert keep.all() and total == 0 and len(pairs) == 0
        keep, pairs, _, total = _run(nat, _rows(d[:, :1]), np.zeros(1, np.int64), 0.5)
        assert keep.tolist() == [True] and total == 0
        keep, pairs, _, total = _run(nat, np.zeros((0, 16), np.uint8), np.zeros(0, np.int64), 0.5)
        assert len(keep) == 0 and total == 0


def test_window_at_the_limit_and_one_past_it():
    rng = np.random.default_rng(11)
    w = native.LD_MAX_WINDOW
    n, v = 96, w + 300
    d = rng.binomial(2, 0.3, size=(n, v)).astype(np.int64)
    d[:, w] = d[:, 0]                                 # partners exactly H = w apart
    d[:, w + 150] = d[:, 150]
    d[:, 200] = d[:, 190]
    lo = np.maximum(0, np.arange(v) - w)
    rows = _rows(d)
    with native.NativePca(n) as nat:
        keep, pairs, _ = _check(nat, rows, n, lo, 0.9)
        assert {(0, w), (150, w + 150), (190, 200)} <= {tuple(p) for p in pairs.tolist()}
        assert not keep[w] and not keep[w + 150] and not keep[200]
        over = lo.copy()
        over[w + 1] = 0                               # H = w + 1
        with pytest.raises(native.VpcaError) as ei:
            nat.ldPruneBed(rows, over, 0.9)
        assert ei.value.code == native.VPCA_ERR_UNSUPPORTED and f"variant {w + 1}" in str(ei.value)


def test_max_pairs_truncation_and_repeats():
    rng = np.random.default_rng(12)
    n, v = 200, 1500
    d = _planted(rng, n, v)
    lo = np.maximum(0, np.arange(v) - 120)
    rows = _rows(d)
    with native.NativePca(n) as nat:
        keep, pairs, r2, total = _run(nat, rows, lo, 0.1)
        assert total > 100
        for m in (1, 7, total // 3, total - 1, total, total + 5):
            k2, p2, r2b = nat.ldPruneBed(rows, lo, 0.1, max_pairs=m)
            assert np.array_equal(k2, keep)
            np.testing.assert_array_equal(p2, pairs[:m])
            np.testing.assert_array_equal(_bits(r2b), _bits(r2[:m]))
        k3, p3, r3 = nat.ldPruneBed(rows, lo, 0.1, max_pairs=total)
        np.testing.assert_array_equal(p3, pairs)
        np.testing.assert_array_equal(_bits(r3), _bits(r2))
        np.testing.assert_array_equal(k3, keep)


def test_counted_allele_does_not_matter():
    rng = np.random.default_rng(13)
    n, v = 333, 700
    d = _planted(rng, n, v)
    flipped = np.where(d >= 0, 2 - d, -1)             # what counting A2 sees
    lo = np.maximum(0, np.arange(v) - 60)
    with native.NativePca(n) as nat:
        ka, pa, ra, _ = _run(nat, _rows(d), lo, 0.2)
        kb, pb, rb, _ = _run(nat, _rows(flipped), lo, 0.2)
    np.testing.assert_array_equal(ka, kb)
    np.testing.assert_array_equal(pa, pb)
    np.testing.assert_array_equal(_bits(ra), _bits(rb))


def test_bad_arguments():
    n = 10
    L = native.load_library()
    rows = np.zeros((4, 3), np.uint8)
    lo = np.zeros(4, np.int64)
    keep = np.zeros(4, np.uint8)
    tot = ctypes.c_int64(0)
    with native.NativePca(n) as nat:
        def call(r=rows.ctypes.data, nv=4, stride=3, w=lo.ctypes.data, r2=0.5, k=keep.ctypes.data, mp=0, op=None, orr=None):
            return L.vpca_ld_prune_bed(nat._h, r, nv, stride, w, r2, k, mp, op, orr, ctypes.byref(tot))
        assert call() == native.VPCA_OK
        assert call(r=None) == native.VPCA_ERR_BAD_ARG
        assert call(w=None) == native.VPCA_ERR_BAD_ARG
        assert call(k=None) == native.VPCA_ERR_BAD_ARG
        assert call(stride=2) == native.VPCA_ERR_BAD_ARG                     # < ceil(10 / 4)
        for r2 in (float("nan"), float("inf"), -0.01, 1.0):
            assert call(r2=r2) == native.VPCA_ERR_BAD_ARG
        for bad in ([0, 2, 1, 1], [0, 0, 1, 0], [-1, 0, 0, 0], [0, 1, 1, 2]):
            wl = np.asarray(bad, np.int64)
            assert call(w=wl.ctypes.data) == (native.VPCA_OK if bad == [0, 1, 1, 2] else native.VPCA_ERR_BAD_ARG)
        assert call(mp=3) == native.VPCA_ERR_BAD_ARG                         # listing without outputs


def test_leaves_gram_and_kinship_alone():
    rng = np.random.default_rng(14)
    n, v = 150, 900
    d = _planted(rng, n, v)
    rows = _rows(d)
    lo = np.maximum(0, np.arange(v) - 50)
    with native.NativePca(n, num_pc=3) as nat:
        nat.kinshipBed(rows)
        nat.accumulateBed(0, rows, plink.COUNT_A1)
        nat.commit(0)
        nat.finalizeGram()
        vecs0, ev0, _ = nat.computePca(3)
        S0, (ids0, c0, k0) = nat.getGram(), nat.kinshipPairs()
        keep, pairs, r2, _ = _run(nat, rows, lo, 0.2)
        S1, (ids1, c1, k1) = nat.getGram(), nat.kinshipPairs()
        np.testing.assert_array_equal(S0, S1)
        np.testing.assert_array_equal(ids0, ids1)
        np.testing.assert_array_equal(c0, c1)
        np.testing.assert_array_equal(_bits(k0), _bits(k1))
        w0, _ = nat.loadingsBed(3, rows, plink.COUNT_A1)
        nat.ldPruneBed(rows, lo, 0.2)
        w1, _ = nat.loadingsBed(3, rows, plink.COUNT_A1)
        np.testing.assert_array_equal(_bits(w0), _bits(w1))                 # U untouched
        keep2, pairs2, r22, _ = _run(nat, rows, lo, 0.2)
    np.testing.assert_array_equal(keep, keep2)
    np.testing.assert_array_equal(pairs, pairs2)
    np.testing.assert_array_equal(_bits(r2), _bits(r22))


def _sample_lines(text):
    return {ln.split("\t")[0]: ln for ln in text.splitlines() if ln.count("\t") == 3}


def _driver_gram(argv):
    conf = PcaConf(argv)
    driver = VariantsPcaDriver(conf)
    calls = driver.getCallsRdd(driver.getData)
    if conf.ldPrune.isDefined:
        driver.ldPrune(calls, check_ld_flags(conf, plink.read_bim(conf.bedPath())))
    S = driver.getSimilarityMatrix(calls).toArray().copy()
    driver.stop()
    return S


def test_driver_end_to_end_matches_a_run_on_the_kept_variants(tmp_path, capsys):
    rng = np.random.default_rng(15)
    n, v = 240, 3000
    d = _planted(rng, n, v, block=5)
    d[: n // 2] = np.where(d[: n // 2] >= 0, np.minimum(2, d[: n // 2] + (rng.random((n // 2, v)) < 0.2)), -1)
    d[7] = d[3]                                                              # a duplicate sample for the KING table
    contigs, pos = _layout(rng, v, contigs=2)
    fam = [(f"F{i % 5}", f"S{i:03d}") for i in range(n)]
    prefix = str(tmp_path / "all")
    plink.write_fileset(prefix, d, fam=fam, contigs=contigs, positions=pos)
    out = str(tmp_path / "run")
    common = ["--variants-per-partition", "700", "--num-pc", "3"]
    variants_pca.main(["--bed-path", prefix, "--ld-prune", "0.25", "--ld-window-kb", "120", "--output-path", out,
                       "--make-king-table", out + ".kin0", "--save-loadings", out + ".npz"] + common)
    text = capsys.readouterr().out
    bim = plink.read_bim(prefix)
    lo = plink.window_starts(bim, 120)
    keep, _, _ = ld_ref.prune(plink.BedFile(prefix).rows(0, v), n, lo, 0.25)
    m = int(keep.sum())
    assert 0 < m < v
    assert f"LD prune r2 > 0.25 within 120 kb: {m} of {v} variants kept." in text
    kept_ids = open(out + ".prune.in").read().split()
    assert kept_ids == [bim[j].id for j in np.flatnonzero(keep)]
    assert open(out + ".prune.out").read().split() == [bim[j].id for j in np.flatnonzero(~keep)]
    sub = str(tmp_path / "kept")
    plink.write_fileset(sub, d[:, keep], fam=fam, contigs=[c for c, k in zip(contigs, keep) if k], positions=pos[keep])
    ref = str(tmp_path / "ref")
    variants_pca.main(["--bed-path", sub, "--make-king-table", ref + ".kin0", "--save-loadings", ref + ".npz"] + common)
    plain = capsys.readouterr().out
    got_lines, want_lines = _sample_lines(text), _sample_lines(plain)
    assert len(got_lines) == n and got_lines == want_lines                 # PCs: the same bits
    assert open(out + ".kin0").read() == open(ref + ".kin0").read()
    ids, _, _ = king_pairs(dosage_codes(d[:, keep]), -np.inf)
    assert len(open(ref + ".kin0").read().splitlines()) == len(ids) + 1
    with np.load(out + ".npz") as a, np.load(ref + ".npz") as b:
        np.testing.assert_array_equal(a["keys"], b["keys"])
        np.testing.assert_array_equal(_bits(a["loadings"]), _bits(b["loadings"]))
        np.testing.assert_array_equal(a["count"], b["count"])
        assert a["keys"].shape[0] == m
    S_pruned = _driver_gram(["--bed-path", prefix, "--ld-prune", "0.25", "--ld-window-kb", "120"] + common)
    S_plain = _driver_gram(["--bed-path", sub] + common)
    capsys.readouterr()
    np.testing.assert_array_equal(S_pruned, S_plain)
    # the counted allele does not change the kept set
    variants_pca.main(["--bed-path", prefix, "--ld-prune", "0.25", "--ld-window-kb", "120", "--bed-counted-allele", "A2",
                       "--output-path", str(tmp_path / "a2")] + common)
    capsys.readouterr()
    assert open(str(tmp_path / "a2") + ".prune.in").read() == open(out + ".prune.in").read()
