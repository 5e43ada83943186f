"""Variant QC on the GPU (vpca_variant_qc_bed, vpca_hwe_exact, vpca_ld_prune_bed_masked; DESIGN.md 10): counts bit-exact
against numpy from 1 to 100 000 samples (padding bits, wide strides, all-missing rows, staging-chunk edges, any split of
the rows), HWE p-value bits against the Python-float restatement (tests/qc_ref.py) up to 10^6 samples, bad arguments, the
state left alone, the masked LD prune against a prune of the compacted rows, and the driver end to end against plain
runs on a fileset of the QC-passing variants."""
import ctypes

import numpy as np
import pytest

import ld_ref
import qc_ref
from kinship_ref import dosage_codes
from spark_examples_b200 import native, plink, variants_pca
from spark_examples_b200.conf import PcaConf
from spark_examples_b200.variants_pca import VariantsPcaDriver, check_ld_flags, variant_qc_keep

pytestmark = pytest.mark.gpu

STAGE_BYTES = 64 << 20   # vpca_variant_qc_bed stages this many row bytes per chunk


def _bits(a):
    return np.ascontiguousarray(a, np.float64).view(np.int64)


def _rows(dosage):
    """(n, v) A1 counts, -1 missing -> (v, ceil(n / 4)) .bed rows."""
    codes = dosage_codes(dosage)
    pad = (-codes.shape[1]) % 4
    codes = np.concatenate([codes, np.zeros((codes.shape[0], pad), np.uint8)], axis=1)
    c4 = codes.reshape(codes.shape[0], -1, 4)
    return (c4[:, :, 0] | (c4[:, :, 1] << 2) | (c4[:, :, 2] << 4) | (c4[:, :, 3] << 6)).astype(np.uint8)


def _random_rows(rng, n, nv, extra=0):
    """Random bytes: every code, random padding bits in the last byte, `extra` junk bytes past ceil(n / 4)."""
    rows = rng.integers(0, 256, size=(nv, (n + 3) // 4 + extra), dtype=np.uint8)
    if nv >= 4:
        rows[1, :] = 0x55                                                  # all missing
        rows[2, :] = 0x00                                                  # all HOM_A1, padding read as 00 too
        rows[3, :] = 0xFF                                                  # all HOM_A2, padding bits set
    return rows


def _check_counts(nat, rows, n, hwe=True):
    c, p = nat.variantQcBed(rows, hwe=hwe)
    want = qc_ref.counts(rows, n)
    np.testing.assert_array_equal(c, want)
    assert np.all(c.sum(1) == n)
    return c, p


@pytest.mark.parametrize("n", [2, 3, 4, 5, 129, 1000, 2504, 100000])   # a context holds at least 2 samples
def test_counts_are_exact(n):
    rng = np.random.default_rng(n)
    nv = 300 if n < 100000 else 64
    with native.NativePca(n) as nat:
        for extra in (0, 5, 8 - ((n + 3) // 4) % 8):                       # tight, odd and 8-byte-aligned strides
            rows = _random_rows(rng, n, nv, extra)
            c, p = _check_counts(nat, rows, n)
            np.testing.assert_array_equal(_bits(p), _bits(qc_ref.hwe_p_many(c)))
        # any split of the rows into calls gives the same counts
        rows = _random_rows(rng, n, nv)
        whole, _ = nat.variantQcBed(rows, hwe=False)
        parts = [nat.variantQcBed(rows[a:b], hwe=False)[0] for a, b in ((0, 1), (1, 77), (77, nv))]
        np.testing.assert_array_equal(np.concatenate(parts), whole)
        assert nat.variantQcBed(rows, hwe=False)[1] is None


@pytest.mark.parametrize("n", [2504, 100000])
def test_counts_across_staging_chunks(n):
    rng = np.random.default_rng(7)
    stride = (n + 3) // 4
    per_chunk = STAGE_BYTES // stride
    with native.NativePca(n) as nat:
        # 2504 samples: two chunks make one HWE batch of 2^18 rows at most, so 2 per_chunk + 1 rows cross a batch edge
        for nv in (per_chunk - 1, per_chunk, per_chunk + 1) + ((2 * per_chunk + 1,) if n == 2504 else ()):
            rows = _random_rows(rng, n, nv)
            c, p = _check_counts(nat, rows, n)
            edge = per_chunk if nv <= per_chunk + 1 else 2 * per_chunk
            sel = np.r_[0:40, edge - 20:nv]                                  # both sides of the chunk / batch edge
            np.testing.assert_array_equal(_bits(p[sel]), _bits(qc_ref.hwe_p_many(c[sel])))


def _hw_counts(rng, n, v, deviation=0.0):
    """Counts drawn at HWE (deviation 0) or with a planted het deficit / excess, some missing calls."""
    q = rng.uniform(0.01, 0.5, size=v)
    f = deviation * rng.choice([-1.0, 1.0], size=v)
    het = np.clip(2 * q * (1 - q) * (1 - f), 0, 1)
    a = np.clip(q * q + f * q * (1 - q), 0, 1)
    b = np.clip(1 - a - het, 0, 1)
    pr = np.stack([a, het, b], 1)
    pr /= pr.sum(1, keepdims=True)
    called = n - rng.binomial(n, 0.01, size=v)
    c = np.stack([rng.multinomial(m, p) for m, p in zip(called, pr)])
    return np.concatenate([c, (n - called)[:, None]], axis=1).astype(np.int32)


@pytest.mark.parametrize("n", [7, 500, 2504, 20000])
def test_hwe_bits_match_the_restatement(n):
    rng = np.random.default_rng(50 + n)
    c = np.concatenate([_hw_counts(rng, n, 200), _hw_counts(rng, n, 200, 0.3), _hw_counts(rng, n, 50, 0.9)])
    with native.NativePca(max(n, 2)) as nat:
        p = nat.hweExact(c)
    want = qc_ref.hwe_p_many(c)
    np.testing.assert_array_equal(_bits(p), _bits(want))
    assert np.all((p >= 0) & (p <= 1))
    if n >= 500:
        assert (p < 1e-6).sum() > 20 and (p > 0.05).sum() > 100             # both regimes are exercised


def test_hwe_at_a_million_samples():
    rng = np.random.default_rng(3)
    n = 1000000
    c = np.concatenate([_hw_counts(rng, n, 12), _hw_counts(rng, n, 12, 0.005)])
    c[0] = [250000, 500000, 250000, 0]                                      # the mode at q = 0.5
    c[1] = [n - 1, 1, 0, 0]                                                 # a singleton
    with native.NativePca(2) as nat:                                       # host counts: any n, whatever the context
        p = nat.hweExact(c)
    np.testing.assert_array_equal(_bits(p), _bits(qc_ref.hwe_p_many(c)))
    assert p[0] == 1.0


def test_special_variants():
    c = np.array([[0, 0, 0, 9],                # nothing called
                  [40, 0, 0, 0], [0, 0, 40, 0],  # monomorphic
                  [0, 1, 0, 0], [1, 0, 0, 0],    # n = 1
                  [0, 40, 0, 0],                 # all het
                  [20, 0, 20, 0],                # no het at q = 0.5
                  [10, 20, 10, 0]],              # the mode
                 np.int32)
    with native.NativePca(4) as nat:
        p = nat.hweExact(c)
        empty = nat.hweExact(np.zeros((0, 4), np.int32))
    assert empty.shape == (0,)
    np.testing.assert_array_equal(_bits(p), _bits(qc_ref.hwe_p_many(c)))
    assert p[:5].tolist() == [1.0] * 5 and p[7] == 1.0
    assert p[5] < 1e-10 and p[6] < 1e-10 and np.all(p <= 1.0)


def test_bad_arguments():
    n = 10
    L = native.load_library()
    rows = np.zeros((4, 3), np.uint8)
    out = np.zeros((4, 4), np.int32)
    p = np.zeros(4)
    with native.NativePca(n) as nat:
        def qc(r=rows.ctypes.data, nv=4, stride=3, o=out.ctypes.data, pp=p.ctypes.data):
            return L.vpca_variant_qc_bed(nat._h, r, nv, stride, o, pp)
        assert qc() == native.VPCA_OK and qc(pp=None) == native.VPCA_OK
        assert qc(r=None) == native.VPCA_ERR_BAD_ARG
        assert qc(o=None) == native.VPCA_ERR_BAD_ARG
        assert qc(stride=2) == native.VPCA_ERR_BAD_ARG                       # < ceil(10 / 4)
        assert qc(nv=-1) == native.VPCA_ERR_BAD_ARG
        assert qc(r=None, o=None, nv=0) == native.VPCA_OK

        def hwe(c, nv=None, pp=p.ctypes.data):
            c = np.ascontiguousarray(c, np.int32)
            return L.vpca_hwe_exact(nat._h, c.ctypes.data, len(c) if nv is None else nv, pp)
        good = np.array([[1, 2, 3, 4]], np.int32)
        assert hwe(good) == native.VPCA_OK
        assert hwe(good, pp=None) == native.VPCA_ERR_BAD_ARG
        assert hwe([[1, 2, 3, -4]]) == native.VPCA_OK                        # MISSING is not read
        for bad in ([-1, 2, 3, 0], [1, -2, 3, 0], [1, 2, -3, 0], [2 ** 30, 2 ** 30, 0, 0], [2 ** 31 - 1, 1, 0, 0]):
            assert hwe([[0, 1, 1, 0], bad]) == native.VPCA_ERR_BAD_ARG
        assert hwe([[2 ** 31 - 3, 1, 1, 0]]) == native.VPCA_OK              # sum exactly 2^31 - 1
        with pytest.raises(native.VpcaError):
            nat.hweExact([[0, 0, -1, 0]])
        lo = np.zeros(4, np.int64)
        keep = np.zeros(4, np.uint8)
        tot = ctypes.c_int64(0)
        for el, rc in (([1, 1, 0, 1], native.VPCA_OK), ([1, 2, 0, 1], native.VPCA_ERR_BAD_ARG)):
            e = np.asarray(el, np.uint8)
            assert L.vpca_ld_prune_bed_masked(nat._h, rows.ctypes.data, 4, 3, lo.ctypes.data, e.ctypes.data, 0.5,
                                              keep.ctypes.data, 0, None, None, ctypes.byref(tot)) == rc


def _planted(rng, n, v, block=6, copy=0.85, missing=0.02):
    d = np.empty((n, v), np.int64)
    for b0 in range(0, v, block):
        founder = rng.binomial(2, rng.uniform(0.02, 0.5), size=n)
        for j in range(b0, min(v, b0 + block)):
            own = rng.binomial(2, rng.uniform(0.005, 0.5), size=n)
            d[:, j] = np.where(rng.random(n) < copy, founder, own)
    d[rng.random((n, v)) < missing] = -1
    return d


def test_leaves_gram_kinship_and_ld_alone():
    rng = np.random.default_rng(14)
    n, v = 150, 900
    rows = _rows(_planted(rng, n, v))
    lo = np.maximum(0, np.arange(v) - 50)
    with native.NativePca(n, num_pc=3) as nat:
        nat.kinshipBed(rows)
        nat.accumulateBed(0, rows, plink.COUNT_A1)
        nat.commit(0)
        nat.finalizeGram()
        nat.computePca(3)
        S0, (ids0, c0, k0) = nat.getGram(), nat.kinshipPairs()
        w0, _ = nat.loadingsBed(3, rows, plink.COUNT_A1)
        ld0 = nat.ldPruneBed(rows, lo, 0.2, max_pairs=10 ** 6)
        c1, p1 = nat.variantQcBed(rows)
        nat.hweExact(c1)
        S1, (ids1, c_1, k1) = nat.getGram(), nat.kinshipPairs()
        w1, _ = nat.loadingsBed(3, rows, plink.COUNT_A1)
        ld1 = nat.ldPruneBed(rows, lo, 0.2, max_pairs=10 ** 6)
        c2, p2 = nat.variantQcBed(rows)
    np.testing.assert_array_equal(S0, S1)
    np.testing.assert_array_equal(ids0, ids1)
    np.testing.assert_array_equal(c0, c_1)
    np.testing.assert_array_equal(_bits(k0), _bits(k1))
    np.testing.assert_array_equal(_bits(w0), _bits(w1))
    for a, b in zip(ld0, ld1):
        np.testing.assert_array_equal(a, b)
    np.testing.assert_array_equal(c1, c2)
    np.testing.assert_array_equal(_bits(p1), _bits(p2))


def _layout(rng, v, contigs=2):
    names = np.repeat([str(c + 1) for c in range(contigs)], -(-v // contigs))[:v].tolist()
    pos = np.maximum.accumulate(np.cumsum(rng.integers(200, 3000, size=v))) + 1
    return names, pos


def test_masked_prune_matches_the_compacted_rows():
    rng = np.random.default_rng(21)
    n, v = 400, 3000
    rows = _rows(_planted(rng, n, v))
    contigs, pos = _layout(rng, v)
    lo = plink.window_starts([plink.BimRecord(c, "x", int(p), "A", "G") for c, p in zip(contigs, pos)], 150)
    with native.NativePca(n) as nat:
        plain = nat.ldPruneBed(rows, lo, 0.2, max_pairs=10 ** 6)
        ones = nat.ldPruneBed(rows, lo, 0.2, max_pairs=10 ** 6, eligible=np.ones(v, bool))
        for a, b in zip(plain, ones):                                      # an all-ones mask: the same bits
            np.testing.assert_array_equal(np.asarray(a).view(np.uint8), np.asarray(b).view(np.uint8))
        for share in (0.9, 0.5, 0.1, 0.0):
            el = rng.random(v) < share
            keep, pairs, r2 = nat.ldPruneBed(rows, lo, 0.2, max_pairs=10 ** 6, eligible=el)
            idx = np.flatnonzero(el)
            sub_lo = np.searchsorted(idx, lo[idx], side="left")
            k, p, r = nat.ldPruneBed(rows[idx], sub_lo, 0.2, max_pairs=10 ** 6)
            want_keep = np.zeros(v, bool)
            want_keep[idx] = k
            np.testing.assert_array_equal(keep, want_keep)
            np.testing.assert_array_equal(pairs, idx[p].reshape(-1, 2))
            np.testing.assert_array_equal(_bits(r2), _bits(r))
            if len(idx) == 0:
                assert not keep.any() and len(pairs) == 0
                continue
            wk, wp, _ = ld_ref.prune(rows[idx], n, sub_lo, 0.2)
            np.testing.assert_array_equal(k, wk)
            np.testing.assert_array_equal(p, wp)


def _qc_dosage(rng, n, v):
    d = _planted(rng, n, v, block=5)
    d[: n // 2] = np.where(d[: n // 2] >= 0, np.minimum(2, d[: n // 2] + (rng.random((n // 2, v)) < 0.2)), -1)
    bad = rng.choice(v, size=v // 10, replace=False)
    for k, j in enumerate(bad.tolist()):
        if k % 3 == 0:
            d[:, j] = np.where(rng.random(n) < 0.1, -1, d[:, j])           # often missing
        elif k % 3 == 1:
            d[:, j] = np.where(rng.random(n) < 0.9, 1, d[:, j])            # mostly het
        else:
            d[:, j] = np.where(rng.random(n) < 0.98, 0, d[:, j])           # rare
    d[7] = d[3]                                                            # a duplicate sample for the KING table
    return d


def _sample_lines(text):
    return {ln.split("\t")[0]: ln for ln in text.splitlines() if ln.count("\t") == 3}


def _driver_gram(argv):
    conf = PcaConf(argv)
    driver = VariantsPcaDriver(conf)
    calls = driver.getCallsRdd(driver.getData)
    qc = driver.variantQc(calls) if conf.maf.isDefined else None
    if conf.ldPrune.isDefined:
        driver.ldPrune(calls, check_ld_flags(conf, plink.read_bim(conf.bedPath())), qc)
    S = driver.getSimilarityMatrix(calls).toArray().copy()
    driver.stop()
    return S


def test_driver_end_to_end_matches_a_run_on_the_passing_variants(tmp_path, capsys):
    rng = np.random.default_rng(15)
    n, v = 240, 3000
    d = _qc_dosage(rng, n, v)
    contigs, pos = _layout(rng, v)
    fam = [(f"F{i % 5}", f"S{i:03d}") for i in range(n)]
    prefix = str(tmp_path / "all")
    plink.write_fileset(prefix, d, fam=fam, contigs=contigs, positions=pos)
    flags = ["--maf", "0.05", "--geno", "0.02", "--hwe", "1e-6"]
    common = ["--variants-per-partition", "700", "--num-pc", "3"]
    out = str(tmp_path / "run")
    variants_pca.main(["--bed-path", prefix] + flags + ["--output-path", out, "--make-king-table", out + ".kin0",
                                                        "--save-loadings", out + ".npz"] + common)
    text = capsys.readouterr().out
    c = qc_ref.counts(plink.BedFile(prefix).rows(0, v), n)
    keep, by = variant_qc_keep(c, qc_ref.hwe_p_many(c), 0.05, 0.02, 1e-6)
    m = int(keep.sum())
    g, h, f = (int((by == k).sum()) for k in (1, 2, 3))
    assert 0 < m < v and g > 0 and h > 0 and f > 0
    assert (f"Variant QC: {m} of {v} variants kept ({g} by --geno 0.02, {h} by --hwe 1e-06, {f} by --maf 0.05 "
            f"removed).") in text
    hardy = open(out + ".hardy").read().splitlines()
    assert len(hardy) == v + 1
    np.testing.assert_array_equal(_bits([float(ln.split("\t")[9]) for ln in hardy[1:]]), _bits(qc_ref.hwe_p_many(c)))
    sub = str(tmp_path / "kept")
    plink.write_fileset(sub, d[:, keep], fam=fam, contigs=[x for x, k in zip(contigs, keep) if k], positions=pos[keep])
    ref = str(tmp_path / "ref")
    variants_pca.main(["--bed-path", sub, "--make-king-table", ref + ".kin0", "--save-loadings", ref + ".npz"] + common)
    plain = capsys.readouterr().out
    got_lines, want_lines = _sample_lines(text), _sample_lines(plain)
    assert len(got_lines) == n and got_lines == want_lines                 # PCs: the same bits
    assert open(out + ".kin0").read() == open(ref + ".kin0").read()
    with np.load(out + ".npz") as a, np.load(ref + ".npz") as b:
        np.testing.assert_array_equal(a["keys"], b["keys"])
        np.testing.assert_array_equal(_bits(a["loadings"]), _bits(b["loadings"]))
        np.testing.assert_array_equal(a["count"], b["count"])
        assert a["keys"].shape[0] == m
    np.testing.assert_array_equal(_driver_gram(["--bed-path", prefix] + flags + common),
                                  _driver_gram(["--bed-path", sub] + common))
    # QC, then LD pruning of the passing variants: --ld-prune on the fileset of the passing variants
    ld = ["--ld-prune", "0.2", "--ld-window-kb", "120"]
    variants_pca.main(["--bed-path", prefix] + flags + ld + ["--output-path", out + "_ld"] + common)
    text = capsys.readouterr().out
    variants_pca.main(["--bed-path", sub] + ld + ["--output-path", ref + "_ld"] + common)
    plain = capsys.readouterr().out
    assert _sample_lines(text) == _sample_lines(plain)
    idx = np.flatnonzero(keep)                                             # variant k of `sub` is variant idx[k]
    for suffix in (".prune.in", ".prune.out"):
        sub_ids = open(ref + "_ld" + suffix).read().split()
        assert open(out + "_ld" + suffix).read().split() == [f"rs{idx[int(i[2:]) - 1] + 1}" for i in sub_ids]
    k_ld = len(open(ref + "_ld.prune.in").read().split())
    assert 0 < k_ld < m and f"LD prune r2 > 0.2 within 120 kb: {k_ld} of {m} variants kept." in text
    np.testing.assert_array_equal(_driver_gram(["--bed-path", prefix] + flags + ld + common),
                                  _driver_gram(["--bed-path", sub] + ld + common))
