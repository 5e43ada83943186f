"""--maf / --geno / --hwe without a GPU: the float restatement of the exact HWE test (tests/qc_ref.py) against exact
rational p-values, the count reference, `variant_qc_keep` and its attribution order, every refusal of the flags (raised
before a context exists), the PLINK 2 reports read back, and the driver's masks with and without --ld-prune."""
from fractions import Fraction

import numpy as np
import pytest

import ld_ref
import qc_ref
from spark_examples_b200 import plink, variants_pca
from spark_examples_b200.conf import PcaConf
from spark_examples_b200.variants_common import BedSlice
from spark_examples_b200.variants_pca import (VariantsPcaDriver, check_ld_flags, check_qc_flags, variant_qc_keep,
                                              write_qc_reports)


def _pack(dosage):
    """(n, v) A1 counts, -1 missing -> (v, ceil(n / 4)) .bed rows, through plink.write_fileset's encoding."""
    d = np.asarray(dosage)
    code = np.full(d.T.shape, 1, np.uint8)
    code[d.T == 2], code[d.T == 1], code[d.T == 0] = 0, 2, 3
    pad = (-d.shape[0]) % 4
    code = np.concatenate([code, np.zeros((code.shape[0], pad), np.uint8)], axis=1)
    c4 = code.reshape(code.shape[0], -1, 4)
    return (c4[:, :, 0] | (c4[:, :, 1] << 2) | (c4[:, :, 2] << 4) | (c4[:, :, 3] << 6)).astype(np.uint8)


def test_count_reference():
    rng = np.random.default_rng(1)
    d = rng.integers(-1, 3, size=(13, 9))
    c = qc_ref.counts(_pack(d), 13)
    for k, code in ((qc_ref.HOM_A1, 2), (qc_ref.HET, 1), (qc_ref.HOM_A2, 0), (qc_ref.MISSING, -1)):
        np.testing.assert_array_equal(c[:, k], (d == code).sum(0))
    assert np.all(c.sum(1) == 13)


def _random_counts(rng, n, v):
    out = []
    for _ in range(v):
        q = rng.uniform(0.001, 0.5)
        f = rng.uniform(0.0, 0.3)                                  # inbreeding-like deviation, both signs below
        if rng.random() < 0.5:
            f = -f * 0.5
        p_het = min(1.0, max(0.0, 2 * q * (1 - q) * (1 - f)))
        p_a = max(0.0, q * q + f * q * (1 - q))
        g = rng.choice(3, size=n, p=np.array([p_a, p_het, max(0.0, 1 - p_a - p_het)]) / (p_a + p_het +
                                                                                          max(0.0, 1 - p_a - p_het)))
        out.append([(g == 0).sum(), (g == 1).sum(), (g == 2).sum(), 0])
    return np.asarray(out, np.int64)


@pytest.mark.parametrize("n", [1, 2, 3, 7, 50, 333, 2000])
def test_restatement_matches_exact_rational(n):
    rng = np.random.default_rng(n)
    c = _random_counts(rng, n, 40 if n < 2000 else 12)
    edge = [[n, 0, 0, 0], [0, 0, n, 0], [0, n, 0, 0], [n - n // 2, n // 2, 0, 0], [0, 1, n - 1, 0]]
    for a, h, b, _ in np.concatenate([c, np.asarray(edge, np.int64)]).tolist():
        got = qc_ref.hwe_p(a, h, b)
        want, gap = qc_ref.hwe_p_exact(a, h, b)
        assert gap > 1e-9, f"near-tie at {(a, h, b)}: the tolerance would decide"
        assert 0.0 <= got <= 1.0
        w = float(want)
        if w >= 1e-280:
            assert abs(got - w) <= 1e-9 * w, (a, h, b, got, w)
        else:
            assert got < 1e-270


def test_special_cases():
    assert qc_ref.hwe_p(0, 0, 0) == 1.0                            # nothing called
    assert qc_ref.hwe_p(10, 0, 0) == 1.0 and qc_ref.hwe_p(0, 0, 10) == 1.0   # monomorphic
    assert qc_ref.hwe_p(0, 1, 0) == 1.0                            # n = 1: one het is the only configuration
    assert qc_ref.hwe_p(1, 0, 0) == 1.0
    assert qc_ref.hwe_p(0, 100, 0) < 1e-25                         # all het
    assert qc_ref.hwe_p(0, 100, 0) == float(qc_ref.hwe_p_exact(0, 100, 0)[0]) or \
        abs(qc_ref.hwe_p(0, 100, 0) / float(qc_ref.hwe_p_exact(0, 100, 0)[0]) - 1) < 1e-9
    assert qc_ref.hwe_p(50, 0, 50) < 1e-25                         # no het at q = 0.5
    assert qc_ref.hwe_p_exact(25, 50, 25)[0] == Fraction(1)        # the mode itself
    # the counted allele (which homozygote is A1) makes no difference
    assert qc_ref.hwe_p(30, 17, 3) == qc_ref.hwe_p(3, 17, 30)


def test_extreme_deviation_underflows_to_zero():
    # at n = 1e5 all het is e^-(~7e4) away from the mode: every term reached from the mode underflows first
    assert qc_ref.hwe_p(0, 100000, 0) == 0.0


def test_keep_and_attribution_order():
    #             HOM_A1 HET HOM_A2 MISSING
    c = np.array([[40, 40, 20, 0],      # kept
                  [40, 40, 10, 10],     # 10 % missing: --geno
                  [0, 100, 0, 0],       # all het: --hwe
                  [99, 1, 0, 0],        # maf 0.005: --maf
                  [0, 100, 0, 20],      # fails --geno and --hwe: --geno first
                  [0, 0, 0, 100],       # nothing called: --geno, and --maf when alone
                  [50, 0, 0, 0]],       # monomorphic: --maf
                 np.int32)
    p = qc_ref.hwe_p_many(c)
    keep, by = variant_qc_keep(c, p, 0.01, 0.05, 1e-6)
    np.testing.assert_array_equal(keep, [1, 0, 0, 0, 0, 0, 0])
    np.testing.assert_array_equal(by, [0, 1, 2, 3, 1, 1, 3])
    keep, by = variant_qc_keep(c, p, 0.01, None, None)
    np.testing.assert_array_equal(by, [0, 0, 0, 3, 0, 3, 3])
    keep, by = variant_qc_keep(c, p, None, None, 1e-6)
    np.testing.assert_array_equal(by, [0, 0, 2, 0, 2, 0, 0])
    keep, by = variant_qc_keep(c, None, None, 0.1, None)           # F_MISS = 0.1 is not > 0.1
    np.testing.assert_array_equal(by, [0, 0, 0, 0, 1, 1, 0])
    keep, _ = variant_qc_keep(c, p, 0.0, 1.0, 0.0)                 # the loosest values remove only n = 0 (by --maf)
    np.testing.assert_array_equal(keep, [1, 1, 1, 1, 1, 0, 1])
    # the kept set is the intersection, whatever the order
    for maf, geno, hwe in ((0.01, None, None), (None, 0.05, None), (None, None, 1e-6)):
        k1, _ = variant_qc_keep(c, p, maf, geno, hwe)
        all_keep, _ = variant_qc_keep(c, p, 0.01, 0.05, 1e-6)
        assert np.all(all_keep <= k1)


def test_maf_boundary_follows_the_definition():
    # f = 20 / 200 = 0.1 exactly: kept (the test is MAF < X); f = 180 / 200 = 0.9 gives 1 - f = 0.09999999999999998,
    # rounded once as defined, so the mirrored variant falls just below 0.1
    c = np.array([[10, 0, 90, 0], [90, 0, 10, 0], [91, 0, 9, 0], [9, 0, 91, 0]], np.int32)
    assert 1.0 - 0.9 < 0.1
    keep, _ = variant_qc_keep(c, None, 0.1, None, None)
    np.testing.assert_array_equal(keep, [1, 0, 0, 0])
    keep, _ = variant_qc_keep(c, None, 0.09, None, None)                # 1 - 0.91 = 0.08999999999999997 < 0.09
    np.testing.assert_array_equal(keep, [1, 1, 0, 1])


@pytest.fixture
def no_context(monkeypatch):
    """Any attempt to create a context fails the test: the refusals must come first."""
    def _native(self, n):
        raise AssertionError("a native context was requested")
    monkeypatch.setattr(VariantsPcaDriver, "_native", _native)


def _fileset(tmp_path, d=None, n=12, v=40):
    rng = np.random.default_rng(0)
    prefix = str(tmp_path / "c")
    d = rng.integers(0, 3, size=(n, v)) if d is None else d
    plink.write_fileset(prefix, d, fam=[(f"F{i}", f"I{i}") for i in range(d.shape[0])])
    return prefix


@pytest.mark.parametrize("argv, match", [
    (["--synthetic", "20,100", "--maf", "0.05"], "--bed-path"),
    (["--synthetic", "20,100", "--geno", "0.1", "--hwe", "1e-6"], "--bed-path"),
    (["BED", "--maf", "0.05", "--checkpoint-path", "ck"], "checkpoint"),
    (["BED", "--hwe", "1e-6", "--project-loadings", "l.npz"], "project-loadings"),
    (["BED", "--maf", "0.6"], r"--maf takes a value in \[0, 0.5\]"),
    (["BED", "--maf=-0.01"], r"--maf takes a value in \[0, 0.5\]"),
    (["BED", "--maf", "nan"], r"--maf takes a value in \[0, 0.5\]"),
    (["BED", "--geno", "1.5"], r"--geno takes a value in \[0, 1\]"),
    (["BED", "--geno", "inf"], r"--geno takes a value in \[0, 1\]"),
    (["BED", "--hwe", "2"], r"--hwe takes a value in \[0, 1\]"),
    (["BED", "--hwe=-1e-6"], r"--hwe takes a value in \[0, 1\]"),
    (["BED", "--hwe=-inf"], r"--hwe takes a value in \[0, 1\]"),
])
def test_flag_refusals(tmp_path, no_context, argv, match):
    prefix = _fileset(tmp_path)
    argv = [a if a != "BED" else "--bed-path" for a in argv]
    if argv[0] == "--bed-path":
        argv.insert(1, prefix)
    with pytest.raises(ValueError, match=match):
        variants_pca.main(argv)


def test_multi_rank_refused(tmp_path, no_context, monkeypatch):
    monkeypatch.setenv("WORLD_SIZE", "2")
    with pytest.raises(ValueError, match="WORLD_SIZE"):
        variants_pca.main(["--bed-path", _fileset(tmp_path), "--geno", "0.1"])


def test_flags_parse():
    conf = PcaConf(["--bed-path", "c", "--maf", "0.05", "--geno", "0.02", "--hwe", "1e-6"])
    assert conf.maf() == 0.05 and conf.geno() == 0.02 and conf.hwe() == 1e-6
    check_qc_flags(conf)
    plain = PcaConf([])
    assert not (plain.maf.isDefined or plain.geno.isDefined or plain.hwe.isDefined)
    check_qc_flags(plain)
    check_qc_flags(PcaConf(["--bed-path", "c", "--maf", "0.5", "--geno", "0", "--hwe", "1"]))   # the range ends


def _read_table(path):
    lines = open(path, encoding="utf-8").read().splitlines()
    return lines[0].split("\t"), [ln.split("\t") for ln in lines[1:]]


def test_reports_read_back(tmp_path):
    c = np.array([[40, 40, 20, 0], [0, 0, 0, 7], [3, 1, 0, 3], [0, 7, 0, 0]], np.int32)
    p = qc_ref.hwe_p_many(c)
    bim = [plink.BimRecord("1", f"rs{j}", 100 + j, "A", "G") for j in range(4)]
    write_qc_reports(str(tmp_path / "q"), bim, c, p)
    head, rows = _read_table(tmp_path / "q.afreq")
    assert head == ["#CHROM", "ID", "REF", "ALT", "ALT_FREQS", "OBS_CT"]
    assert [r[:4] for r in rows] == [["1", f"rs{j}", "G", "A"] for j in range(4)]
    assert [float(r[4]) for r in rows][0] == 0.6 and np.isnan(float(rows[1][4]))
    assert float(rows[2][4]) == 7 / 8 and float(rows[3][4]) == 0.5
    assert [int(r[5]) for r in rows] == [200, 0, 8, 14]
    head, rows = _read_table(tmp_path / "q.vmiss")
    assert head == ["#CHROM", "ID", "MISSING_CT", "OBS_CT", "F_MISS"]
    assert [(int(r[2]), int(r[3]), float(r[4])) for r in rows] == [(0, 100, 0.0), (7, 7, 1.0), (3, 7, 3 / 7), (0, 7, 0.0)]
    head, rows = _read_table(tmp_path / "q.hardy")
    assert head == ["#CHROM", "ID", "A1", "AX", "HOM_A1_CT", "HET_A1_CT", "TWO_AX_CT", "O(HET_A1)", "E(HET_A1)", "P"]
    assert rows[0][2:7] == ["A", "G", "40", "40", "20"]
    assert float(rows[0][7]) == 0.4 and float(rows[0][8]) == (2 * 0.6) * (1 - 0.6)
    assert [float(r[9]) for r in rows] == p.tolist()                  # the same doubles
    assert np.isnan(float(rows[1][7])) and float(rows[1][9]) == 1.0


class QcDouble:
    """vpca_variant_qc_bed and vpca_ld_prune_bed_masked computed with the host references: the masked prune is the plain
    prune of the eligible rows alone, its window starts recomputed, mapped back to all rows."""

    def __init__(self, n):
        self.n = n

    def variantQcBed(self, rows, hwe=True):
        c = qc_ref.counts(np.asarray(rows), self.n)
        return c, (qc_ref.hwe_p_many(c) if hwe else None)

    def ldPruneBed(self, rows, window_lo, r2_max, max_pairs=0, eligible=None):
        rows = np.asarray(rows)
        lo = np.asarray(window_lo, np.int64)
        if eligible is None:
            eligible = np.ones(len(rows), bool)
        idx = np.flatnonzero(eligible)
        sub_lo = np.searchsorted(idx, lo[idx], side="left")              # first eligible variant at or after window_lo
        k, pairs, r2 = ld_ref.prune(rows[idx], self.n, sub_lo, r2_max)
        keep = np.zeros(len(rows), bool)
        keep[idx] = k
        return keep, idx[pairs][:max_pairs], r2[:max_pairs]


def _qc_fileset(tmp_path, n=60, v=90):
    rng = np.random.default_rng(9)
    base = rng.integers(0, 3, size=(n, 1))
    d = np.where(rng.random((n, v)) < 0.6, base, rng.integers(0, 3, size=(n, v)))
    d[:, 5] = 0                                                       # monomorphic
    d[:, 11] = np.where(rng.random(n) < 0.2, -1, d[:, 11])            # often missing
    d[:, 17] = 1                                                      # all het
    d[:, 23] = np.where(np.arange(n) == 0, 1, 0)                      # a singleton
    positions = np.arange(v) * 300 + 1
    prefix = str(tmp_path / "c")
    plink.write_fileset(prefix, d, contigs=["1"] * 45 + ["2"] * 45, positions=positions)
    return prefix, d


def test_driver_masks_slices_and_writes_reports(tmp_path, monkeypatch, capsys):
    prefix, d = _qc_fileset(tmp_path)
    n, v = d.shape
    argv = ["--bed-path", prefix, "--maf", "0.05", "--geno", "0.05", "--hwe", "1e-6", "--variants-per-partition", "16",
            "--output-path", str(tmp_path / "out")]
    driver = VariantsPcaDriver(PcaConf(argv))
    monkeypatch.setattr(VariantsPcaDriver, "_native", lambda self, n: QcDouble(n))
    calls = driver.getCallsRdd(driver.getData)
    keep = driver.variantQc(calls)
    rows = plink.BedFile(prefix).rows(0, v)
    c = qc_ref.counts(rows, n)
    want, by = variant_qc_keep(c, qc_ref.hwe_p_many(c), 0.05, 0.05, 1e-6)
    np.testing.assert_array_equal(keep, want)
    assert not keep[[5, 11, 17, 23]].any() and by[11] == 1 and by[17] == 2 and by[5] == 3 and by[23] == 3
    g, h, f = (int((by == k).sum()) for k in (1, 2, 3))
    assert (f"Variant QC: {int(want.sum())} of {v} variants kept ({g} by --geno 0.05, {h} by --hwe 1e-06, "
            f"{f} by --maf 0.05 removed).") in capsys.readouterr().out
    for ext in (".afreq", ".vmiss", ".hardy"):
        assert len(open(str(tmp_path / "out") + ext).read().splitlines()) == v + 1
    parts = [p for p in calls.partitions if isinstance(p, BedSlice)]
    assert np.array_equal(np.concatenate([p.rows() for p in parts]), rows[want])
    assert calls.count() == int(want.sum())


def test_driver_message_names_only_the_flags_given(tmp_path, monkeypatch, capsys):
    prefix, d = _qc_fileset(tmp_path)
    driver = VariantsPcaDriver(PcaConf(["--bed-path", prefix, "--hwe", "0.001"]))
    monkeypatch.setattr(VariantsPcaDriver, "_native", lambda self, n: QcDouble(n))
    keep = driver.variantQc(driver.getCallsRdd(driver.getData))
    out = capsys.readouterr().out
    assert f"Variant QC: {int(keep.sum())} of {d.shape[1]} variants kept (" in out
    assert "by --hwe 0.001 removed)." in out and "--maf" not in out and "--geno" not in out
    assert not (tmp_path / "c.afreq").exists()


def test_qc_then_ld_prune_lists_only_passing_variants(tmp_path, monkeypatch, capsys):
    prefix, d = _qc_fileset(tmp_path)
    n, v = d.shape
    out = str(tmp_path / "out")
    conf = PcaConf(["--bed-path", prefix, "--maf", "0.05", "--hwe", "1e-6", "--ld-prune", "0.3", "--ld-window-kb", "2",
                    "--variants-per-partition", "16", "--output-path", out])
    driver = VariantsPcaDriver(conf)
    monkeypatch.setattr(VariantsPcaDriver, "_native", lambda self, n: QcDouble(n))
    calls = driver.getCallsRdd(driver.getData)
    qc = driver.variantQc(calls)
    keep = driver.ldPrune(calls, check_ld_flags(conf, plink.read_bim(prefix)), qc)
    q = int(qc.sum())
    assert 0 < keep.sum() < q < v and np.all(keep <= qc)
    # the same as pruning a fileset of the QC-passing variants
    sub = str(tmp_path / "sub")
    bim = plink.read_bim(prefix)
    plink.write_fileset(sub, d[:, qc], contigs=[b.contig for b, k in zip(bim, qc) if k],
                        positions=[b.position for b, k in zip(bim, qc) if k])
    sub_keep, _, _ = ld_ref.prune(plink.BedFile(sub).rows(0, q), n, plink.window_starts(plink.read_bim(sub), 2), 0.3)
    np.testing.assert_array_equal(keep[qc], sub_keep)
    text = capsys.readouterr().out
    assert f"LD prune r2 > 0.3 within 2 kb: {int(keep.sum())} of {q} variants kept." in text
    ids = [b.id for b in bim]
    assert open(out + ".prune.in").read().split() == [ids[j] for j in np.flatnonzero(keep)]
    assert open(out + ".prune.out").read().split() == [ids[j] for j in np.flatnonzero(qc & ~keep)]
    parts = [p for p in calls.partitions if isinstance(p, BedSlice)]
    assert np.array_equal(np.concatenate([p.rows() for p in parts]), plink.BedFile(prefix).rows(0, v)[keep])


def test_qc_that_keeps_nothing_is_refused(tmp_path, monkeypatch):
    prefix, _ = _fileset(tmp_path, d=np.zeros((8, 6), np.int64)), None
    driver = VariantsPcaDriver(PcaConf(["--bed-path", prefix, "--maf", "0.01"]))
    monkeypatch.setattr(VariantsPcaDriver, "_native", lambda self, n: QcDouble(n))
    with pytest.raises(ValueError, match="keeps none of the 6 variants"):
        driver.variantQc(driver.getCallsRdd(driver.getData))
