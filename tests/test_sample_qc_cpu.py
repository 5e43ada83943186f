"""--keep / --remove / --mind without a GPU: the ID-file reader and matcher, `sample_qc_keep` and its attribution order,
every refusal of the flags (raised before a context exists, or before any Gram, kinship, variant-QC or LD work), the
.smiss / .mindrem.id reports read back, and the driver on a numpy double of the two library calls."""
import numpy as np
import pytest

import qc_ref
import sample_qc_ref
from spark_examples_b200 import native, plink, variants_pca
from spark_examples_b200.conf import PcaConf
from spark_examples_b200.variants_common import BedSlice
from spark_examples_b200.variants_pca import (VariantsPcaDriver, check_sample_flags, sample_qc_keep,
                                              write_king_cutoff_ids, write_sample_qc_reports)


def _write(path, text):
    path.write_text(text, encoding="utf-8")
    return str(path)


FAM = [("F1", "A"), ("F1", "B"), ("F2", "A"), ("F2", "C"), ("F3", "D")]


def test_id_file_parsing(tmp_path):
    p = _write(tmp_path / "ids", "#FID IID extra\n\nF1 A\n   \nC\nF3\tD\tjunk more\n\n")
    assert plink.read_id_file(p) == [("F1", "A"), (None, "C"), ("F3", "D")]
    # without a header the first line is an ID; a later '#' line is just an ID that matches nothing
    p = _write(tmp_path / "ids2", "F2 C\n#F9 Z\n")
    assert plink.read_id_file(p) == [("F2", "C"), ("#F9", "Z")]
    assert plink.read_id_file(_write(tmp_path / "empty", "")) == []
    assert plink.read_id_file(_write(tmp_path / "head", "#FID\tIID\n")) == []


def test_id_matching(tmp_path):
    listed, unmatched = plink.match_sample_ids(FAM, [("F1", "A"), (None, "C"), ("F3", "D"), ("F9", "A"), (None, "Q")])
    np.testing.assert_array_equal(listed, [1, 0, 0, 1, 1])
    assert unmatched == 2
    # file order does not matter, repeats are harmless
    again, u2 = plink.match_sample_ids(FAM, [("F3", "D"), (None, "C"), ("F1", "A"), ("F1", "A")])
    np.testing.assert_array_equal(again, listed)
    assert u2 == 0
    # a bare IID held by two families is refused; with its FID it is fine
    with pytest.raises(ValueError, match="bare IID A is ambiguous: it occurs in families F1, F2"):
        plink.match_sample_ids(FAM, [(None, "A")], "ids")
    listed, _ = plink.match_sample_ids(FAM, [("F2", "A")])
    np.testing.assert_array_equal(listed, [0, 0, 1, 0, 0])


def test_project_id_lists_read_back(tmp_path):
    keep = np.array([1, 0, 1, 1, 0], bool)
    write_king_cutoff_ids(str(tmp_path / "k"), FAM, keep)
    for suffix, want in ((".king.cutoff.in.id", keep), (".king.cutoff.out.id", ~keep)):
        listed, unmatched = plink.match_sample_ids(FAM, plink.read_id_file(str(tmp_path / "k") + suffix))
        np.testing.assert_array_equal(listed, want)
        assert unmatched == 0


def test_keep_and_attribution_order():
    n = 8
    lk = np.array([1, 1, 1, 1, 1, 1, 0, 0], bool)
    lr = np.array([0, 1, 0, 0, 0, 0, 1, 0], bool)
    miss = np.array([0, 9, 1, 2, 3, 10, 10, 0])
    keep, by = sample_qc_keep(n, lk, lr, miss, 10, 0.2)
    np.testing.assert_array_equal(by, [0, 2, 0, 0, 3, 3, 1, 1])      # keep first, then remove, then mind
    np.testing.assert_array_equal(keep, by == 0)
    _, by = sample_qc_keep(n, None, lr, miss, 10, 0.2)
    np.testing.assert_array_equal(by, [0, 2, 0, 0, 3, 3, 2, 0])
    _, by = sample_qc_keep(n, None, None, miss, 10, 0.2)              # F_MISS = 0.2 is not > 0.2
    np.testing.assert_array_equal(by, [0, 3, 0, 0, 3, 3, 3, 0])
    _, by = sample_qc_keep(n, None, None, miss, 10, 0.0)              # --mind 0: any missing call
    np.testing.assert_array_equal(by, [0, 3, 3, 3, 3, 3, 3, 0])
    keep, _ = sample_qc_keep(n, None, None, miss, 10, 1.0)            # --mind 1: nothing, even all missing
    assert keep.all()
    keep, _ = sample_qc_keep(n, None, None, np.zeros(n), 0, 0.0)      # no variants: F_MISS is NaN, nothing removed
    assert keep.all()
    keep, by = sample_qc_keep(n, lk)
    np.testing.assert_array_equal(by, [0, 0, 0, 0, 0, 0, 1, 1])


def test_mind_uses_one_rounded_division():
    # 1 / 3 rounds below 0.33333333333333337 and above 0.3333333333333333 - 1 ulp
    third = 1.0 / 3.0
    keep, _ = sample_qc_keep(2, missing=np.array([1, 0]), n_variants=3, mind=third)
    assert keep.all()
    keep, _ = sample_qc_keep(2, missing=np.array([1, 0]), n_variants=3, mind=np.nextafter(third, 0))
    np.testing.assert_array_equal(keep, [0, 1])


def test_reports_read_back(tmp_path):
    left = np.array([1, 1, 0, 1, 1], bool)
    miss = np.array([0, 3, 5, 7, 1])
    mind_removed = np.array([0, 0, 0, 1, 0], bool)
    write_sample_qc_reports(str(tmp_path / "q"), FAM, left, miss, 7, mind_removed)
    lines = (tmp_path / "q.smiss").read_text().splitlines()
    assert lines[0] == "#FID\tIID\tMISSING_CT\tOBS_CT\tF_MISS"
    rows = [ln.split("\t") for ln in lines[1:]]
    assert [tuple(r[:2]) for r in rows] == [FAM[s] for s in (0, 1, 3, 4)]
    assert [(int(r[2]), int(r[3]), float(r[4])) for r in rows] == [(0, 7, 0.0), (3, 7, 3 / 7), (7, 7, 1.0), (1, 7, 1 / 7)]
    assert (tmp_path / "q.mindrem.id").read_text() == "#FID\tIID\nF2\tC\n"
    write_sample_qc_reports(str(tmp_path / "e"), FAM, left, miss, 7, np.zeros(5, bool))
    assert (tmp_path / "e.mindrem.id").read_text() == "#FID\tIID\n"            # written even when empty
    listed, _ = plink.match_sample_ids(FAM, plink.read_id_file(str(tmp_path / "q.mindrem.id")))
    np.testing.assert_array_equal(listed, mind_removed)


def test_reference_pack_and_counts():
    rng = np.random.default_rng(2)
    d = rng.integers(-1, 3, size=(13, 9))
    rows = sample_qc_ref._pack(np.where(d.T == -1, 1, np.where(d.T == 2, 0, np.where(d.T == 1, 2, 3))))
    np.testing.assert_array_equal(sample_qc_ref.missing_counts(rows, 13), (d == -1).sum(1))
    keep = [0, 3, 4, 12]
    sub = sample_qc_ref.subset_rows(rows, 13, keep)
    np.testing.assert_array_equal(sample_qc_ref.missing_counts(sub, 4), (d[keep] == -1).sum(1))
    assert sub.shape == (9, 1)


# ---- the driver ----------------------------------------------------------------------------------------------------
@pytest.fixture
def no_context(monkeypatch):
    """Any attempt to create a context fails the test: the refusals must come first."""
    def refuse(self, *a):
        raise AssertionError("a native context was requested")
    monkeypatch.setattr(VariantsPcaDriver, "_native", refuse)
    monkeypatch.setattr(VariantsPcaDriver, "_sampleQcNative", refuse)


class SampleDouble:
    """vpca_sample_missing_bed / vpca_subset_bed_samples computed with tests/sample_qc_ref.py."""
    made = 0

    def __init__(self):
        SampleDouble.made += 1
        self.closed = False

    def sampleMissingBed(self, rows, n):
        assert not self.closed
        return sample_qc_ref.missing_counts(np.asarray(rows), n).astype(np.int32)

    def subsetBedSamples(self, rows, n, keep):
        assert not self.closed
        return sample_qc_ref.subset_rows(np.asarray(rows), n, keep)

    def close(self):
        self.closed = True


class QcDouble:
    """vpca_variant_qc_bed and vpca_kinship_pairs on the host."""

    def __init__(self, n):
        self.n = n

    def variantQcBed(self, rows, hwe=True):
        c = qc_ref.counts(np.asarray(rows), self.n)
        return c, (qc_ref.hwe_p_many(c) if hwe else None)

    def kinshipPairs(self, min_kinship=float("-inf")):
        ids = np.array([[a, b] for a in range(self.n) for b in range(a + 1, self.n)], np.int64).reshape(-1, 2)
        return ids, np.zeros((len(ids), 5), np.int64), np.zeros(len(ids))


@pytest.fixture
def doubles(monkeypatch):
    SampleDouble.made = 0
    monkeypatch.setattr(VariantsPcaDriver, "_sampleQcNative", lambda self: SampleDouble())
    monkeypatch.setattr(VariantsPcaDriver, "_native", lambda self, n: QcDouble(n))


def _fileset(tmp_path, n=12, v=40, missing=None, fam=None):
    rng = np.random.default_rng(0)
    d = rng.integers(0, 3, size=(n, v))
    if missing is not None:
        for s, k in enumerate(missing):
            d[s, :k] = -1
    prefix = str(tmp_path / "c")
    plink.write_fileset(prefix, d, fam=fam or [(f"F{i % 3}", f"I{i}") for i in range(n)])
    return prefix, d


@pytest.mark.parametrize("argv, match", [
    (["--synthetic", "20,100", "--keep", "KEEP"], "--bed-path"),
    (["--synthetic", "20,100", "--mind", "0.1"], "--bed-path"),
    (["BED", "--remove", "KEEP", "--checkpoint-path", "ck"], "checkpoint"),
    (["BED", "--mind", "0.1", "--checkpoint-path", "ck"], "checkpoint"),
    (["BED", "--keep", "MISSING"], r"--keep .*cannot read the ID file"),
    (["BED", "--remove", "DIR"], r"--remove .*cannot read the ID file"),
    (["BED", "--keep", "AMBIG"], "bare IID I1 is ambiguous"),
    (["BED", "--mind", "1.5"], r"--mind takes a value in \[0, 1\]"),
    (["BED", "--mind=-0.01"], r"--mind takes a value in \[0, 1\]"),
    (["BED", "--mind", "nan"], r"--mind takes a value in \[0, 1\]"),
    (["BED", "--mind", "inf"], r"--mind takes a value in \[0, 1\]"),
    (["BED", "--keep", "ONE"], r"sample QC keeps 1 of 12 samples: at least max\(2, --num-pc = 2\)"),
    (["BED", "--remove", "KEEP", "--num-pc", "11"], r"sample QC keeps 10 of 12 samples: at least max\(2, --num-pc = 11\)"),
])
def test_refused_before_any_context(tmp_path, no_context, argv, match):
    fam = [(f"F{i % 3}", f"I{i}") for i in range(12)]
    fam[4] = ("F9", "I1")                                   # I1 in two families
    prefix, _ = _fileset(tmp_path, fam=fam)
    files = {"KEEP": _write(tmp_path / "keep", "F0 I0\nF1 I7\n"), "MISSING": str(tmp_path / "nope"),
             "DIR": str(tmp_path), "AMBIG": _write(tmp_path / "ambig", "I1\n"), "ONE": _write(tmp_path / "one", "F0 I0\n")}
    argv = [files.get(a, a) for a in argv]
    argv = [a if a != "BED" else "--bed-path" for a in argv]
    if argv[0] == "--bed-path":
        argv.insert(1, prefix)
    with pytest.raises(ValueError, match=match):
        variants_pca.main(argv)


def test_multi_rank_refused(tmp_path, no_context, monkeypatch):
    prefix, _ = _fileset(tmp_path)
    monkeypatch.setenv("WORLD_SIZE", "2")
    with pytest.raises(ValueError, match="WORLD_SIZE"):
        variants_pca.main(["--bed-path", prefix, "--mind", "0.1"])


def test_too_few_after_mind_refused_before_gram(tmp_path, monkeypatch, capsys):
    prefix, _ = _fileset(tmp_path, n=6, v=10, missing=[5, 5, 5, 5, 5, 0])
    monkeypatch.setattr(VariantsPcaDriver, "_sampleQcNative", lambda self: SampleDouble())

    def refuse(self, n):
        raise AssertionError("the run's context was requested")
    monkeypatch.setattr(VariantsPcaDriver, "_native", refuse)
    with pytest.raises(ValueError, match=r"sample QC keeps 1 of 6 samples"):
        variants_pca.main(["--bed-path", prefix, "--mind", "0.4", "--maf", "0.01", "--ld-prune", "0.5"])
    assert "Sample QC: 1 of 6 samples kept (5 by --mind 0.4 removed)." in capsys.readouterr().out


def _big_fam(tmp_path, n):
    prefix = str(tmp_path / "big")
    plink.write_fileset(prefix, np.zeros((n, 2), np.int64), fam=[("F", f"S{i}") for i in range(n)])
    return prefix


def test_kinship_limit_is_checked_on_the_kept_samples(tmp_path, no_context, monkeypatch):
    lim = native.KINSHIP_MAX_SAMPLES
    prefix = _big_fam(tmp_path, lim + 100)
    over = _write(tmp_path / "over", "".join(f"F S{i}\n" for i in range(lim + 1)))
    with pytest.raises(ValueError, match=f"--make-king-table is limited to {lim} samples; the cohort has {lim + 1}"):
        variants_pca.main(["--bed-path", prefix, "--keep", over, "--make-king-table", str(tmp_path / "k.kin0")])
    # exactly at the limit: past the check, on to the subset pass (here the double)
    monkeypatch.setattr(VariantsPcaDriver, "_sampleQcNative", lambda self: SampleDouble())
    at = _write(tmp_path / "at", "".join(f"F S{i}\n" for i in range(lim)))
    driver = VariantsPcaDriver(PcaConf(["--bed-path", prefix, "--keep", at, "--make-king-table", "k.kin0"]))
    assert len(driver.common.indexes) == lim


def test_driver_on_the_kept_samples(tmp_path, doubles, capsys):
    n, v = 12, 40
    prefix, d = _fileset(tmp_path, n=n, v=v, missing=[0, 3, 0, 9, 0, 0, 1, 0, 0, 0, 20, 0])
    fam = plink.read_fam_ids(prefix)
    keep_file = _write(tmp_path / "keep", "#FID IID\n" + "".join(f"{f} {i}\n" for f, i in fam[:10]) + "X Y\n")
    remove_file = _write(tmp_path / "remove", "I2\nF0 I9\n")
    out = str(tmp_path / "out")
    conf = PcaConf(["--bed-path", prefix, "--keep", keep_file, "--remove", remove_file, "--mind", "0.2",
                    "--maf", "0.0", "--output-path", out, "--variants-per-partition", "16",
                    "--make-king-table", out + ".kin0"])
    driver = VariantsPcaDriver(conf)
    text = capsys.readouterr().out
    # keep: 0..9; remove: 2, 9; mind (F_MISS > 0.2, i.e. > 8 of 40): 3 (10 and 11 already gone)
    kept = [0, 1, 4, 5, 6, 7, 8]
    assert f"--keep {keep_file}: 1 IDs match no sample." in text
    assert "--remove" not in text.split("Sample QC")[0]
    assert "Sample QC: 7 of 12 samples kept (2 by --keep, 2 by --remove, 1 by --mind 0.2 removed)." in text
    assert text.index("Sample QC:") < text.index("Matrix size: 7.")
    assert SampleDouble.made == 1                             # one short-lived context for both calls
    assert list(driver.common.indexes) == [f"{fam[k][0]}-{fam[k][1]}" for k in kept]
    calls = driver.getCallsRdd(driver.getData)
    assert calls.n_samples == 7
    rows = np.concatenate([p.rows() for p in calls.partitions if isinstance(p, BedSlice)])
    np.testing.assert_array_equal(rows, sample_qc_ref.subset_rows(plink.BedFile(prefix).rows(0, v), n, kept))
    # the reports: .smiss over the 8 samples left by --keep / --remove, the one --mind removed
    smiss = [ln.split("\t") for ln in open(out + ".smiss").read().splitlines()[1:]]
    assert [r[1] for r in smiss] == [fam[k][1] for k in (0, 1, 3, 4, 5, 6, 7, 8)]
    assert [(int(r[2]), int(r[3])) for r in smiss][:3] == [(0, 40), (3, 40), (9, 40)]
    assert open(out + ".mindrem.id").read() == f"#FID\tIID\n{fam[3][0]}\t{fam[3][1]}\n"
    # variant QC counts only the kept samples
    driver.variantQc(calls)
    vmiss = [ln.split("\t") for ln in open(out + ".vmiss").read().splitlines()[1:]]
    assert len(vmiss) == v and all(int(r[3]) == 7 for r in vmiss)
    # the KING table names the kept samples
    driver._nat = QcDouble(7)
    driver.writeKingTable()
    pairs = [ln.split("\t")[:4] for ln in open(out + ".kin0").read().splitlines()[1:]]
    names = [fam[k] for k in kept]
    assert pairs[0] == [*names[0], *names[1]] and pairs[-1] == [*names[5], *names[6]] and len(pairs) == 21


def test_every_sample_kept_uses_the_fileset(tmp_path, monkeypatch, capsys):
    prefix, _ = _fileset(tmp_path)
    monkeypatch.setattr(VariantsPcaDriver, "_sampleQcNative", lambda self: SampleDouble())
    driver = VariantsPcaDriver(PcaConf(["--bed-path", prefix, "--mind", "1"]))
    assert isinstance(driver.samples.bed, plink.BedFile)
    assert "Sample QC: 12 of 12 samples kept (0 by --mind 1.0 removed)." in capsys.readouterr().out
    keep = _write(tmp_path / "all", "".join(f"F{i % 3} I{i}\n" for i in range(12)))
    driver = VariantsPcaDriver(PcaConf(["--bed-path", prefix, "--keep", keep]))
    assert isinstance(driver.samples.bed, plink.BedFile)
    assert len(driver.common.indexes) == 12


def test_flags_parse():
    conf = PcaConf(["--bed-path", "c", "--keep", "k.txt", "--remove", "r.txt", "--mind", "0.05"])
    assert conf.keep() == "k.txt" and conf.remove() == "r.txt" and conf.mind() == 0.05
    plain = PcaConf([])
    assert not (plain.keep.isDefined or plain.remove.isDefined or plain.mind.isDefined)
    check_sample_flags(plain)
    check_sample_flags(PcaConf(["--bed-path", "c", "--mind", "0"]))
    check_sample_flags(PcaConf(["--bed-path", "c", "--mind", "1"]))
