"""KING-robust kinship without a GPU: the numpy restatement (tests/kinship_ref.py) on hand-derived cases, the
--make-king-table / --king-table-filter flags, every driver refusal (raised before a context exists), and the table
writer on given arrays with a test double for the native class."""
import numpy as np
import pytest

from kinship_ref import HET, HOM_A1, HOM_A2, MISSING, bed_codes, count_matrices, king_pairs, pack_codes, pair_counts
from spark_examples_b200 import native, plink, variants_pca
from spark_examples_b200.conf import PcaConf
from spark_examples_b200.variants_pca import VariantsPcaDriver


def _codes(*columns):
    return np.stack([np.asarray(c, np.uint8) for c in columns], axis=1)    # (nv, n)


def test_identical_genotypes_give_one_half():
    g = [HET, HOM_A1, HOM_A2, HET, HOM_A1, MISSING]
    ids, counts, kin = king_pairs(_codes(g, g))
    assert ids.tolist() == [[0, 1]] and kin[0] == 0.5
    assert counts.tolist() == [[5, 2, 0, 0, 0]]                     # NSNP, HETHET, IBS0, HET1_HOM2, HET2_HOM1


def test_hand_counts_give_minus_one_third():
    """HETHET = 1, IBS0 = 1, HET1_HOM2 = 1: (1 - 2) / (2 + 1 + 0)."""
    a = [HET, HOM_A1, HET, MISSING]
    b = [HET, HOM_A2, HOM_A1, HET]
    ids, counts, kin = king_pairs(_codes(a, b))
    assert counts.tolist() == [[3, 1, 1, 1, 0]]
    assert kin[0] == -1.0 / 3.0
    assert pair_counts(_codes(a, b), 0, 1) == (3, 1, 1, 1, 0)


def test_no_heterozygote_gives_nan():
    ids, counts, kin = king_pairs(_codes([HOM_A1, HOM_A2, HOM_A1], [HOM_A2, HOM_A2, MISSING]))
    assert counts.tolist() == [[2, 0, 1, 0, 0]] and np.isnan(kin[0])
    assert len(king_pairs(_codes([HOM_A1], [HOM_A2]), -1e300)[0]) == 0     # NaN never passes a finite threshold


def test_order_and_pack_round_trip():
    rng = np.random.default_rng(1)
    codes = rng.integers(0, 4, size=(50, 7)).astype(np.uint8)
    np.testing.assert_array_equal(bed_codes(pack_codes(codes), 7), codes)
    ids, counts, _ = king_pairs(codes)
    assert ids.tolist() == [[a, b] for b in range(7) for a in range(b)]
    nsnp, hethet, ibs0, h1 = count_matrices(codes)
    for (a, b), c in zip(ids.tolist(), counts.tolist()):
        assert tuple(c) == pair_counts(codes, a, b) == (nsnp[a, b], hethet[a, b], ibs0[a, b], h1[a, b], h1[b, a])


def test_flags_parse():
    conf = PcaConf(["--bed-path", "c", "--make-king-table", "c.kin0", "--king-table-filter", "0.0442"])
    assert conf.makeKingTable() == "c.kin0" and conf.kingTableFilter() == 0.0442
    conf = PcaConf(["--bed-path", "c", "--make-king-table", "c.kin0", "--king-table-filter=-inf"])
    assert np.isneginf(conf.kingTableFilter())
    conf = PcaConf([])
    assert not conf.makeKingTable.isDefined and not conf.kingTableFilter.isDefined


@pytest.fixture
def no_context(monkeypatch):
    """Any attempt to create a context fails the test: the refusals must come first."""
    def _native(self, n):
        raise AssertionError("a native context was requested")
    monkeypatch.setattr(VariantsPcaDriver, "_native", _native)


def _fileset(tmp_path, n=12, nv=40):
    rng = np.random.default_rng(0)
    prefix = str(tmp_path / "c")
    plink.write_fileset(prefix, rng.integers(0, 3, size=(n, nv)), fam=[(f"F{i}", f"I{i}") for i in range(n)])
    return prefix


@pytest.mark.parametrize("argv, match", [
    (["--synthetic", "20,100", "--make-king-table", "x"], "--bed-path"),
    (["--synthetic", "20,100", "--king-table-filter", "0.1"], "needs --make-king-table"),
    (["BED", "--king-table-filter", "0.1"], "needs --make-king-table"),
    (["BED", "--make-king-table", "x", "--checkpoint-path", "ck"], "checkpoint"),
    (["BED", "--make-king-table", "x", "--project-loadings", "l.npz"], "project-loadings"),
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
        variants_pca.main(["--bed-path", _fileset(tmp_path), "--make-king-table", str(tmp_path / "k")])


def test_too_many_samples_refused(tmp_path, no_context):
    n = native.KINSHIP_MAX_SAMPLES + 1
    prefix = str(tmp_path / "big")
    plink.write_fileset(prefix, np.zeros((n, 1), np.int64))
    with pytest.raises(ValueError, match=str(native.KINSHIP_MAX_SAMPLES)):
        variants_pca.main(["--bed-path", prefix, "--make-king-table", str(tmp_path / "k")])


def test_sample_limit_itself_is_accepted(tmp_path):
    conf = PcaConf(["--bed-path", "x", "--make-king-table", "k"])
    variants_pca.check_king_flags(conf, native.KINSHIP_MAX_SAMPLES)


class KinshipDouble:
    """The kinship calls of native.NativePca, computed with the numpy restatement."""

    def __init__(self, n):
        self.n, self.rows = n, []

    def kinshipBed(self, rows):
        self.rows.append(np.array(rows, np.uint8))

    def kinshipPairs(self, min_kinship=float("-inf")):
        return king_pairs(bed_codes(np.concatenate(self.rows), self.n), min_kinship)


def test_table_writer_on_given_arrays(tmp_path):
    fam = [("famA", "a1"), ("famA", "a2"), ("famB", "b1")]
    ids = np.array([[0, 1], [0, 2], [1, 2]], np.int32)
    counts = np.array([[10, 4, 0, 2, 1, ], [9, 1, 3, 0, 2], [0, 0, 0, 0, 0]], np.int32)
    kin = np.array([0.1 + 0.2, -1.0 / 3.0, np.nan])
    path = tmp_path / "t.kin0"
    variants_pca.write_king_table(str(path), fam, ids, counts, kin, batch=2)
    lines = path.read_text().splitlines()
    assert lines == ["#FID1\tIID1\tFID2\tIID2\tNSNP\tHETHET\tIBS0\tKINSHIP",
                     "famA\ta1\tfamA\ta2\t10\t4\t0\t0.30000000000000004",
                     "famA\ta1\tfamB\tb1\t9\t1\t3\t-0.3333333333333333",
                     "famA\ta2\tfamB\tb1\t0\t0\t0\tnan"]
    assert float(lines[1].split("\t")[7]) == kin[0] and float(lines[2].split("\t")[7]) == kin[1]


def test_driver_table_through_a_test_double(tmp_path):
    rng = np.random.default_rng(4)
    n, nv = 9, 300
    d = rng.integers(0, 3, size=(n, nv))
    d[:, 7] = -1
    d[5] = d[2]
    fam = [(f"F{i % 2}", f"S{i}") for i in range(n)]
    prefix = str(tmp_path / "c")
    plink.write_fileset(prefix, d, fam=fam)
    conf = PcaConf(["--bed-path", prefix, "--make-king-table", str(tmp_path / "k.kin0"), "--king-table-filter", "0.3"])
    drv = VariantsPcaDriver(conf)
    drv._nat = KinshipDouble(n)
    bed = plink.BedFile(prefix)
    drv._nat.kinshipBed(bed.rows(0, nv))
    drv.writeKingTable()
    lines = (tmp_path / "k.kin0").read_text().splitlines()
    assert lines[0].startswith("#FID1") and lines[1:] == ["F0\tS2\tF1\tS5\t299\t" + lines[1].split("\t")[5] + "\t0\t0.5"]
