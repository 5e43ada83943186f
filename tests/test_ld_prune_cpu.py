"""--ld-prune without a GPU: the numpy restatement of r2 (tests/ld_ref.py) against np.corrcoef, its allele-flip
invariance and zero-variance rule, the two properties that characterise the keep-first set, `plink.window_starts`, every
refusal of the flags (raised before a context exists), the .prune.in / .prune.out writer and the driver's keep masks."""
import itertools

import numpy as np
import pytest

import ld_ref
from spark_examples_b200 import native, plink, variants_pca
from spark_examples_b200.conf import PcaConf
from spark_examples_b200.plink import BimRecord
from spark_examples_b200.variants_common import BedSlice
from spark_examples_b200.variants_pca import VariantsPcaDriver, check_ld_flags, write_prune_lists


def _pack(dosage):
    """(n, v) A1 counts, -1 missing -> (v, ceil(n / 4)) .bed rows, through plink.write_fileset's encoding."""
    d = np.asarray(dosage)
    code = np.full(d.T.shape, 1, np.uint8)
    code[d.T == 2], code[d.T == 1], code[d.T == 0] = 0, 2, 3
    pad = (-d.shape[0]) % 4
    code = np.concatenate([code, np.zeros((code.shape[0], pad), np.uint8)], axis=1)
    c4 = code.reshape(code.shape[0], -1, 4)
    return (c4[:, :, 0] | (c4[:, :, 1] << 2) | (c4[:, :, 2] << 4) | (c4[:, :, 3] << 6)).astype(np.uint8)


def test_decode_round_trip():
    rng = np.random.default_rng(1)
    d = rng.integers(-1, 3, size=(13, 7))
    D, M = ld_ref.decode(_pack(d), 13)
    assert np.array_equal(M, (d.T >= 0).astype(np.int64))
    assert np.array_equal(D, np.where(d.T >= 0, d.T, 0))


def test_r2_matches_corrcoef_on_complete_data():
    rng = np.random.default_rng(2)
    n, v = 300, 40
    base = rng.integers(0, 3, size=(n, 1))
    d = np.where(rng.random((n, v)) < 0.7, base, rng.integers(0, 3, size=(n, v)))   # correlated columns
    r2, ok = ld_ref.r2_matrix(*ld_ref.decode(_pack(d), n))
    want = np.corrcoef(d.T.astype(np.float64)) ** 2
    assert ok.all()
    assert np.max(np.abs(r2 - want)) < 1e-12
    assert np.all(r2 <= 1.0)
    assert np.all(np.diag(r2) == 1.0)                                        # a variant against itself: exactly 1


def test_allele_flip_leaves_r2_bits_unchanged():
    rng = np.random.default_rng(3)
    d = rng.integers(-1, 3, size=(57, 30))
    flipped = np.where(d >= 0, 2 - d, -1)
    r2a, oka = ld_ref.r2_matrix(*ld_ref.decode(_pack(d), 57))
    r2b, okb = ld_ref.r2_matrix(*ld_ref.decode(_pack(flipped), 57))
    assert np.array_equal(oka, okb)
    assert np.array_equal(r2a.view(np.int64), r2b.view(np.int64))


def test_zero_variance_pairs_are_never_in_ld():
    # variant 0 monomorphic; variant 1 varies only on samples where variant 2 is missing; 3 all missing
    d = np.array([[1, 0, -1, -1],
                  [1, 0, -1, -1],
                  [1, 2, 1, -1],
                  [1, 2, 1, -1],
                  [1, 1, 0, -1]]).astype(np.int64)
    d[:2, 1] = [0, 2]
    d[:2, 2] = -1
    d[2:, 1] = 1                                                             # 1 is constant where 2 is called
    D, M = ld_ref.decode(_pack(d), 5)
    r2, ok = ld_ref.r2_matrix(D, M)
    assert not ok[0].any() and not ok[:, 0].any()
    assert not ok[1, 2] and not ok[2, 1]
    assert not ok[3].any() and not ok[:, 3].any()
    pairs, _ = ld_ref.ld_pairs(D, M, np.zeros(4, np.int64), 0.0)
    assert len(pairs) == 0                                                   # R2 = 0 still needs both variances > 0


def test_comparison_is_strict():
    d = np.array([[0, 0, 0], [1, 1, 2], [2, 2, 1], [2, 1, 0]])
    D, M = ld_ref.decode(_pack(d), 4)
    r2, _ = ld_ref.r2_matrix(D, M)
    lo = np.zeros(3, np.int64)
    pairs, got = ld_ref.ld_pairs(D, M, lo, r2[0, 2])
    assert (0, 2) not in {tuple(p) for p in pairs.tolist()}
    pairs, _ = ld_ref.ld_pairs(D, M, lo, np.nextafter(r2[0, 2], 0))
    assert (0, 2) in {tuple(p) for p in pairs.tolist()}


def _properties_hold(v, lo, pairs, keep):
    """1. no two kept variants of a window in LD; 2. every pruned variant in LD with an earlier kept one of its window."""
    ld = {tuple(p) for p in np.asarray(pairs).reshape(-1, 2).tolist()}
    for i, j in ld:
        assert lo[j] <= i < j
    one = all(not (keep[i] and keep[j]) for i, j in ld)
    two = all(keep[j] or any(keep[i] and (i, j) in ld for i in range(lo[j], j)) for j in range(v))
    return one and two


def _random_graph(rng, v):
    lo = np.maximum.accumulate(np.array([max(0, j - int(rng.integers(0, 5))) for j in range(v)], np.int64))
    lo = np.minimum(lo, np.arange(v))
    pairs = [(i, j) for j in range(v) for i in range(lo[j], j) if rng.random() < 0.4]
    return lo, np.asarray(pairs, np.int64).reshape(-1, 2)


def test_keep_first_is_the_only_set_with_both_properties():
    rng = np.random.default_rng(4)
    for _ in range(60):
        v = int(rng.integers(1, 11))
        lo, pairs = _random_graph(rng, v)
        keep = ld_ref.sweep(v, pairs)
        assert _properties_hold(v, lo, pairs, keep)
        others = [np.array(bits, bool) for bits in itertools.product([False, True], repeat=v)
                  if _properties_hold(v, lo, pairs, np.array(bits, bool))]
        assert len(others) == 1 and np.array_equal(others[0], keep)


def test_keep_first_on_larger_random_graphs():
    rng = np.random.default_rng(5)
    for _ in range(20):
        v = int(rng.integers(50, 300))
        lo, pairs = _random_graph(rng, v)
        keep = ld_ref.sweep(v, pairs)
        assert keep[0] if v else True
        assert _properties_hold(v, lo, pairs, keep)


def _bim(contigs, positions):
    return [BimRecord(c, f"rs{j + 1}", int(p), "A", "G") for j, (c, p) in enumerate(zip(contigs, positions))]


def test_window_starts_with_contigs_and_ties():
    contigs = ["1"] * 6 + ["2"] * 4 + ["X"] * 3
    positions = [100, 100, 600, 1100, 1101, 5000, 50, 50, 50, 550, 7, 8, 2000000]
    lo = plink.window_starts(_bim(contigs, positions), 0.5)
    assert lo.dtype == np.int64
    assert lo.tolist() == [0, 0, 0, 2, 3, 5, 6, 6, 6, 6, 10, 10, 12]
    assert np.array_equal(lo, ld_ref.window_starts(contigs, positions, 0.5))
    rng = np.random.default_rng(6)
    for kb in (0.001, 0.2, 1.0, 3.5, 1000.0):
        contigs = sorted(rng.choice(["1", "2", "3"], size=200).tolist())
        positions = np.concatenate([np.sort(rng.integers(1, 5000, size=contigs.count(c))) for c in ("1", "2", "3")])
        assert np.array_equal(plink.window_starts(_bim(contigs, positions), kb),
                              ld_ref.window_starts(contigs, positions, kb))


def test_window_starts_refuses_unsorted():
    with pytest.raises(ValueError, match=r"rs3, 1:90"):
        plink.window_starts(_bim(["1", "1", "1"], [100, 200, 90]), 500)
    with pytest.raises(ValueError, match=r"contig 1 comes back at variant 2"):
        plink.window_starts(_bim(["1", "2", "1"], [100, 200, 300]), 500)
    assert plink.window_starts([], 500).tolist() == []


def test_write_fileset_defaults_are_unchanged(tmp_path):
    d = np.array([[0, 1, 2], [-1, 2, 0]])
    plink.write_fileset(str(tmp_path / "a"), d)
    assert (tmp_path / "a.bim").read_text() == "".join(f"17\trs{j + 1}\t0\t{41196311 + j}\tA\tG\n" for j in range(3))
    plink.write_fileset(str(tmp_path / "b"), d, contigs=["17"] * 3, positions=[41196311 + j for j in range(3)])
    for ext in (".bed", ".bim", ".fam"):
        assert (tmp_path / ("a" + ext)).read_bytes() == (tmp_path / ("b" + ext)).read_bytes()
    plink.write_fileset(str(tmp_path / "c"), d, contigs=["1", "1", "2"], positions=[5, 9, 5])
    bim = plink.read_bim(str(tmp_path / "c"))
    assert [(b.contig, b.position) for b in bim] == [("1", 5), ("1", 9), ("2", 5)]


@pytest.fixture
def no_context(monkeypatch):
    """Any attempt to create a context fails the test: the refusals must come first."""
    def _native(self, n):
        raise AssertionError("a native context was requested")
    monkeypatch.setattr(VariantsPcaDriver, "_native", _native)


def _fileset(tmp_path, positions=None, contigs=None, n=12):
    rng = np.random.default_rng(0)
    v = 40 if positions is None else len(positions)
    prefix = str(tmp_path / "c")
    plink.write_fileset(prefix, rng.integers(0, 3, size=(n, v)), fam=[(f"F{i}", f"I{i}") for i in range(n)],
                        contigs=contigs, positions=positions)
    return prefix


@pytest.mark.parametrize("argv, match", [
    (["--synthetic", "20,100", "--ld-prune", "0.2"], "--bed-path"),
    (["--synthetic", "20,100", "--ld-window-kb", "100"], "needs --ld-prune"),
    (["BED", "--ld-window-kb", "100"], "needs --ld-prune"),
    (["BED", "--ld-prune", "0.2", "--checkpoint-path", "ck"], "checkpoint"),
    (["BED", "--ld-prune", "0.2", "--project-loadings", "l.npz"], "project-loadings"),
    (["BED", "--ld-prune", "1.0"], r"\[0, 1\)"),
    (["BED", "--ld-prune=-0.1"], r"\[0, 1\)"),
    (["BED", "--ld-prune", "nan"], r"\[0, 1\)"),
    (["BED", "--ld-prune", "0.2", "--ld-window-kb", "0"], "positive"),
    (["BED", "--ld-prune", "0.2", "--ld-window-kb=-5"], "positive"),
    (["BED", "--ld-prune", "0.2", "--ld-window-kb", "inf"], "positive"),
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
        variants_pca.main(["--bed-path", _fileset(tmp_path), "--ld-prune", "0.2"])


def test_unsorted_bim_refused(tmp_path, no_context):
    prefix = _fileset(tmp_path, positions=[10, 20, 15, 30], contigs=["1"] * 4)
    with pytest.raises(ValueError, match=r"sorted .*rs3, 1:15"):
        variants_pca.main(["--bed-path", prefix, "--ld-prune", "0.2"])
    prefix = _fileset(tmp_path, positions=[10, 20, 30, 40], contigs=["1", "2", "2", "1"])
    with pytest.raises(ValueError, match="contig 1 comes back"):
        variants_pca.main(["--bed-path", prefix, "--ld-prune", "0.2"])


def test_window_wider_than_the_limit_refused(tmp_path, no_context):
    w = native.LD_MAX_WINDOW
    positions = list(range(1, w + 3))                                         # one bp apart: H = w + 1 at variant w + 1
    prefix = _fileset(tmp_path, positions=positions, contigs=["3"] * len(positions), n=4)
    with pytest.raises(ValueError, match=rf"variant {w + 1} \(rs{w + 2}, 3:{w + 2}\) holds {w + 1} earlier"):
        variants_pca.main(["--bed-path", prefix, "--ld-prune", "0.2", "--ld-window-kb", "100"])
    conf = PcaConf(["--bed-path", prefix, "--ld-prune", "0.2", "--ld-window-kb", "100"])
    lo = check_ld_flags(conf, plink.read_bim(prefix)[: w + 1])               # H = w itself is accepted
    assert int(np.max(np.arange(w + 1) - lo)) == w


def test_flags_parse():
    conf = PcaConf(["--bed-path", "c", "--ld-prune", "0.2"])
    assert conf.ldPrune() == 0.2 and conf.ldWindowKb() == 500.0 and not conf.ldWindowKb.isSupplied
    assert check_ld_flags(conf) is None
    assert check_ld_flags(PcaConf([])) is None


def test_prune_lists(tmp_path):
    bim = _bim(["1"] * 5, [1, 2, 3, 4, 5])
    write_prune_lists(str(tmp_path / "p"), bim, np.array([1, 0, 0, 1, 1], bool))
    assert (tmp_path / "p.prune.in").read_text() == "rs1\nrs4\nrs5\n"
    assert (tmp_path / "p.prune.out").read_text() == "rs2\nrs3\n"
    write_prune_lists(str(tmp_path / "q"), bim, np.ones(5, bool))
    assert (tmp_path / "q.prune.out").read_text() == ""


class LdDouble:
    """vpca_ld_prune_bed computed with the numpy restatement."""

    def __init__(self, n):
        self.n = n

    def ldPruneBed(self, rows, window_lo, r2_max, max_pairs=0):
        keep, pairs, r2 = ld_ref.prune(np.asarray(rows), self.n, window_lo, r2_max)
        return keep, pairs[:max_pairs], r2[:max_pairs]


def test_driver_masks_slices_and_writes_lists(tmp_path, monkeypatch, capsys):
    rng = np.random.default_rng(9)
    n, v = 30, 50
    base = rng.integers(0, 3, size=(n, 1))
    d = np.where(rng.random((n, v)) < 0.6, base, rng.integers(0, 3, size=(n, v)))
    positions = np.arange(v) * 300 + 1
    prefix = str(tmp_path / "c")
    plink.write_fileset(prefix, d, contigs=["1"] * 25 + ["2"] * 25, positions=positions)
    argv = ["--bed-path", prefix, "--ld-prune", "0.3", "--ld-window-kb", "2", "--variants-per-partition", "16",
            "--output-path", str(tmp_path / "out")]
    conf = PcaConf(argv)
    driver = VariantsPcaDriver(conf)
    monkeypatch.setattr(VariantsPcaDriver, "_native", lambda self, n: LdDouble(n))
    calls = driver.getCallsRdd(driver.getData)
    lo = check_ld_flags(conf, plink.read_bim(prefix))
    keep = driver.ldPrune(calls, lo)
    want, _, _ = ld_ref.prune(plink.BedFile(prefix).rows(0, v), n, lo, 0.3)
    assert np.array_equal(keep, want) and 0 < keep.sum() < v
    assert f"LD prune r2 > 0.3 within 2 kb: {int(want.sum())} of {v} variants kept." in capsys.readouterr().out
    kept_ids = [f"rs{j + 1}" for j in np.flatnonzero(want)]
    assert (tmp_path / "out.prune.in").read_text().split() == kept_ids
    assert len((tmp_path / "out.prune.out").read_text().split()) == v - len(kept_ids)
    parts = [p for p in calls.partitions if isinstance(p, BedSlice)]
    assert np.array_equal(np.concatenate([p.rows() for p in parts]), plink.BedFile(prefix).rows(0, v)[want])
    assert calls.count() == int(want.sum())
    keys = np.concatenate([driver._partition_keys(p, 0) for p in parts])
    full = BedSlice(parts[0].bed, 0, v, parts[0].counted)
    assert np.array_equal(keys, driver._partition_keys(full, 0)[want])
