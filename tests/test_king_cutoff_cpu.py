"""--king-cutoff without a GPU: the selection rule (independent, maximal, deterministic) on hand-built relationship graphs,
the strict `> X` at a pair exactly on the cutoff, the PLINK 2 id files, and every refusal of the flag (raised before a
context exists, or right after the selection)."""
import itertools

import numpy as np
import pytest

from spark_examples_b200 import native, plink, variants_pca
from spark_examples_b200.conf import PcaConf
from spark_examples_b200.variants_pca import VariantsPcaDriver, king_cutoff_keep


def _keep(n, pairs, kin=None, cutoff=0.1):
    ids = np.asarray(pairs, np.int32).reshape(-1, 2)
    kin = np.full(len(ids), 0.25) if kin is None else np.asarray(kin, np.float64)
    return king_cutoff_keep(n, ids, kin, cutoff)


def _check_maximal_independent(n, pairs, keep):
    related = {frozenset(p) for p in pairs if p[0] != p[1]}
    for a, b in related:
        assert not (keep[a] and keep[b]), (a, b)                         # independent
    for r in np.flatnonzero(~keep):
        assert any(keep[j] for p in related if r in p for j in p if j != r), r   # maximal: every removed one has a reason


@pytest.mark.parametrize("n, pairs, kept", [
    (0, [], []),
    (5, [], [0, 1, 2, 3, 4]),                                            # nobody related
    (4, [(0, 1), (1, 2), (2, 3)], [0, 3]),                               # chain: ties go to the larger index
    (4, [(a, b) for a, b in itertools.combinations(range(4), 2)], [0]),   # clique
    (6, [(0, j) for j in range(1, 6)], [1, 2, 3, 4, 5]),                 # star: the hub goes
    (3, [(0, 2)], [0, 1]),                                               # duplicate pair: the larger index goes
    (3, [(0, 2), (1, 2)], [0, 1]),                                       # trio: the child (2) goes, both parents stay
    (4, [(0, 1), (2, 3)], [0, 2]),                                       # two tied pairs
])
def test_selection_cases(n, pairs, kept):
    keep = _keep(n, pairs)
    assert keep.dtype == bool and keep.shape == (n,)
    assert np.flatnonzero(keep).tolist() == kept
    _check_maximal_independent(n, pairs, keep)


def test_put_back_pass_restores_a_sample_whose_relatives_all_left():
    """Sample 20 and its partners 0..3 all have 4 related partners; 20 goes first (the larger index), then 3, 2, 1, 0 for
    their 3 private relatives each, which leaves 20 without a relative in the set: it returns."""
    pairs = [(j, 20) for j in range(4)] + [(j, 4 + 3 * j + i) for j in range(4) for i in range(3)]
    keep = _keep(21, pairs)
    _check_maximal_independent(21, pairs, keep)
    assert keep[20] and not keep[:4].any() and keep[4:].all()


def test_random_graphs_are_independent_maximal_and_deterministic():
    rng = np.random.default_rng(8)
    for trial in range(40):
        n = int(rng.integers(2, 60))
        m = int(rng.integers(0, 3 * n))
        pairs = [tuple(sorted(rng.choice(n, 2, replace=False).tolist())) for _ in range(m)]
        kin = rng.uniform(-0.2, 0.5, size=len(pairs))
        keep = _keep(n, pairs, kin, 0.0884)
        related = [p for p, k in zip(pairs, kin) if k > 0.0884]
        _check_maximal_independent(n, related, keep)
        perm = rng.permutation(len(pairs))                               # the pair order does not matter
        np.testing.assert_array_equal(_keep(n, [pairs[i] for i in perm], kin[perm], 0.0884), keep)


def test_strictly_greater_than_the_cutoff_and_nan_never_related():
    x = 0.0884
    assert _keep(2, [(0, 1)], [x], x).all()                             # exactly on the cutoff: not related
    assert not _keep(2, [(0, 1)], [np.nextafter(x, np.inf)], x).all()
    assert _keep(2, [(0, 1)], [np.nan], x).all()
    assert _keep(2, [(0, 1)], [np.nan], -np.inf).all()


def test_id_files(tmp_path):
    fam = [("fa", "a"), ("fa", "b"), ("fb", "c"), ("fc", "d")]
    prefix = str(tmp_path / "out")
    variants_pca.write_king_cutoff_ids(prefix, fam, np.array([True, False, True, False]))
    assert (tmp_path / "out.king.cutoff.in.id").read_text() == "#FID\tIID\nfa\ta\nfb\tc\n"
    assert (tmp_path / "out.king.cutoff.out.id").read_text() == "#FID\tIID\nfa\tb\nfc\td\n"
    variants_pca.write_king_cutoff_ids(prefix, fam, np.ones(4, bool))
    assert (tmp_path / "out.king.cutoff.out.id").read_text() == "#FID\tIID\n"


def test_flag_parses():
    assert PcaConf(["--bed-path", "c", "--king-cutoff", "0.0884"]).kingCutoff() == 0.0884
    assert not PcaConf([]).kingCutoff.isDefined


@pytest.fixture
def no_context(monkeypatch):
    def _native(self, n):
        raise AssertionError("a native context was requested")
    monkeypatch.setattr(VariantsPcaDriver, "_native", _native)


def _fileset(tmp_path, n=12, nv=40):
    rng = np.random.default_rng(0)
    prefix = str(tmp_path / "c")
    plink.write_fileset(prefix, rng.integers(0, 3, size=(n, nv)), fam=[(f"F{i}", f"I{i}") for i in range(n)])
    return prefix


@pytest.mark.parametrize("argv, match", [
    (["--synthetic", "20,100", "--king-cutoff", "0.1"], "--bed-path"),
    (["BED", "--king-cutoff", "0.1", "--checkpoint-path", "ck"], "checkpoint"),
    (["BED", "--king-cutoff", "0.1", "--project-loadings", "l.npz"], "project-loadings"),
    (["BED", "--king-cutoff", "nan"], "finite"),
    (["BED", "--king-cutoff", "inf"], "finite"),
    (["BED", "--king-cutoff=-inf"], "finite"),
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
        variants_pca.main(["--bed-path", _fileset(tmp_path), "--king-cutoff", "0.1"])


def test_too_many_samples_refused(tmp_path, no_context):
    n = native.KINSHIP_MAX_SAMPLES + 1
    prefix = str(tmp_path / "big")
    plink.write_fileset(prefix, np.zeros((n, 1), np.int64))
    with pytest.raises(ValueError, match=str(native.KINSHIP_MAX_SAMPLES)):
        variants_pca.main(["--bed-path", prefix, "--king-cutoff", "0.1"])


@pytest.mark.parametrize("kept, num_pc, ok", [(1, 2, False), (2, 2, True), (4, 5, False), (5, 5, True), (0, 2, False)])
def test_too_few_kept_refused(kept, num_pc, ok):
    if ok:
        variants_pca.check_king_cutoff_kept(kept, num_pc)
    else:
        with pytest.raises(ValueError, match="--king-cutoff keeps"):
            variants_pca.check_king_cutoff_kept(kept, num_pc)


class SubsetDouble:
    """The kinship and PCA calls of native.NativePca the cutoff path makes, as a test double: every pair related, so only
    one sample would stay."""

    def __init__(self, n):
        self.n = n

    def kinshipPairs(self, min_kinship=float("-inf")):
        a, b = np.tril_indices(self.n, -1)
        return np.stack([b, a], axis=1).astype(np.int32), np.zeros((len(a), 5), np.int32), np.full(len(a), 0.5)

    def computePcaSubset(self, keep, k):
        raise AssertionError("the selection must be refused before the solve")


def test_driver_refuses_a_selection_of_one_sample(tmp_path):
    prefix = _fileset(tmp_path, n=6)
    conf = PcaConf(["--bed-path", prefix, "--king-cutoff", "0.1", "--output-path", str(tmp_path / "o")])
    drv = VariantsPcaDriver(conf)
    with pytest.raises(ValueError, match="keeps 1 samples"):
        drv._computePcaUnrelated(SubsetDouble(6), 6, 2)
    assert not (tmp_path / "o.king.cutoff.in.id").exists()
