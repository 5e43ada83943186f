"""The variance-standardized relationship matrix without a GPU (DESIGN.md 13): the z table in Python floats against exact
rationals, hand-worked cohorts of three samples, the orientation and used/skipped rules, the flag refusals, the output
formats read back, and the driver end to end against a numpy-backed double of the four NativePca GRM calls."""
import math

import numpy as np
import pytest

import grm_ref
import qc_ref
from spark_examples_b200 import native, plink, variants_pca
from spark_examples_b200.conf import PcaConf
from spark_examples_b200.variants_pca import VariantsPcaDriver, check_grm_flags

FLIP = np.array([3, 1, 2, 0], np.uint8)   # .bed code with A1 and A2 swapped


def _G(code):
    rows = grm_ref.pack(np.asarray(code, np.uint8))
    return grm_ref.grm(rows, np.asarray(code).shape[1])


def test_three_samples_by_hand():
    # dosages 2, 0, 0: a = 2 of 2n = 6, A1 the minor allele; mu = 2/3, q = 1/3, s = 1 / sqrt(4/9) = 3/2
    G, M, Z = _G([[0, 3, 3]])
    assert M == 1
    assert np.allclose(Z[:, 0], [2.0, -1.0, -1.0], rtol=0, atol=4e-16)
    assert np.allclose(G, [[4, -2, -2], [-2, 1, 1], [-2, 1, 1]], rtol=0, atol=2e-15)
    # dosages 2, 1, 0: a tie (a = n = 3), mu = 1, s = sqrt(2); the het sample is 0
    G, M, Z = _G([[0, 2, 3]])
    s = 1.0 / math.sqrt(1.0 * (1.0 - 0.5))
    assert np.array_equal(Z[:, 0], [s, 0.0, -s])
    # dosages 2, missing, 0: n = 2, again a tie; the missing call is 0
    G, M, Z = _G([[0, 1, 3]])
    assert np.array_equal(Z[:, 0], [s, 0.0, -s]) and not G[1].any()
    # two variants: M = 2 and the cells are sums over both, divided once
    G, M, Z = _G([[0, 3, 3], [0, 2, 3]])
    assert M == 2 and np.array_equal(G, (Z @ Z.T) / 2)


@pytest.mark.parametrize("seed", range(4))
def test_table_matches_exact_rationals(seed):
    rng = np.random.default_rng(seed)
    for _ in range(300):
        h1, het, h2 = (int(x) for x in rng.integers(0, 60, 3))
        assert grm_ref.z_table(h1, het, h2) == grm_ref.z_table_exact(h1, het, h2)
    for h1, het, h2 in ((1, 0, 1), (0, 1, 0), (5, 0, 5), (0, 7, 0), (1, 98, 1), (123456, 7, 1)):
        assert grm_ref.z_table(h1, het, h2) == grm_ref.z_table_exact(h1, het, h2)


def test_vectorised_table_is_the_scalar_one():
    rng = np.random.default_rng(7)
    c = np.concatenate([rng.integers(0, 50, (500, 4)), [[3, 0, 0, 1], [0, 0, 4, 0], [0, 0, 0, 9], [2, 4, 2, 0]]])
    tab, used = grm_ref.z_tables(c)
    for v in range(len(c)):
        t = grm_ref.z_table(*(int(x) for x in c[v, :3]))
        assert (t is None) == (not used[v])
        assert np.array_equal(tab[v], t if t is not None else np.zeros(4))


def test_used_and_skipped():
    for h1, het, h2, used in ((4, 0, 0, False), (0, 0, 4, False), (0, 0, 0, False), (0, 4, 0, True), (1, 0, 0, False),
                              (1, 0, 1, True), (0, 1, 0, True)):
        assert (grm_ref.z_table(h1, het, h2) is not None) == used


def test_orientation_same_column_or_exact_negation_at_a_tie():
    rng = np.random.default_rng(3)
    code = grm_ref.balding_nichols(rng, 31, 400, miss=0.05)
    code[0] = [0, 2, 3] * 10 + [1]                 # a tie
    Za, _ = grm_ref.z_matrix(grm_ref.pack(code), 31)
    Zb, _ = grm_ref.z_matrix(grm_ref.pack(FLIP[code]), 31)
    c = qc_ref.counts(grm_ref.pack(code), 31).astype(np.int64)
    tie = (2 * c[:, 0] + c[:, 1] == c[:, 0] + c[:, 1] + c[:, 2])
    tie = tie[grm_ref.z_tables(c)[1]]
    assert tie.any()
    assert np.array_equal(Za[:, ~tie], Zb[:, ~tie]) and np.array_equal(Za[:, tie], -Zb[:, tie])
    Ga, _, _ = grm_ref.grm(grm_ref.pack(code), 31)
    Gb, _, _ = grm_ref.grm(grm_ref.pack(FLIP[code]), 31)
    assert np.array_equal(Ga, Gb)


def test_grm_is_centred():
    G, M, Z = _G(grm_ref.balding_nichols(np.random.default_rng(2), 50, 300))
    assert np.abs(G.sum(axis=1)).max() < 1e-12 * np.abs(G).max()


# ---- flags -----------------------------------------------------------------------------------------------------------
@pytest.fixture
def no_context(monkeypatch):
    def _native(self, n):
        raise AssertionError("a native context was requested")
    monkeypatch.setattr(VariantsPcaDriver, "_native", _native)


def _fileset(tmp_path, n=12, nv=60, seed=0):
    rng = np.random.default_rng(seed)
    prefix = str(tmp_path / "c")
    d = rng.integers(0, 3, size=(n, nv))
    d[rng.random((n, nv)) < 0.02] = -1
    plink.write_fileset(prefix, d, fam=[(f"F{i}", f"I{i}") for i in range(n)])
    return prefix


@pytest.mark.parametrize("argv,match", [
    (["--grm"], "--grm needs allele dosages"),
    (["BED", "--grm", "--king-cutoff", "0.1"], "--king-cutoff"),
    (["BED", "--grm", "--save-loadings", "x.npz"], "--save-loadings"),
    (["BED", "--grm", "--project-loadings", "x.npz"], "--project-loadings"),
    (["BED", "--grm", "--checkpoint-path", "ck"], "--checkpoint-path"),
    (["BED", "--make-rel", "--output-path", "P"], "--make-rel writes the matrix of --grm"),
    (["BED", "--grm", "--make-rel"], "--make-rel writes P.rel.bin"),
])
def test_flag_refusals(tmp_path, no_context, argv, match):
    prefix = _fileset(tmp_path)
    argv = [a if a != "BED" else "--bed-path" for a in argv]
    if argv[0] == "--bed-path":
        argv.insert(1, prefix)
    with pytest.raises(ValueError, match=match):
        variants_pca.main(argv)


def test_world_size_refused(tmp_path, no_context, monkeypatch):
    monkeypatch.setenv("WORLD_SIZE", "2")
    with pytest.raises(ValueError, match="--grm runs on one GPU"):
        variants_pca.main(["--bed-path", _fileset(tmp_path), "--grm"])


def test_sample_limit(tmp_path, no_context):
    check_grm_flags(PcaConf(["--bed-path", "x", "--grm"]), native.GRM_MAX_SAMPLES)
    with pytest.raises(ValueError, match="--grm is limited to 65535"):
        check_grm_flags(PcaConf(["--bed-path", "x", "--grm"]), native.GRM_MAX_SAMPLES + 1)
    n = native.GRM_MAX_SAMPLES + 2
    prefix = str(tmp_path / "big")
    plink.write_fileset(prefix, np.zeros((n, 1), np.int64))
    keep = tmp_path / "keep.id"
    keep.write_text("".join(f"synth S{i:06d}\n" for i in range(n - 1)))
    with pytest.raises(ValueError, match="--grm is limited to 65535"):
        variants_pca.main(["--bed-path", prefix, "--keep", str(keep), "--grm"])


# ---- formats ---------------------------------------------------------------------------------------------------------
def test_output_formats_read_back(tmp_path):
    fam = [("famA", "a1"), ("famA", "a2"), ("famB", "b1")]
    rng = np.random.default_rng(1)
    G = rng.standard_normal((3, 3))
    G = G + G.T
    prefix = str(tmp_path / "P")
    variants_pca.write_rel(prefix, fam, G)
    back = np.fromfile(prefix + ".rel.bin", dtype="<f8").reshape(3, 3)
    assert np.array_equal(back.view(np.int64), G.view(np.int64))
    assert (tmp_path / "P.rel.id").read_text() == "#FID\tIID\nfamA\ta1\nfamA\ta2\nfamB\tb1\n"
    vecs = rng.standard_normal((3, 2)) / 3.0
    evals = np.array([1.0 / 3.0, 0.1 + 0.2])
    variants_pca.write_eigen(prefix, fam, vecs, evals)
    lines = (tmp_path / "P.eigenvec").read_text().splitlines()
    assert lines[0] == "#FID\tIID\tPC1\tPC2"
    got = np.array([[float(x) for x in ln.split("\t")[2:]] for ln in lines[1:]])
    assert [ln.split("\t")[:2] for ln in lines[1:]] == [list(f) for f in fam]
    assert np.array_equal(got.view(np.int64), vecs.view(np.int64))
    ev = np.array([float(x) for x in (tmp_path / "P.eigenval").read_text().splitlines()])
    assert np.array_equal(ev.view(np.int64), evals.view(np.int64))


# ---- the driver through a numpy double ---------------------------------------------------------------------------------
class GrmDouble:
    """The GRM calls of native.NativePca, computed with tests/grm_ref.py."""

    def __init__(self, n):
        self.n, self.rows, self.kin_rows, self.G, self.M = n, [], [], None, None

    def reset(self):
        self.rows, self.kin_rows, self.G = [], [], None

    def grmBed(self, rows):
        self.rows.append(np.array(rows, np.uint8)[:, :(self.n + 3) // 4])

    def kinshipBed(self, rows):
        self.kin_rows.append(np.array(rows, np.uint8))

    def grmFinalize(self):
        self.G, self.M, _ = grm_ref.grm(np.concatenate(self.rows), self.n)
        if self.M == 0:
            raise native.VpcaError(native.VPCA_ERR_STATE, "M = 0")
        return self.M

    def getGrm(self):
        return self.G.copy()

    def computePcaGrm(self, k):
        w, V = np.linalg.eigh(self.G)
        w, V = w[::-1][:k].copy(), V[:, ::-1][:, :k].copy()
        V *= np.where(V[np.abs(V).argmax(axis=0), np.arange(k)] < 0, -1.0, 1.0)
        return V, w

    def stats(self):
        return dict(variants_accumulated=0, gram_launches=0, kernel_launches=0, h2d_bytes=0, last_gram_ms=0.0,
                    last_eig_ms=0.0)

    def close(self):
        pass


@pytest.fixture
def grm_double(monkeypatch):
    made = []

    def _native(self, n):
        if self._nat is None:
            self._nat = GrmDouble(n)
            made.append(self._nat)
        return self._nat
    monkeypatch.setattr(VariantsPcaDriver, "_native", _native)
    return made


def test_driver_end_to_end(tmp_path, capsys, grm_double):
    n, nv = 14, 90
    rng = np.random.default_rng(5)
    d = rng.integers(0, 3, size=(n, nv))
    d[rng.random((n, nv)) < 0.02] = -1
    d[:, 10] = 0                                            # three variants without variation among called samples
    d[:, 50] = 2
    d[:, 70] = -1
    prefix = str(tmp_path / "c")
    plink.write_fileset(prefix, d, fam=[(f"F{i}", f"I{i}") for i in range(n)])
    bed = plink.BedFile(prefix)
    rows = bed.rows(0, nv)
    P = str(tmp_path / "out")
    variants_pca.main(["--bed-path", prefix, "--grm", "--make-rel", "--num-pc", "3", "--output-path", P,
                       "--variants-per-partition", "40"])
    out = capsys.readouterr().out.splitlines()
    G, M, Z = grm_ref.grm(rows, n)
    assert M <= nv - 3
    assert f"GRM: {M} of {nv} variants used ({nv - M} skipped: no variation among called samples)." in out
    assert len(grm_double[0].rows) == 3                    # one call per partition
    back = np.fromfile(P + ".rel.bin", dtype="<f8").reshape(n, n)
    assert np.array_equal(back, G)
    vecs, evals = grm_double[0].computePcaGrm(3)
    lines = (tmp_path / "out.eigenvec").read_text().splitlines()
    assert lines[0] == "#FID\tIID\tPC1\tPC2\tPC3" and len(lines) == n + 1
    got = np.array([[float(x) for x in ln.split("\t")[2:]] for ln in lines[1:]])
    assert np.array_equal(got, vecs)
    assert [float(x) for x in (tmp_path / "out.eigenval").read_text().splitlines()] == evals.tolist()
    pcs = {ln.split("\t")[0]: ln for ln in out if ln.startswith("I") and "\t" in ln}
    assert len(pcs) == n


def test_driver_refuses_m_zero(tmp_path, grm_double):
    n = 8
    prefix = str(tmp_path / "mono")
    d = np.zeros((n, 5), np.int64)
    d[:, 2] = -1
    plink.write_fileset(prefix, d)
    with pytest.raises(ValueError, match="M = 0"):
        variants_pca.main(["--bed-path", prefix, "--grm"])
