"""GRM loadings and projection without a GPU (DESIGN.md 14): the flag refusals before any context is requested, the fields
of a --save-grm-loadings file, the .bim key matching of --project-loadings with the A1/A2 swap and its exchange of the
HOM_A1 / HOM_A2 table entries, the `GRM projection:` line, the refusal of a cohort without a loadings variant, P.eigenvec
read back, and carrier files still taking the carrier path, through a numpy double of the NativePca calls."""
import numpy as np
import pytest

import grm_projection_ref as ref
import grm_ref
from qc_ref import codes
from spark_examples_b200 import plink, variants_pca
from spark_examples_b200.variants_pca import VariantsPcaDriver, bimKeyBytes, _hash_words
from test_grm_cpu import GrmDouble


class GrmProjectionDouble(GrmDouble):
    """GrmDouble with the GRM loadings and projection calls, computed with tests/grm_projection_ref.py."""

    def __init__(self, n):
        super().__init__(n)
        self.U, self.acc, self.projected = None, None, []

    def computePcaGrm(self, k):
        V, w = super().computePcaGrm(k)
        self.U = V
        return V, w

    def grmLoadingsBed(self, k, rows):
        W, tab, _ = ref.loadings(np.asarray(rows), self.n, self.U[:, :k])
        return W, tab

    def projectBegin(self, k):
        self.acc = np.zeros((self.n, k))

    def projectGrmBed(self, rows, tab, w):
        self.projected.append((np.array(tab), np.array(w)))
        self.acc += ref.projection(np.asarray(rows), self.n, tab, w)[0]

    def projectGet(self, evals):
        return self.acc / np.asarray(evals)[None, :]


@pytest.fixture
def double(monkeypatch):
    made = []

    def _native(self, n):
        if self._nat is None:
            self._nat = GrmProjectionDouble(n)
            made.append(self._nat)
        return self._nat
    monkeypatch.setattr(VariantsPcaDriver, "_native", _native)
    return made


@pytest.fixture
def no_context(monkeypatch):
    def _native(self, n):
        raise AssertionError("a native context was requested")
    monkeypatch.setattr(VariantsPcaDriver, "_native", _native)


def _swap_bim(prefix, rows):
    """Exchange A1 and A2 of the given .bim rows."""
    lines = open(prefix + ".bim").read().splitlines()
    for j in rows:
        f = lines[j].split("\t")
        f[4], f[5] = f[5], f[4]
        lines[j] = "\t".join(f)
    open(prefix + ".bim", "w").write("\n".join(lines) + "\n")


def _cohort(tmp_path, name, d, positions, swapped=(), fam=None):
    prefix = str(tmp_path / name)
    d = np.array(d)
    d[:, list(swapped)] = np.where(d[:, list(swapped)] < 0, -1, 2 - d[:, list(swapped)])   # the same genotypes, A2 counted
    plink.write_fileset(prefix, d, fam=fam, positions=positions)
    _swap_bim(prefix, swapped)
    return prefix


def _dosages(seed, n, nv):
    rng = np.random.default_rng(seed)
    code = grm_ref.balding_nichols(rng, n, nv, miss=0.03)
    return np.where(code == 0, 2, np.where(code == 2, 1, np.where(code == 3, 0, -1))).T


def _save_reference(tmp_path, n=16, nv=50, k=3):
    d = _dosages(1, n, nv)
    prefix = _cohort(tmp_path, "ref", d, 1000 + np.arange(nv))
    npz = str(tmp_path / "r.npz")
    variants_pca.main(["--bed-path", prefix, "--grm", "--num-pc", str(k), "--save-grm-loadings", npz,
                       "--output-path", str(tmp_path / "R")])
    return prefix, npz, d


# ---- flags -----------------------------------------------------------------------------------------------------------
def test_flag_refusals(tmp_path, no_context, monkeypatch):
    prefix = _cohort(tmp_path, "c", _dosages(0, 12, 30), np.arange(30) + 1)
    with pytest.raises(ValueError, match="--save-grm-loadings writes the loadings of --grm's PCs: give --grm"):
        variants_pca.main(["--bed-path", prefix, "--save-grm-loadings", "x.npz"])
    with pytest.raises(ValueError, match="--save-grm-loadings stores at most 16 components; --num-pc 17"):
        variants_pca.main(["--bed-path", prefix, "--grm", "--num-pc", "17", "--save-grm-loadings", "x.npz"])
    with pytest.raises(ValueError, match="--save-grm-loadings"):   # the refusal of --grm --save-loadings points here
        variants_pca.main(["--bed-path", prefix, "--grm", "--save-loadings", "x.npz"])
    with pytest.raises(ValueError, match="projected without --grm"):
        variants_pca.main(["--bed-path", prefix, "--grm", "--project-loadings", "x.npz"])
    grm_file = str(tmp_path / "g.npz")
    np.savez(grm_file, matrix=np.str_("grm"))
    with pytest.raises(ValueError, match="holds GRM loadings.*--bed-path"):
        variants_pca.main(["--vcf-path", str(tmp_path / "x.vcf"), "--project-loadings", grm_file])
    monkeypatch.setenv("WORLD_SIZE", "2")
    with pytest.raises(ValueError, match="projecting GRM loadings runs on one GPU"):
        variants_pca.main(["--bed-path", prefix, "--project-loadings", grm_file])


# ---- the loadings file -------------------------------------------------------------------------------------------------
def test_file_fields(tmp_path, double):
    prefix, npz, d = _save_reference(tmp_path)
    nat = double[0]
    rows = plink.BedFile(prefix).rows(0, d.shape[1])
    G, M, Z = grm_ref.grm(rows, d.shape[0])
    V, w = nat.computePcaGrm(3)
    W, tab, _ = ref.loadings(rows, d.shape[0], V)
    with np.load(npz) as f:
        assert str(f["matrix"]) == "grm" and str(f["key_kind"]) == "bim"
        assert np.array_equal(f["loadings"], W) and np.array_equal(f["z_table"], tab)
        assert int(f["n_used"]) == M and int(f["n_samples"]) == d.shape[0]
        assert np.array_equal(f["eigenvalues"], w)
        want = np.asarray([_hash_words(bimKeyBytes(b)) for b in plink.read_bim(prefix)], np.uint64)
        assert np.array_equal(f["keys"], want)
        assert f["loadings"].shape == (d.shape[1], 3) and f["z_table"].shape == (d.shape[1], 4)


# ---- projection --------------------------------------------------------------------------------------------------------
def test_projection_matches_keys_swaps_alleles_and_writes_eigenvec(tmp_path, capsys, double):
    _, npz, _ = _save_reference(tmp_path)
    capsys.readouterr()
    # the study: reference variants 0 .. 39 (10 .. 19 with A1 / A2 swapped), then 5 variants the reference lacks
    n2 = 9
    d = _dosages(2, n2, 45)
    positions = np.concatenate([1000 + np.arange(40), 5000 + np.arange(5)])
    fam = [(f"N{i}", f"n{i}") for i in range(n2)]
    study = _cohort(tmp_path, "study", d, positions, swapped=range(10, 20), fam=fam)
    Q = str(tmp_path / "Q")
    variants_pca.main(["--bed-path", study, "--project-loadings", npz, "--output-path", Q])
    out = capsys.readouterr().out
    assert "GRM projection: 40 of 50 loadings variants found in this cohort (10 with A1/A2 swapped)." in out
    nat = double[-1]
    with np.load(npz) as f:
        W, tab, M, evals = f["loadings"], f["z_table"], int(f["n_used"]), f["eigenvalues"]
    (t_got, w_got), = nat.projected
    want_tab = tab[:40].copy()
    want_tab[10:20] = tab[10:20][:, [3, 1, 2, 0]]              # HOM_A1 and HOM_A2 exchanged on the swapped rows
    assert np.array_equal(t_got, want_tab) and np.array_equal(w_got, W[:40])
    # the swapped rows count the reference's allele: the projection equals that of the unswapped study
    rows = plink.BedFile(study).rows(0, 45)[:40]
    P = ref.projection(rows, n2, want_tab, W[:40])[0] / (M * evals)[None, :]
    plain = ref.projection(grm_ref.pack(grm_ref.dosage_codes(d[:, :40].T, d[:, :40].T < 0)), n2, tab[:40], W[:40])[0]
    assert np.allclose(P, plain / (M * evals)[None, :], rtol=1e-12, atol=1e-15)
    lines = open(Q + ".eigenvec").read().splitlines()
    assert lines[0] == "#FID\tIID\tPC1\tPC2\tPC3"
    assert [ln.split("\t")[:2] for ln in lines[1:]] == [list(f) for f in fam]
    got = np.array([[float(x) for x in ln.split("\t")[2:]] for ln in lines[1:]])
    assert np.array_equal(got.view(np.int64), P.view(np.int64))
    pcs = [ln for ln in out.splitlines() if ln.startswith("n") and "\t" in ln]
    assert len(pcs) == n2


def test_direct_match_wins_over_swapped(tmp_path, double):
    n, nv = 14, 30
    d = _dosages(3, n, nv)
    positions = 1000 + np.arange(nv)
    positions[1] = positions[0]                                # variant 1: variant 0's site with A1 / A2 swapped
    prefix = _cohort(tmp_path, "ref", d, positions, swapped=[1])
    npz = str(tmp_path / "r.npz")
    variants_pca.main(["--bed-path", prefix, "--grm", "--num-pc", "2", "--save-grm-loadings", npz])
    study = _cohort(tmp_path, "study", _dosages(4, 6, 2), positions[:2], swapped=[1])
    variants_pca.main(["--bed-path", study, "--project-loadings", npz])
    with np.load(npz) as f:
        W, tab = f["loadings"], f["z_table"]
    (t_got, w_got), = double[-1].projected
    assert np.array_equal(w_got, W[:2]) and np.array_equal(t_got, tab[:2])   # both direct, neither swapped


def test_no_loadings_variant_refused(tmp_path, capsys, double):
    _, npz, _ = _save_reference(tmp_path)
    study = _cohort(tmp_path, "study", _dosages(5, 6, 8), 90000 + np.arange(8))
    with pytest.raises(ValueError, match="none of the 50 variants"):
        variants_pca.main(["--bed-path", study, "--project-loadings", npz])
    assert "GRM projection: 0 of 50 loadings variants found in this cohort (0 with A1/A2 swapped)." in \
        capsys.readouterr().out
    assert double[-1].acc is None                              # refused before any projection


class SubsetDouble:
    """The sample subset call of the sample QC context: rows repacked to the kept samples, in numpy."""

    def subsetBedSamples(self, rows, n, kept):
        return grm_ref.pack(codes(np.asarray(rows), n)[:, np.asarray(kept)])

    def close(self):
        pass


def test_keep_selects_the_projected_samples(tmp_path, monkeypatch, double):
    monkeypatch.setattr(VariantsPcaDriver, "_sampleQcNative", lambda self: SubsetDouble())
    _, npz, _ = _save_reference(tmp_path)
    n2 = 10
    d = _dosages(6, n2, 50)
    study = _cohort(tmp_path, "study", d, 1000 + np.arange(50))
    (tmp_path / "keep.id").write_text("synth S000002\nsynth S000005\nsynth S000007\n")
    Q = str(tmp_path / "Q")
    variants_pca.main(["--bed-path", study, "--keep", str(tmp_path / "keep.id"), "--project-loadings", npz,
                       "--output-path", Q])
    lines = open(Q + ".eigenvec").read().splitlines()[1:]
    assert [ln.split("\t")[1] for ln in lines] == ["S000002", "S000005", "S000007"]
    assert double[-1].n == 3


def test_carrier_file_takes_the_carrier_path(tmp_path, monkeypatch):
    carrier = str(tmp_path / "c.npz")
    np.savez(carrier, loadings=np.ones((3, 2)), count=np.ones(3, np.int32), keys=np.zeros((3, 2), np.uint64),
             n_samples=np.int64(4), eigenvalues=np.ones(2), counted_allele=np.int32(1), key_kind=np.str_("bim"))
    assert variants_pca.loadings_matrix(carrier) == "carrier"

    def grm_path(self, callsets, path):
        raise AssertionError("a carrier file took the GRM path")

    class Reached(Exception):
        pass

    def _native(self, n):
        raise Reached()
    monkeypatch.setattr(VariantsPcaDriver, "projectGrmLoadings", grm_path)
    monkeypatch.setattr(VariantsPcaDriver, "_native", _native)
    prefix = _cohort(tmp_path, "c", _dosages(0, 8, 3), np.arange(3) + 1)
    with pytest.raises(Reached):
        variants_pca.main(["--bed-path", prefix, "--project-loadings", carrier])
