"""--save-loadings / --project-loadings on the CPU: which rows reach the loadings and projection calls, how variants are
matched by key, the .npz round trip, the rejections, and the output format -- with the native library replaced by a
TEST DOUBLE that computes through numpy / the oracle (the same flows run against libvpca.so in
tests/test_projection_gpu.py)."""
import numpy as np
import pytest

import spark_examples_b200 as pkg
from spark_examples_b200 import plink, variants_pca, vcf
from spark_examples_b200.jformat import jdouble
from spark_examples_b200.variants_common import CallsBatch, VariantsDataset
from spark_examples_b200.variants_pca import VariantsPcaDriver

from projection_ref import np_loadings, np_project


def _dense(n, off, idx):
    X = np.zeros((n, len(off) - 1), np.int64)
    rows = np.repeat(np.arange(len(off) - 1), np.diff(np.asarray(off, np.int64)))
    np.add.at(X, (np.asarray(idx[off[0]:off[-1]], np.int64), rows), 1)
    return X


class OracleBackedNative:
    """The NativePca calls the driver makes for a PCA, its loadings and a projection."""

    def __init__(self, oracle, n):
        self.o, self.n = oracle, n
        self.X = []                      # dense columns of every committed partition
        self.staged = {}
        self.log = []
        self.proj = None

    def reset(self):
        self.X, self.staged, self.proj = [], {}, None

    def accumulateCalls(self, pid, off, idx):
        self.staged[pid] = _dense(self.n, off, idx)

    def accumulateBed(self, pid, rows, counted):
        self.staged[pid] = plink.decode_rows(rows, self.n, counted).T.astype(np.int64)

    def commit(self, pid):
        self.X.append(self.staged.pop(pid))

    def abort(self, pid):
        self.staged.pop(pid, None)

    def finalizeGram(self):
        pass

    def getGram(self):
        X = np.concatenate(self.X, axis=1) if self.X else np.zeros((self.n, 0), np.int64)
        return self.o.np_similarity_dense(X)

    def computePca(self, k):
        S = self.getGram()
        U, _ = self.o.compute_pca(S, k)
        C, _, nz = self.o.np_center(S)
        self.U = self.o.sign_normalise(U)
        self.evals = np.sort(np.linalg.eigvalsh(C))[::-1][:k].copy()
        return self.U, self.evals, nz

    def loadingsCalls(self, k, off, idx):
        self.log.append(("loadings", len(off) - 1))
        return np_loadings(_dense(self.n, off, idx), self.U[:, :k])

    def loadingsBed(self, k, rows, counted):
        self.log.append(("loadings_bed", rows.shape[0]))
        return np_loadings(plink.decode_rows(rows, self.n, counted).T.astype(np.int64), self.U[:, :k])

    def projectBegin(self, k):
        self.proj = np.zeros((self.n, k))

    def projectCalls(self, off, idx, w, mean):
        assert self.proj is not None
        Y = _dense(self.n, off, idx)
        self.log.append(("project", Y.shape[1], Y.sum(axis=0).tolist()))
        self.proj += (Y - np.asarray(mean)[None, :]) @ np.asarray(w).reshape(Y.shape[1], -1)

    def projectBed(self, rows, w, mean, counted):
        Y = plink.decode_rows(rows, self.n, counted).T.astype(np.int64)
        self.log.append(("project_bed", Y.shape[1], Y.sum(axis=0).tolist()))
        self.proj += (Y - np.asarray(mean)[None, :]) @ np.asarray(w).reshape(Y.shape[1], -1)

    def projectGet(self, evals):
        return self.proj / np.asarray(evals)[None, :]

    def stats(self):
        return {"variants_accumulated": 0, "gram_launches": 0, "kernel_launches": 0, "h2d_bytes": 0, "last_gram_ms": 0.0,
                "last_eig_ms": 0.0}

    def close(self):
        pass


@pytest.fixture
def fake_native(monkeypatch, oracle):
    made = []

    def _native(self, n):
        if self._nat is None:
            self._nat = OracleBackedNative(oracle, n)
            made.append(self._nat)
        return self._nat
    monkeypatch.setattr(VariantsPcaDriver, "_native", _native)
    return made


GT = {0: "0/0", 1: "0/1", 2: "1/1"}


def _vcf(path, samples, d, positions):
    recs = [dict(chrom="chr17", pos=int(p), ref="A", alt=["C"], gts=[GT[int(x)] for x in d[:, j]])
            for j, p in enumerate(positions)]
    vcf.write_vcf(path, samples, recs)


def _lines(out):
    return [ln for ln in out.splitlines() if ln.count("\t") == 3]


def test_vcf_round_trip_and_key_matching(tmp_path, capsys, oracle, fake_native):
    d = oracle.c_synth_dense(20240901, 60, 0, 400, 1).astype(np.int64)
    samples = [f"NA{i:05d}" for i in range(60)]
    pos = 1000 + 3 * np.arange(400)
    ref = str(tmp_path / "ref.vcf")
    _vcf(ref, samples, d, pos)
    lpath = str(tmp_path / "ref.loadings.npz")
    variants_pca.main(["--vcf-path", ref, "--variants-per-partition", "150", "--save-loadings", lpath])
    capsys.readouterr()
    f = np.load(lpath)
    assert str(f["key_kind"]) == "variant" and int(f["counted_allele"]) == 0 and int(f["n_samples"]) == 60
    has = (d > 0).astype(np.int64)
    kept = has.any(axis=0)                                      # rows without carriers were dropped at :166
    U = fake_native[0].U
    W, C = np_loadings(has[:, kept], U)
    assert np.array_equal(f["count"], C) and np.allclose(f["loadings"], W, rtol=0, atol=1e-12)
    assert np.array_equal(f["eigenvalues"], fake_native[0].evals[:2])
    recs = list(vcf.read_variants(ref, None))
    want_keys = [variants_pca._hash_words(variants_pca.variantKeyBytes(recs[j])) for j in np.flatnonzero(kept)]
    assert [tuple(int(x) for x in r) for r in f["keys"]] == want_keys

    # new cohort: 25 samples, variants reordered, a fifth of the reference's missing, 30 extra sites, one site without
    # carriers in the new cohort
    rng = np.random.default_rng(5)
    new = oracle.c_synth_dense(77, 25, 0, 400, 1).astype(np.int64)
    cols = rng.permutation(400)[:320]
    empty_col = int(np.flatnonzero(kept[cols])[0])
    new[:, cols[empty_col]] = 0
    extra = oracle.c_synth_dense(78, 25, 0, 30, 1).astype(np.int64)
    Y = np.concatenate([new[:, cols], extra], axis=1)
    ypos = np.concatenate([pos[cols], 5000 + np.arange(30)])
    nsamples = [f"NEW{i:03d}" for i in range(25)]
    path = str(tmp_path / "new.vcf")
    _vcf(path, nsamples, Y, ypos)
    variants_pca.main(["--vcf-path", path, "--variants-per-partition", "100", "--project-loadings", lpath,
                       "--output-path", str(tmp_path / "o")])
    got = _lines(capsys.readouterr().out)
    proj = fake_native[-1]
    sent = [e for e in proj.log if e[0] == "project"]
    in_file = kept[cols]                                        # the new rows whose key is in the file
    assert sum(e[1] for e in sent) == int(in_file.sum())
    assert any(0 in e[2] for e in sent)                         # the row without carriers reached projectCalls
    ref_row = np.cumsum(kept) - 1                               # reference column -> row of the file
    P = np_project((Y[:, :320] > 0)[:, in_file], f["loadings"][ref_row[cols[in_file]]], f["count"][ref_row[cols[in_file]]],
                   60, f["eigenvalues"])
    want = sorted((nsamples[i], "new", P[i, 0], P[i, 1]) for i in range(25))
    assert len(got) == 25
    for ln, (nm, ds, a, b) in zip(got, want):
        name, dataset, pc1, pc2 = ln.split("\t")
        assert (name, dataset) == (nm, ds)
        assert abs(float(pc1) - a) <= 1e-12 * abs(P[:, 0]).max() and abs(float(pc2) - b) <= 1e-12 * abs(P[:, 1]).max()
    # emitResult's format: name, dataset, then Java's Double.toString of each coordinate
    res = [(nsamples[i], float(a), float(b)) for i, (a, b) in enumerate(proj.projectGet(f["eigenvalues"])[:, :2])]
    assert got == [f"{nm}\tnew\t{jdouble(a)}\t{jdouble(b)}" for nm, a, b in sorted(res)]
    part = (tmp_path / "o-pca.tsv" / "part-00000").read_text().splitlines()
    assert len(part) == 25 and (tmp_path / "o-pca.tsv" / "_SUCCESS").exists()


def test_bed_keys_and_rows_without_carriers(tmp_path, capsys, oracle, fake_native):
    d = oracle.c_synth_dense(9, 40, 0, 300, 1).astype(np.int64)
    d[:, 7] = 0                                                 # no carriers of A1 at site 7
    plink.write_fileset(str(tmp_path / "r"), d)
    lpath = str(tmp_path / "r.npz")
    variants_pca.main(["--bed-path", str(tmp_path / "r"), "--variants-per-partition", "128", "--save-loadings", lpath])
    capsys.readouterr()
    f = np.load(lpath)
    assert str(f["key_kind"]) == "bim" and int(f["counted_allele"]) == 1 and len(f["count"]) == 300
    assert f["count"][7] == 0 and np.all(f["loadings"][7] == 0)
    assert [e for e in fake_native[0].log if e[0] == "loadings_bed"] == [("loadings_bed", 128), ("loadings_bed", 128),
                                                                         ("loadings_bed", 44)]
    variants_pca.main(["--bed-path", str(tmp_path / "r"), "--project-loadings", lpath])
    got = _lines(capsys.readouterr().out)
    sent = [e for e in fake_native[-1].log if e[0] == "project_bed"]
    assert sum(e[1] for e in sent) == 300 and sent[0][2][7] == 0
    U = fake_native[0].U                                        # self-projection returns the reference's eigenvectors
    for ln in got:
        i = int(ln.split("\t")[0][1:])
        assert np.allclose([float(x) for x in ln.split("\t")[2:]], U[i, :2], rtol=0, atol=1e-10)


def _save(path, **kw):
    base = dict(loadings=np.ones((3, 2)), count=np.ones(3, np.int32), n_samples=np.int64(10),
                eigenvalues=np.ones(2), counted_allele=np.int32(1), keys=np.zeros((3, 2), np.uint64), key_kind=np.str_("bim"))
    base.update(kw)
    with open(path, "wb") as fh:
        np.savez(fh, **base)


def test_rejections(tmp_path, oracle, fake_native):
    d = oracle.c_synth_dense(9, 20, 0, 50, 1).astype(np.int64)
    plink.write_fileset(str(tmp_path / "r"), d)
    argv = ["--bed-path", str(tmp_path / "r"), "--project-loadings"]
    _save(tmp_path / "kind.npz", key_kind=np.str_("variant"))
    with pytest.raises(ValueError, match="keys"):
        variants_pca.main(argv + [str(tmp_path / "kind.npz")])
    _save(tmp_path / "allele.npz", counted_allele=np.int32(2))
    with pytest.raises(ValueError, match="allele"):
        variants_pca.main(argv + [str(tmp_path / "allele.npz")])
    _save(tmp_path / "k1.npz", loadings=np.ones((3, 1)), eigenvalues=np.ones(1))
    with pytest.raises(ValueError, match="at least 2"):
        variants_pca.main(argv + [str(tmp_path / "k1.npz")])
    # joined multi-dataset input (two VCF files) is refused before any Gram is computed
    samples = [f"A{i}" for i in range(5)]
    for nm in ("a", "b"):
        _vcf(str(tmp_path / f"{nm}.vcf"), samples if nm == "a" else [f"B{i}" for i in range(5)], d[:5, :10], 100 + np.arange(10))
    vcfs = f"{tmp_path / 'a.vcf'},{tmp_path / 'b.vcf'}"
    for flag in ("--save-loadings", "--project-loadings"):
        with pytest.raises(ValueError, match="joined"):
            variants_pca.main(["--vcf-path", vcfs, flag, str(tmp_path / "j.npz")])
    assert all(not n.X for n in fake_native)


def test_save_loadings_refuses_more_than_16_components_before_the_gram(tmp_path, monkeypatch, oracle, fake_native):
    """Loadings hold at most 16 components: --num-pc 17 with --save-loadings fails before any Gram is requested, not
    after the Gram and the eigensolve."""
    d = oracle.c_synth_dense(9, 40, 0, 100, 1).astype(np.int64)
    plink.write_fileset(str(tmp_path / "r"), d)
    grams = []
    gram = VariantsPcaDriver.getSimilarityMatrix
    monkeypatch.setattr(VariantsPcaDriver, "getSimilarityMatrix", lambda self, calls: grams.append(1) or gram(self, calls))
    argv = ["--bed-path", str(tmp_path / "r"), "--save-loadings", str(tmp_path / "r.npz")]
    with pytest.raises(ValueError, match="at most 16 components"):
        variants_pca.main(argv + ["--num-pc", "17"])
    assert grams == [] and all(not n.X and not n.staged for n in fake_native)
    assert not (tmp_path / "r.npz").exists()
    variants_pca.main(argv + ["--num-pc", "16"])                 # 16 is still accepted
    assert len(grams) == 1


def test_row_keys_for_in_memory_calls(tmp_path, oracle, fake_native):
    """CSR partitions carry no identity: rows are keyed by their global index, so a re-run on the same rows matches."""
    X = oracle.c_synth_dense(4, 30, 0, 90, 0).astype(np.int64)
    conf = pkg.PcaConf(["--save-loadings", str(tmp_path / "m.npz")])
    off, idx = [], []
    parts = []
    for c0 in (0, 40):
        cols = X[:, c0:c0 + 50 if c0 == 40 else 40]
        o = np.concatenate([[0], np.cumsum(cols.sum(axis=0))]).astype(np.int64)
        ix = np.concatenate([np.nonzero(cols[:, j])[0] for j in range(cols.shape[1])]).astype(np.int32)
        parts.append(CallsBatch(o, ix))
    common = pkg.VariantsCommon(conf, callsets=[(f"c-{i}", f"C{i}") for i in range(30)], datasets=[[]])
    common.data = [VariantsDataset(parts)]
    driver = VariantsPcaDriver(conf, common=common)
    calls = driver.getCallsRdd(driver.getData)
    assert driver.keyKind(calls) == "row"
    driver.computePca(driver.getSimilarityMatrix(calls))
    driver.saveLoadings(calls)
    f = np.load(tmp_path / "m.npz")
    assert str(f["key_kind"]) == "row" and np.array_equal(f["keys"][:, 0], np.arange(90))
    assert np.allclose(f["loadings"], np_loadings(X, fake_native[0].U)[0], rtol=0, atol=1e-12)
