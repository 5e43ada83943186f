"""Linear association tests without a GPU (DESIGN.md 15): the --pheno / --covar file formats, every refusal before any
context is requested, the P.<PHENO>.glm.linear format and the `GLM linear:` line, the driver end to end through a numpy
double of glmBegin / glmLinearBed (every QC-passing variant tested, with --keep, --mind, --grm and --project-loadings),
and the stratification the PCs remove: lambda_GC on a seeded three-population cohort without and with the PCs."""
import numpy as np
import pytest

import glm_ref
import grm_ref
from qc_ref import codes, counts, hwe_p_many
from spark_examples_b200 import native, plink, variants_pca
from spark_examples_b200.variants_pca import VariantsPcaDriver
from test_grm_projection_cpu import GrmProjectionDouble, SubsetDouble


class Double(GrmProjectionDouble, glm_ref.GlmDouble):
    """The GRM, projection and GLM calls in numpy, and variant QC counts."""

    def variantQcBed(self, rows):
        c = counts(np.asarray(rows), self.n)
        return c, hwe_p_many(c)


@pytest.fixture
def double(monkeypatch):
    made = []

    def _native(self, n):
        if self._nat is None:
            self._nat = Double(n)
            made.append(self._nat)
        return self._nat
    monkeypatch.setattr(VariantsPcaDriver, "_native", _native)
    monkeypatch.setattr(VariantsPcaDriver, "_sampleQcNative", lambda self: MissingDouble())
    return made


class MissingDouble(SubsetDouble):
    def sampleMissingBed(self, rows, n):
        return (codes(np.asarray(rows), n) == 1).sum(axis=0)


@pytest.fixture
def no_context(monkeypatch):
    def _native(self, n):
        raise AssertionError("a native context was requested")
    monkeypatch.setattr(VariantsPcaDriver, "_native", _native)


def _pop_sizes(n, pops=3):
    share = 1.12 ** np.arange(pops)
    sizes = np.floor(n * share / share.sum()).astype(np.int64)
    sizes[np.argsort(-(n * share / share.sum() - sizes))[: n - sizes.sum()]] += 1
    return sizes


def _fileset(tmp_path, n=40, nv=120, seed=0, miss=0.02):
    rng = np.random.default_rng(seed)
    code = grm_ref.balding_nichols(rng, n, nv, miss=miss)
    code[5] = 0                                                  # a monomorphic variant
    d = np.where(code == 0, 2, np.where(code == 2, 1, np.where(code == 3, 0, -1))).T
    prefix = str(tmp_path / "c")
    fam = [(f"F{i // 3}", f"I{i}") for i in range(n)]
    plink.write_fileset(prefix, d, fam=fam, positions=100 * np.arange(nv) + 1)
    y = np.repeat([0.0, 0.5, 1.0], _pop_sizes(n)) + rng.normal(size=n)
    return prefix, fam, y


def _pheno_file(tmp_path, fam, y, name="T", header="#FID IID", missing=()):
    lines = [f"{header} {name}"] if header else []
    for i, ((f, iid), v) in enumerate(zip(fam, y)):
        val = "NA" if i in missing else repr(float(v))
        lines.append(f"{iid} {val}" if header == "#IID" else f"{f} {iid} {val}")
    path = tmp_path / f"pheno_{name}.txt"
    path.write_text("\n".join(lines) + "\n")
    return str(path)


# ---- file formats --------------------------------------------------------------------------------------------------
def test_value_file_headers_bare_iids_and_missing_tokens(tmp_path):
    p = tmp_path / "a.txt"
    p.write_text("#FID IID A B\nf1 i1 1.5 NA\nf2 i2 nan -9\n\nf3 i3 -2e3 7\n")
    names, ids, v = plink.read_value_file(str(p), "PHENO")
    assert names == ["A", "B"] and ids == [("f1", "i1"), ("f2", "i2"), ("f3", "i3")]
    assert np.array_equal(v, np.array([[1.5, np.nan], [np.nan, np.nan], [-2e3, 7.0]]), equal_nan=True)
    p.write_text("FID IID X\nf1 i1 3\n")
    assert plink.read_value_file(str(p), "PHENO")[0] == ["X"]
    p.write_text("#IID X Y\ni1 3 4\ni2 5 NA\n")
    names, ids, v = plink.read_value_file(str(p), "COVAR")
    assert names == ["X", "Y"] and ids == [(None, "i1"), (None, "i2")]
    p.write_text("f1 i1 3 4\nf2 i2 5 6\n")
    names, ids, v = plink.read_value_file(str(p), "COVAR")
    assert names == ["COVAR1", "COVAR2"] and ids == [("f1", "i1"), ("f2", "i2")] and v.shape == (2, 2)
    for bad, what in (("f1 i1 3\nf2 i2 abc\n", "line 2: 'abc' is not a number"),
                      ("f1 i1 3\nf2 i2 inf\n", "line 2: 'inf' is not a number"),
                      ("#FID IID A\nf1 i1 3 4\n", "line 2 has 4 fields, 3 expected")):
        p.write_text(bad)
        with pytest.raises(ValueError, match=what):
            plink.read_value_file(str(p), "PHENO")


def test_ids_matched_and_unmatched_counted(tmp_path, capsys, double):
    prefix, fam, y = _fileset(tmp_path)
    lines = ["#IID T"] + [f"{iid} {float(v)!r}" for (_, iid), v in zip(fam, y)] + ["nobody 1.0", "ghost 2.0"]
    (tmp_path / "p.txt").write_text("\n".join(lines) + "\n")
    P = str(tmp_path / "P")
    variants_pca.main(["--bed-path", prefix, "--grm", "--pheno", str(tmp_path / "p.txt"), "--glm", "--output-path", P])
    out = capsys.readouterr().out
    assert f"--pheno {tmp_path / 'p.txt'}: 2 IDs match no sample." in out
    assert np.array_equal(double[0].glm[0], y)


# ---- refusals ------------------------------------------------------------------------------------------------------
def test_refusals_before_any_context(tmp_path, no_context, monkeypatch):
    prefix, fam, y = _fileset(tmp_path)
    ph = _pheno_file(tmp_path, fam, y)
    base = ["--bed-path", prefix, "--output-path", str(tmp_path / "P")]
    for argv, what in (
            (base + ["--pheno", ph], "--pheno is read by --glm: give --glm"),
            (base + ["--pheno-name", "T"], "--pheno-name is read by --glm"),
            (base + ["--covar", ph], "--covar is read by --glm"),
            (base + ["--glm"], "give --pheno FILE"),
            (["--synthetic", "8,8", "--glm", "--pheno", ph, "--output-path", "P"], "give a PLINK fileset with --bed-path"),
            (["--bed-path", prefix, "--glm", "--pheno", ph], "give --output-path P"),
            (base + ["--glm", "--pheno", ph, "--checkpoint-path", str(tmp_path / "ck")], "--checkpoint-path"),
            (base + ["--glm", "--pheno", ph, "--pheno-name", "U"], "--pheno-name U: .* has the columns T"),
            (base + ["--glm", "--pheno", ph, "--num-pc", "32"], "at most 32 covariates.*make 33"),
            (base + ["--glm", "--pheno", _pheno_file(tmp_path, fam, (np.arange(len(fam)) % 2).astype(float), "B"),
                     "--pheno-name", "B"], "case/control traits need logistic regression")):
        with pytest.raises(ValueError, match=what):
            variants_pca.main(argv)
    cov = tmp_path / "cov.txt"
    cov.write_text("".join(f"{f} {i} " + " ".join("1.0" for _ in range(20)) + "\n" for f, i in fam))
    with pytest.raises(ValueError, match=r"the intercept, --num-pc 12 and 20 --covar columns make 33"):
        variants_pca.main(base + ["--glm", "--pheno", ph, "--covar", str(cov), "--num-pc", "12"])
    npz = tmp_path / "l.npz"
    np.savez(npz, matrix=np.str_("grm"), loadings=np.zeros((3, 31)))
    with pytest.raises(ValueError, match=r"the 31 PCs of .*l.npz and 1 --covar columns make 33"):
        cov.write_text("".join(f"{f} {i} 1.0\n" for f, i in fam))
        variants_pca.main(base + ["--glm", "--pheno", ph, "--covar", str(cov), "--project-loadings", str(npz)])
    monkeypatch.setenv("WORLD_SIZE", "2")
    with pytest.raises(ValueError, match="--glm runs on one GPU"):
        variants_pca.main(base + ["--glm", "--pheno", ph])


def test_refusals_after_sample_qc(tmp_path, double):
    prefix, fam, y = _fileset(tmp_path, n=12)
    few = np.full(len(y), np.nan)
    few[:4] = [1.0, 2.0, 3.0, 4.0]
    with pytest.raises(ValueError, match="4 of 12 samples have a phenotype and every covariate; 3 covariates .* at least 5"):
        variants_pca.main(["--bed-path", prefix, "--grm", "--glm", "--pheno", _pheno_file(tmp_path, fam, few),
                           "--output-path", str(tmp_path / "P")])
    two = np.where(np.arange(len(y)) < 6, 1.0, 2.0)
    two[:3] = 5.0                                               # three values, but only two among the kept samples
    (tmp_path / "keep.id").write_text("".join(f"{f} {i}\n" for f, i in fam[3:]))
    with pytest.raises(ValueError, match="case/control"):
        variants_pca.main(["--bed-path", prefix, "--grm", "--keep", str(tmp_path / "keep.id"), "--glm", "--pheno",
                           _pheno_file(tmp_path, fam, two), "--output-path", str(tmp_path / "P")])
    assert all(nat.G is None for nat in double)                 # refused before the GRM


# ---- output ----------------------------------------------------------------------------------------------------------
def _read(path):
    lines = open(path).read().splitlines()
    return lines[0].split("\t"), [ln.split("\t") for ln in lines[1:]]


def _numbers(rows):
    return np.array([[np.nan if x == "NA" else float(x) for x in (r[8], r[6], r[9], r[10], r[11], r[12])] for r in rows])


@pytest.mark.parametrize("extra", [[], ["--keep", "keep"], ["--mind", "0.5", "--maf", "0.05"]])
def test_grm_run_end_to_end(tmp_path, capsys, double, extra):
    prefix, fam, y = _fileset(tmp_path)
    miss = {2, 9}
    ph = _pheno_file(tmp_path, fam, y, missing=miss)
    cov = tmp_path / "cov.txt"
    z = np.random.default_rng(4).normal(size=len(fam))
    cov.write_text("#FID IID AGE\n" + "".join(f"{f} {i} {'NA' if k == 11 else repr(float(z[k]))}\n"
                                              for k, (f, i) in enumerate(fam)))
    if extra[:1] == ["--keep"]:
        (tmp_path / "keep.id").write_text("".join(f"{f} {i}\n" for f, i in fam[4:]))
        extra = ["--keep", str(tmp_path / "keep.id")]
    P = str(tmp_path / "P")
    variants_pca.main(["--bed-path", prefix, "--grm", "--num-pc", "3", "--glm", "--pheno", ph, "--covar", str(cov),
                       "--output-path", P] + extra)
    out = capsys.readouterr().out
    nat = double[-1]
    kept = np.array([fam.index(tuple(ln.split("\t")[:2])) for ln in open(P + ".eigenvec").read().splitlines()[1:]])
    ev = np.array([[float(x) for x in ln.split("\t")[2:]] for ln in open(P + ".eigenvec").read().splitlines()[1:]])
    bed = plink.BedFile(prefix)
    rows = grm_ref.pack(codes(bed.rows(0, bed.n_variants), len(fam))[:, kept])
    keep = np.ones(bed.n_variants, bool)
    if "--maf" in extra:
        keep, _ = variants_pca.variant_qc_keep(counts(rows, len(kept)), None, 0.05, None, None)
    yk = y[kept].copy()
    yk[np.isin(kept, list(miss))] = np.nan
    zk = z[kept].copy()
    zk[kept == 11] = np.nan
    want, werr = glm_ref.linear(rows[keep], len(kept), yk, np.concatenate([ev, zk[:, None]], axis=1))
    head, got = _read(P + ".T.glm.linear")
    assert head == ["#CHROM", "POS", "ID", "REF", "ALT", "A1", "A1_FREQ", "TEST", "OBS_CT", "BETA", "SE", "T_STAT", "P",
                    "ERRCODE"]
    bim = [b for b, k in zip(plink.read_bim(prefix), keep) if k]
    assert [r[:6] for r in got] == [[b.contig, str(b.position), b.id, b.a2, b.a1, b.a1] for b in bim]
    assert all(r[7] == "ADD" for r in got)
    assert [r[13] for r in got] == [glm_ref.ERRCODES[e] for e in werr]
    assert np.array_equal(_numbers(got), want, equal_nan=True)   # the double's numbers, read back bit for bit
    assert "nan" not in open(P + ".T.glm.linear").read().lower().replace("na\t", "")
    reg = int((np.isfinite(yk) & np.isfinite(zk)).sum())
    lam = glm_ref.lambda_gc(want, werr)
    assert (f"GLM linear: T on {reg} of {len(kept)} samples ({len(kept) - reg} without a phenotype or covariate), 5 "
            f"covariates (intercept, 3 PCs, 1 from {cov}); {int(keep.sum())} variants tested, "
            f"{int(np.count_nonzero(werr))} with an ERRCODE; lambda_GC = {lam!r}.") in out
    assert werr[list(np.flatnonzero(keep)).index(5)] == 2 if keep[5] else True


def test_every_qc_passing_variant_not_only_the_pruned(tmp_path, capsys, double, monkeypatch):
    prefix, fam, y = _fileset(tmp_path)
    pruned = np.zeros(120, bool)
    pruned[::3] = True

    def ld_prune(self, callsets, window_lo, eligible=None):
        for p in callsets.partitions:
            p.keep = pruned[p.v0:p.v0 + p.nv]
        return pruned
    monkeypatch.setattr(VariantsPcaDriver, "ldPrune", ld_prune)
    P = str(tmp_path / "P")
    variants_pca.main(["--bed-path", prefix, "--grm", "--ld-prune", "0.2", "--variants-per-partition", "50", "--glm",
                       "--pheno", _pheno_file(tmp_path, fam, y), "--output-path", P])
    _, got = _read(P + ".T.glm.linear")
    assert len(got) == 120
    assert sum(len(r) for r in double[0].rows) // 1 and sum(r.shape[0] for r in double[0].rows) == 40   # PCs: pruned
    assert double[0].glm_calls == [50, 50, 20]                   # tests: every variant, partition by partition


def test_projection_run(tmp_path, capsys, double):
    prefix, fam, y = _fileset(tmp_path)
    npz = str(tmp_path / "r.npz")
    variants_pca.main(["--bed-path", prefix, "--grm", "--num-pc", "2", "--save-grm-loadings", npz])
    study, fam2, y2 = _fileset(tmp_path / ".." / tmp_path.name, n=25, seed=3)
    P = str(tmp_path / "Q")
    variants_pca.main(["--bed-path", study, "--project-loadings", npz, "--glm", "--pheno",
                       _pheno_file(tmp_path, fam2, y2, "Z"), "--output-path", P])
    out = capsys.readouterr().out
    ev = np.array([[float(x) for x in ln.split("\t")[2:]] for ln in open(P + ".eigenvec").read().splitlines()[1:]])
    rows = plink.BedFile(study).rows(0, 120)
    want, werr = glm_ref.linear(rows, 25, y2, ev)
    _, got = _read(P + ".Z.glm.linear")
    assert np.array_equal(_numbers(got), want, equal_nan=True)
    assert "3 covariates (intercept, 2 PCs); 120 variants tested" in out


def test_write_format_numbers():
    b = plink.BimRecord("3", "rs9", 77, "T", "C")
    import io, os, tempfile
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "x.glm.linear")
        st = np.array([[10, 0.15, 0.1, 0.2, 0.5, 0.6170750774519738], [3, np.nan, np.nan, np.nan, np.nan, np.nan]])
        variants_pca.write_glm_linear(path, [b, b], 2, st, np.array([0, 1]))
        lines = open(path).read().splitlines()
    assert lines[1] == "3\t77\trs9\tC\tT\tC\t0.15\tADD\t10\t0.1\t0.2\t0.5\t0.6170750774519738\t."
    assert lines[2] == "3\t77\trs9\tC\tT\tC\tNA\tADD\t3\tNA\tNA\tNA\tNA\tTOO_FEW_OBS"


# ---- the stratification the PCs remove -----------------------------------------------------------------------------------
def test_pcs_remove_the_stratification():
    """The seeded cohort: 600 samples of 3 populations, 4000 variants, 1 % missing calls, a phenotype of population mean
    (0, 0.5, 1) plus N(0, 1) noise and no causal variant."""
    rng = np.random.default_rng(7)
    n = 600
    code = grm_ref.balding_nichols(rng, n, 4000, pops=3, miss=0.01)
    y = np.repeat([0.0, 0.5, 1.0], _pop_sizes(n)) + rng.normal(size=n)
    rows = grm_ref.pack(code)
    G, M, Z = grm_ref.grm(rows, n)
    pcs = grm_ref.Pcs(Z, 2).U
    sub = rows[::4]                                              # 1000 of the variants keep the reference quick
    plain = glm_ref.lambda_gc(*glm_ref.linear(sub, n, y))
    adjusted = glm_ref.lambda_gc(*glm_ref.linear(sub, n, y, pcs))
    assert plain > 2.0
    assert 0.9 <= adjusted <= 1.1


class KingGlmDouble(glm_ref.GlmDouble):
    """The carrier path with --king-cutoff in numpy: samples 0 and 1 and samples 7 and 8 are the related pairs, and the
    subset solve returns fixed PCs for every sample (kept and projected), which the tests read back as the covariates."""

    def __init__(self, n):
        self.n = n
        self.vecs = np.random.default_rng(99).normal(size=(n, 3))

    def reset(self):
        pass

    def kinshipBed(self, rows):
        pass

    def accumulateBed(self, pid, rows, counted):
        pass

    def commit(self, pid):
        pass

    def abort(self, pid):
        pass

    def finalizeGram(self):
        pass

    def kinshipPairs(self, min_kinship=float("-inf")):
        ids = np.array([[0, 1], [7, 8]], np.int32)
        return ids, np.zeros((2, 5), np.int32), np.array([0.3, 0.25])

    def computePcaSubset(self, keep, k):
        self.keep = np.array(keep)
        return self.vecs[:, :k].copy(), np.arange(k, 0, -1).astype(float), int(keep.sum())

    def stats(self):
        return dict(variants_accumulated=0, gram_launches=0, kernel_launches=0, h2d_bytes=0, last_gram_ms=0.0,
                    last_eig_ms=0.0)

    def close(self):
        pass


def test_king_cutoff_run_end_to_end(tmp_path, capsys, monkeypatch):
    made = []

    def _native(self, n):
        if self._nat is None:
            self._nat = KingGlmDouble(n)
            made.append(self._nat)
        return self._nat
    monkeypatch.setattr(VariantsPcaDriver, "_native", _native)
    prefix, fam, y = _fileset(tmp_path)
    P = str(tmp_path / "P")
    variants_pca.main(["--bed-path", prefix, "--king-cutoff", "0.177", "--num-pc", "3", "--glm", "--pheno",
                       _pheno_file(tmp_path, fam, y, missing={4}), "--output-path", P])
    nat = made[0]
    assert int(nat.keep.sum()) == len(fam) - 2                   # one of each related pair projected, not dropped
    yk = y.copy()
    yk[4] = np.nan
    rows = plink.BedFile(prefix).rows(0, 120)
    want, werr = glm_ref.linear(rows, len(fam), yk, nat.vecs)   # every sample, the projected ones included
    _, got = _read(P + ".T.glm.linear")
    assert np.array_equal(_numbers(got), want, equal_nan=True)
    assert [r[13] for r in got] == [glm_ref.ERRCODES[e] for e in werr]
    assert f"GLM linear: T on {len(fam) - 1} of {len(fam)} samples (1 without a phenotype or covariate), 4 covariates " \
           "(intercept, 3 PCs); 120 variants tested" in capsys.readouterr().out


def test_ids_of_samples_removed_by_sample_qc_are_not_unmatched(tmp_path, capsys, double):
    prefix, fam, y = _fileset(tmp_path)
    (tmp_path / "keep.id").write_text("".join(f"{f} {i}\n" for f, i in fam[5:]))
    lines = ["#FID IID T"] + [f"{f} {i} {float(v)!r}" for (f, i), v in zip(fam, y)] + ["X nobody 1.0"]
    (tmp_path / "p.txt").write_text("\n".join(lines) + "\n")
    variants_pca.main(["--bed-path", prefix, "--keep", str(tmp_path / "keep.id"), "--grm", "--pheno",
                       str(tmp_path / "p.txt"), "--glm", "--output-path", str(tmp_path / "P")])
    out = capsys.readouterr().out
    assert f"--pheno {tmp_path / 'p.txt'}: 1 IDs match no sample." in out   # not the 5 samples --keep left out
    assert np.array_equal(double[-1].glm[0], y[5:])
