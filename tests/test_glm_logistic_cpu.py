"""Logistic association tests without a GPU (DESIGN.md 16): the reference against scipy.optimize, the case/control coding
and every refusal before any context is requested, --glm alone still refusing a case/control trait, the
P.<PHENO>.glm.logistic format and the `GLM logistic:` line, the driver end to end through a numpy double of
glmLogisticBegin / glmLogisticBed on the --grm, --king-cutoff and --project-loadings paths, and the stratification the
PCs remove from a case/control trait."""
import numpy as np
import pytest
import scipy.optimize

import glm_logistic_ref as ref
import grm_ref
from qc_ref import codes
from spark_examples_b200 import native, plink, variants_pca
from spark_examples_b200.variants_pca import VariantsPcaDriver
from test_glm_cpu import Double, KingGlmDouble, MissingDouble, _fileset, _pheno_file, _pop_sizes, _read


class LogDouble(Double, ref.LogisticDouble):
    pass


class KingLogDouble(KingGlmDouble, ref.LogisticDouble):
    pass


@pytest.fixture
def double(monkeypatch):
    made = []

    def _native(self, n):
        if self._nat is None:
            self._nat = LogDouble(n)
            made.append(self._nat)
        return self._nat
    monkeypatch.setattr(VariantsPcaDriver, "_native", _native)
    monkeypatch.setattr(VariantsPcaDriver, "_sampleQcNative", lambda self: MissingDouble())
    return made


@pytest.fixture
def no_context(monkeypatch):
    def _native(self, n):
        raise AssertionError("a native context was requested")
    monkeypatch.setattr(VariantsPcaDriver, "_native", _native)


def _cc(fam, seed=1, rate=0.3):
    """A PLINK-coded case/control phenotype (1 control, 2 case) of the fileset's samples."""
    rng = np.random.default_rng(seed)
    return np.where(rng.random(len(fam)) < rate, 2.0, 1.0)


# ---- the reference -----------------------------------------------------------------------------------------------------
def _rare_rows(rng, y, n):
    """Rows of A2 carriers among a fixed-A1 background: 1 to 7 carriers among the cases and 0 to 3 among the controls."""
    cases, ctrl = np.flatnonzero(y == 1), np.flatnonzero(y == 0)
    out = []
    for nc in range(1, 8):
        for nk in range(4):
            c = np.full(n, 3, np.uint8)
            c[np.concatenate([rng.choice(cases, nc, replace=False), rng.choice(ctrl, nk, replace=False)])] = 2
            out.append(c)
    return np.array(out)


@pytest.mark.parametrize("seed", [0, 2, 13])
def test_reference_against_scipy_minimize(seed):
    """The converged reference and the mirror's BETA / SE against BFGS on the negative log-likelihood of the raw design
    [1, covar, g] (gradient and Hessian inverse at the optimum), to 1e-6; the seeds include step-halving variants."""
    rng = np.random.default_rng(seed)
    n = 300
    code = grm_ref.balding_nichols(rng, n, 30, miss=0.02)
    g = np.where(code == 0, 2, np.where(code == 2, 1, 0))
    cov = rng.normal(size=(n, 2))
    y = (rng.random(n) < 1 / (1 + np.exp(-(-2.2 + 0.5 * cov[:, 0] + 0.8 * g[7])))).astype(float)
    code = np.concatenate([code, _rare_rows(rng, y, n)])
    rows = grm_ref.pack(code)
    halvings = []
    got, err, passes = ref.mirror(rows, n, y, cov, halvings=halvings)
    assert max(halvings) > 0                                     # a step-halving variant is present
    want = ref.converged(rows, n, y, cov)
    gd, called = ref.dosages(rows, n)
    checked = 0
    for v in np.flatnonzero(err == 0):
        A = called[v]
        X = np.concatenate([np.ones((A.sum(), 1)), cov[A], gd[v, A][:, None]], axis=1)

        def nll(t):
            eta = X @ t
            return float(np.sum(np.logaddexp(0.0, eta) - y[A] * eta))

        def grad(t):
            return X.T @ (1 / (1 + np.exp(-(X @ t))) - y[A])
        res = scipy.optimize.minimize(nll, np.zeros(X.shape[1]), jac=grad, method="BFGS",
                                      options={"gtol": 1e-10, "maxiter": 10000})
        t = res.x
        mu = 1 / (1 + np.exp(-(X @ t)))
        se = np.sqrt(np.linalg.inv(X.T @ ((mu * (1 - mu))[:, None] * X))[-1, -1])
        for stats in (want, got):
            assert abs(stats[v, 2] - t[-1]) <= 1e-6 * max(abs(t[-1]), se), (v, stats[v, 2], t[-1])
            assert abs(stats[v, 3] - se) <= 1e-6 * se, (v, stats[v, 3], se)
        checked += 1
    assert checked >= 40
    assert np.all(want[err == 0, 5] == 2 * scipy.stats.norm.sf(np.abs(want[err == 0, 4])))
    # separated rows (carriers among the cases only) do not converge
    sep = np.arange(30, 30 + 28)[np.arange(28) % 4 == 0]
    assert np.all(err[sep] == ref.CONVERGE_FAIL) and np.all(passes[sep] == 25)


def test_mirror_counted_allele_symmetry():
    rng = np.random.default_rng(3)
    n = 200
    code = grm_ref.balding_nichols(rng, n, 40, miss=0.05)
    y = (rng.random(n) < 0.3).astype(float)
    cov = rng.normal(size=(n, 1))
    a, ea, pa = ref.mirror(grm_ref.pack(code), n, y, cov, counted=1)
    b, eb, pb = ref.mirror(grm_ref.pack(code), n, y, cov, counted=2)
    assert np.array_equal(ea, eb) and np.array_equal(pa, pb)
    ok = ea == 0
    assert np.allclose(a[ok, 2], -b[ok, 2], rtol=1e-12, atol=0) and np.allclose(a[ok, 3], b[ok, 3], rtol=1e-12)


# ---- coding and refusals -----------------------------------------------------------------------------------------------
def test_case_control_coding():
    ids = [("F", "a"), (None, "b"), ("F", "c"), ("F", "d"), ("F", "e")]
    got = variants_pca.case_control_coding(np.array([1.0, 2.0, 0.0, np.nan, 2.0]), ids, "D")
    assert np.array_equal(got, [0.0, 1.0, np.nan, np.nan, 1.0], equal_nan=True)
    with pytest.raises(ValueError, match=r"phenotype D of sample b is 3.0; case/control phenotypes are 1 \(control\), "
                                         r"2 \(case\), or 0, -9, NA or nan \(missing\)"):
        variants_pca.case_control_coding(np.array([1.0, 3.0]), ids[:2], "D")
    with pytest.raises(ValueError, match="of sample F a is 0.5"):
        variants_pca.case_control_coding(np.array([0.5]), ids[:1], "D")


def test_refusals_before_any_context(tmp_path, no_context):
    prefix, fam, _ = _fileset(tmp_path)
    cc = _cc(fam)
    ph = _pheno_file(tmp_path, fam, cc, "D")
    base = ["--bed-path", prefix, "--output-path", str(tmp_path / "P")]
    bad = cc.copy()
    bad[7] = 3.0
    for argv, what in (
            (base + ["--glm-logistic", "--pheno", ph], "--pheno is read by --glm: give --glm"),
            (base + ["--glm-logistic"], "--glm-logistic is a mode of --glm: give --glm"),
            (base + ["--glm", "--glm-logistic"], "give --pheno FILE"),
            (base + ["--glm", "--glm-logistic", "--pheno", _pheno_file(tmp_path, fam, bad, "E")],
             f"phenotype E of sample {fam[7][0]} {fam[7][1]} is 3.0"),
            (base + ["--glm", "--glm-logistic", "--pheno", ph, "--num-pc", "32"], "at most 32 covariates.*make 33"),
            # --glm alone still refuses a case/control trait, and now names the flag
            (base + ["--glm", "--pheno", ph], "case/control traits need logistic regression: add --glm-logistic")):
        with pytest.raises(ValueError, match=what):
            variants_pca.main(argv)


def test_refusals_after_sample_qc(tmp_path, double):
    prefix, fam, _ = _fileset(tmp_path, n=12)
    cc = np.where(np.arange(12) < 3, 2.0, 1.0)                   # the cases are the first three samples
    (tmp_path / "keep.id").write_text("".join(f"{f} {i}\n" for f, i in fam[3:]))
    with pytest.raises(ValueError, match=r"--glm-logistic: phenotype T has 0 cases and 9 controls among the 9 samples "
                                         "with a phenotype and every covariate; a logistic test needs both"):
        variants_pca.main(["--bed-path", prefix, "--grm", "--keep", str(tmp_path / "keep.id"), "--glm",
                           "--glm-logistic", "--pheno", _pheno_file(tmp_path, fam, cc), "--output-path",
                           str(tmp_path / "P")])
    missing = np.where(np.arange(12) < 8, 0.0, cc)               # 0 is missing: four samples remain
    with pytest.raises(ValueError, match="4 of 12 samples have a phenotype and every covariate; 3 covariates .* 5"):
        variants_pca.main(["--bed-path", prefix, "--grm", "--glm", "--glm-logistic", "--pheno",
                           _pheno_file(tmp_path, fam, missing), "--output-path", str(tmp_path / "P")])
    assert all(nat.G is None for nat in double)                 # refused before the GRM


# ---- output ------------------------------------------------------------------------------------------------------------
def _numbers(rows):
    """OBS_CT, A1_FREQ, log(OR), LOG(OR)_SE, Z_STAT, P of the file's rows."""
    x = np.array([[np.nan if v == "NA" else float(v) for v in (r[8], r[6], r[9], r[10], r[11], r[12])] for r in rows])
    x[:, 2] = np.log(x[:, 2])
    return x


def test_write_format_numbers(tmp_path):
    b = plink.BimRecord("3", "rs9", 77, "T", "C")
    path = str(tmp_path / "x.glm.logistic")
    st = np.array([[10, 0.15, 0.5, 0.2, 2.5, 0.012419330651552318], [3, np.nan, np.nan, np.nan, np.nan, np.nan],
                   [40, 0.25, np.nan, np.nan, np.nan, np.nan]])
    variants_pca.write_glm_logistic(path, [b, b, b], 1, st, np.array([0, 1, 5]))
    lines = open(path).read().splitlines()
    assert lines[0] == "#CHROM\tPOS\tID\tREF\tALT\tA1\tA1_FREQ\tTEST\tOBS_CT\tOR\tLOG(OR)_SE\tZ_STAT\tP\tERRCODE"
    assert lines[1] == f"3\t77\trs9\tC\tT\tT\t0.15\tADD\t10\t{float(np.exp(0.5))!r}\t0.2\t2.5\t0.012419330651552318\t."
    assert lines[2] == "3\t77\trs9\tC\tT\tT\tNA\tADD\t3\tNA\tNA\tNA\tNA\tTOO_FEW_OBS"
    assert lines[3] == "3\t77\trs9\tC\tT\tT\t0.25\tADD\t40\tNA\tNA\tNA\tNA\tLOGISTIC_CONVERGE_FAIL"
    assert native.GLM_ERRCODES[5] == "LOGISTIC_CONVERGE_FAIL"


def _check_file(path, want, werr, bim):
    _, got = _read(path)
    assert [r[:6] for r in got] == [[b.contig, str(b.position), b.id, b.a2, b.a1, b.a1] for b in bim]
    assert all(r[7] == "ADD" for r in got)
    assert [r[13] for r in got] == [ref.ERRCODES[e] for e in werr]
    x = _numbers(got)
    assert np.array_equal(x[:, [0, 1, 3, 4, 5]], want[:, [0, 1, 3, 4, 5]], equal_nan=True)
    assert np.allclose(x[:, 2], want[:, 2], rtol=1e-13, atol=1e-15, equal_nan=True)   # log(exp(BETA))


@pytest.mark.parametrize("extra", [[], ["--keep", "keep"]])
def test_grm_run_end_to_end(tmp_path, capsys, double, extra):
    prefix, fam, _ = _fileset(tmp_path)
    cc = _cc(fam)
    cc[[2, 9]] = [0.0, -9.0]                                     # missing by code
    ph = _pheno_file(tmp_path, fam, cc)
    cov = tmp_path / "cov.txt"
    z = np.random.default_rng(4).normal(size=len(fam))
    cov.write_text("#FID IID AGE\n" + "".join(f"{f} {i} {'NA' if k == 11 else repr(float(z[k]))}\n"
                                              for k, (f, i) in enumerate(fam)))
    if extra:
        (tmp_path / "keep.id").write_text("".join(f"{f} {i}\n" for f, i in fam[4:]))
        extra = ["--keep", str(tmp_path / "keep.id")]
    P = str(tmp_path / "P")
    variants_pca.main(["--bed-path", prefix, "--grm", "--num-pc", "3", "--glm", "--glm-logistic", "--pheno", ph,
                       "--covar", str(cov), "--output-path", P] + extra)
    out = capsys.readouterr().out
    lines = open(P + ".eigenvec").read().splitlines()[1:]
    kept = np.array([fam.index(tuple(ln.split("\t")[:2])) for ln in lines])
    ev = np.array([[float(x) for x in ln.split("\t")[2:]] for ln in lines])
    bed = plink.BedFile(prefix)
    rows = grm_ref.pack(codes(bed.rows(0, bed.n_variants), len(fam))[:, kept])
    y = np.where(cc == 2.0, 1.0, np.where(cc == 1.0, 0.0, np.nan))[kept]
    zk = z[kept].copy()
    zk[kept == 11] = np.nan
    want, werr, _ = ref.mirror(rows, len(kept), y, np.concatenate([ev, zk[:, None]], axis=1))
    _check_file(P + ".T.glm.logistic", want, werr, plink.read_bim(prefix))
    reg = np.isfinite(y) & np.isfinite(zk)
    cases = int(np.count_nonzero(y[reg] == 1))
    lam = variants_pca.lambda_gc(want, werr)
    assert (f"GLM logistic: T on {reg.sum()} of {len(kept)} samples ({cases} cases, {reg.sum() - cases} controls, "
            f"{len(kept) - reg.sum()} without a phenotype or covariate), 5 covariates (intercept, 3 PCs, 1 from {cov}); "
            f"120 variants tested, {int(np.count_nonzero(werr))} with an ERRCODE; lambda_GC = {lam!r}.") in out
    assert werr[5] == 2                                          # the monomorphic variant
    assert double[-1].glm_calls == [120]


def test_projection_run(tmp_path, capsys, double):
    prefix, fam, _ = _fileset(tmp_path)
    npz = str(tmp_path / "r.npz")
    variants_pca.main(["--bed-path", prefix, "--grm", "--num-pc", "2", "--save-grm-loadings", npz])
    study, fam2, _ = _fileset(tmp_path / ".." / tmp_path.name, n=30, seed=3)
    cc = _cc(fam2, seed=5, rate=0.4)
    P = str(tmp_path / "Q")
    variants_pca.main(["--bed-path", study, "--project-loadings", npz, "--glm", "--glm-logistic", "--pheno",
                       _pheno_file(tmp_path, fam2, cc, "Z"), "--output-path", P])
    out = capsys.readouterr().out
    ev = np.array([[float(x) for x in ln.split("\t")[2:]] for ln in open(P + ".eigenvec").read().splitlines()[1:]])
    want, werr, _ = ref.mirror(plink.BedFile(study).rows(0, 120), 30, (cc == 2.0).astype(float), ev)
    _check_file(P + ".Z.glm.logistic", want, werr, plink.read_bim(study))
    assert "3 covariates (intercept, 2 PCs); 120 variants tested" in out


def test_king_cutoff_run_end_to_end(tmp_path, capsys, monkeypatch):
    made = []

    def _native(self, n):
        if self._nat is None:
            self._nat = KingLogDouble(n)
            made.append(self._nat)
        return self._nat
    monkeypatch.setattr(VariantsPcaDriver, "_native", _native)
    prefix, fam, _ = _fileset(tmp_path)
    cc = _cc(fam, seed=2, rate=0.4)
    cc[4] = np.nan
    P = str(tmp_path / "P")
    variants_pca.main(["--bed-path", prefix, "--king-cutoff", "0.177", "--num-pc", "3", "--glm", "--glm-logistic",
                       "--pheno", _pheno_file(tmp_path, fam, cc, missing={4}), "--output-path", P])
    nat = made[0]
    y = np.where(cc == 2.0, 1.0, np.where(cc == 1.0, 0.0, np.nan))
    want, werr, _ = ref.mirror(plink.BedFile(prefix).rows(0, 120), len(fam), y, nat.vecs)
    _check_file(P + ".T.glm.logistic", want, werr, plink.read_bim(prefix))
    assert f"GLM logistic: T on {len(fam) - 1} of {len(fam)} samples" in capsys.readouterr().out


# ---- the stratification the PCs remove -----------------------------------------------------------------------------------
def test_pcs_remove_the_stratification():
    """test_glm_cpu's seeded cohort (600 samples of 3 populations, 4000 variants, 1 % missing calls) with a case
    probability of 0.2, 0.35 and 0.5 by population and no causal variant.  The seeded run gives lambda_GC 2.94 with the
    intercept alone and 1.07 with two PCs; the bounds are > 2 and [0.9, 1.1]."""
    rng = np.random.default_rng(7)
    n = 600
    code = grm_ref.balding_nichols(rng, n, 4000, pops=3, miss=0.01)
    pop = np.repeat(np.arange(3), _pop_sizes(n))
    y = (rng.random(n) < np.array([0.2, 0.35, 0.5])[pop]).astype(float)
    rows = grm_ref.pack(code)
    G, M, Z = grm_ref.grm(rows, n)
    pcs = grm_ref.Pcs(Z, 2).U
    sub = rows[::4]                                              # 1000 of the variants keep the reference quick
    plain = variants_pca.lambda_gc(*ref.mirror(sub, n, y)[:2])
    adjusted = variants_pca.lambda_gc(*ref.mirror(sub, n, y, pcs)[:2])
    assert plain > 2.0
    assert 0.9 <= adjusted <= 1.1
