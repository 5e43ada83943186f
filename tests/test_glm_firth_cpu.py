"""Firth-penalized logistic tests without a GPU (DESIGN.md 17): the mirror and the converged reference against
scipy.optimize on the penalized likelihood, the 2 x 2 closed form, the counted-allele symmetry of the mirror, the
--glm-firth refusals before any context is requested, and the .glm.logistic.hybrid / .glm.firth files and summary lines
through a numpy double of glmFirthBed on the --grm, --king-cutoff and --project-loadings paths."""
import numpy as np
import pytest
import scipy.optimize

import glm_firth_ref as ref
import glm_logistic_ref as lref
import grm_ref
from qc_ref import codes
from spark_examples_b200 import native, plink, variants_pca
from spark_examples_b200.variants_pca import VariantsPcaDriver
from test_glm_cpu import Double, KingGlmDouble, MissingDouble, _fileset, _pheno_file, _read
from test_glm_logistic_cpu import _cc


class FirthDouble(Double, lref.LogisticDouble, ref.FirthDouble):
    pass


class KingFirthDouble(KingGlmDouble, lref.LogisticDouble, ref.FirthDouble):
    pass


@pytest.fixture
def double(monkeypatch):
    made = []

    def _native(self, n):
        if self._nat is None:
            self._nat = FirthDouble(n)
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


# ---- the reference -----------------------------------------------------------------------------------------------------
def _rare_rows(rng, y, n):
    """Rows of A2 carriers on an A1 background: 0 to 3 carriers among the cases and 0 to 3 among the controls."""
    cases, ctrl = np.flatnonzero(y == 1), np.flatnonzero(y == 0)
    out = []
    for a in range(4):
        for b in range(4):
            c = np.full(n, 3, np.uint8)
            c[np.concatenate([rng.choice(cases, a, replace=False), rng.choice(ctrl, b, replace=False)])] = 2
            out.append(c)
    return np.array(out)


@pytest.mark.parametrize("seed,n,rate", [(0, 300, 0.3), (2, 400, 0.1), (13, 60, 0.5)])
def test_reference_against_scipy_minimize(seed, n, rate):
    """The mirror and the converged fit against BFGS on -l* of the raw design [1, covar, g] with gradient -U*, to 1e-6;
    the rows include singletons and carriers among the cases alone."""
    rng = np.random.default_rng(seed)
    code = grm_ref.balding_nichols(rng, n, 12, miss=0.02)
    cov = rng.normal(size=(n, 2))
    y = (rng.random(n) < rate).astype(float)
    y[:2] = [0.0, 1.0]
    code = np.concatenate([code, _rare_rows(rng, y, n)])
    rows = grm_ref.pack(code)
    got, err, passes, firth = ref.mirror(rows, n, y, cov)
    want = ref.converged(rows, n, y, cov)
    gd, called = ref.dosages(rows, n)
    checked = 0
    for v in np.flatnonzero(err == 0):
        A = called[v]
        X = np.concatenate([np.ones((A.sum(), 1)), cov[A], gd[v, A][:, None]], axis=1)
        res = scipy.optimize.minimize(lambda t: ref.penalized(X, y[A], t), np.zeros(X.shape[1]), jac=True,
                                      method="BFGS", options={"gtol": 1e-9, "maxiter": 20000})
        t = res.x
        _, _, H = lref.evaluate(X, y[A], t)
        se = np.sqrt(np.linalg.inv(H)[-1, -1])
        for stats in (want, got):
            assert abs(stats[v, 2] - t[-1]) <= 1e-6 * max(abs(t[-1]), se), (v, stats[v, 2], t[-1])
            assert abs(stats[v, 3] - se) <= 1e-6 * se, (v, stats[v, 3], se)
        checked += 1
    assert checked >= 20
    assert np.all(firth[err != 2] == 1)                           # every variant but the monomorphic ones is fitted
    assert np.all(err[12:] != ref.FIRTH_FAIL)                     # the separated rows converge


def test_closed_form_at_q_1():
    """The intercept and a binary dosage: BETA is log((a + 1/2)(d + 1/2) / ((b + 1/2)(c + 1/2))) of the 2 x 2 table,
    zero cells included."""
    for seed, n, rate in ((1, 60, 0.5), (4, 400, 0.1), (5, 2504, 0.02)):
        rng = np.random.default_rng(seed)
        y = (rng.random(n) < rate).astype(float)
        y[:2] = [0.0, 1.0]
        rows = grm_ref.pack(_rare_rows(rng, y, n)[1:])            # without the all-A1 row (CONST_ALLELE)
        got, err, _, _ = ref.mirror(rows, n, y)
        g, _ = ref.dosages(rows, n)
        assert np.all(err == 0)
        for v in range(rows.shape[0]):
            a, b = np.sum(g[v][y == 1] != 0), np.sum(g[v][y == 0] != 0)
            c, d = np.sum(y == 1) - a, np.sum(y == 0) - b
            want = np.log((a + 0.5) * (d + 0.5) / ((b + 0.5) * (c + 0.5)))
            assert abs(got[v, 2] - want) <= 1e-7 * max(abs(want), got[v, 3]), (seed, v, got[v, 2], want)


def test_mirror_counted_allele_symmetry():
    rng = np.random.default_rng(3)
    n = 200
    y = (rng.random(n) < 0.2).astype(float)
    code = np.concatenate([grm_ref.balding_nichols(rng, n, 20, miss=0.05), _rare_rows(rng, y, n)])
    cov = rng.normal(size=(n, 1))
    for mode in (ref.FALLBACK, ref.ALWAYS):
        a, ea, pa, fa = ref.mirror(grm_ref.pack(code), n, y, cov, counted=1, mode=mode)
        b, eb, pb, fb = ref.mirror(grm_ref.pack(code), n, y, cov, counted=2, mode=mode)
        assert np.array_equal(ea, eb) and np.array_equal(pa, pb) and np.array_equal(fa, fb)
        ok = ea == 0
        assert np.allclose(a[ok, 2], -b[ok, 2], rtol=1e-10, atol=0) and np.allclose(a[ok, 3], b[ok, 3], rtol=1e-10)


def test_fallback_refits_what_the_plain_fit_cannot():
    rng = np.random.default_rng(9)
    n = 400
    y = (rng.random(n) < 0.1).astype(float)
    code = np.concatenate([grm_ref.balding_nichols(rng, n, 10), _rare_rows(rng, y, n)])
    rows = grm_ref.pack(code)
    ml, mlerr, mlpass = lref.mirror(rows, n, y)
    fb, fberr, fbpass, firth = ref.mirror(rows, n, y, mode=ref.FALLBACK)
    refit = (mlerr == ref.CONVERGE_FAIL) & (mlpass > 0)
    assert refit.sum() >= 3 and np.array_equal(firth == 1, refit)
    assert np.array_equal(fb[~refit], ml[~refit], equal_nan=True) and np.array_equal(fbpass[~refit], mlpass[~refit])
    al, alerr, alpass, _ = ref.mirror(rows, n, y, mode=ref.ALWAYS)
    assert np.array_equal(fb[refit], al[refit]) and np.array_equal(fbpass[refit], alpass[refit])
    assert np.all(fberr[refit] == 0)


# ---- refusals ------------------------------------------------------------------------------------------------------------
def test_refusals_before_any_context(tmp_path, no_context):
    prefix, fam, _ = _fileset(tmp_path)
    ph = _pheno_file(tmp_path, fam, _cc(fam), "D")
    base = ["--bed-path", prefix, "--output-path", str(tmp_path / "P"), "--pheno", ph]
    for argv, what in (
            (base + ["--glm", "--glm-firth", "fallback"], "--glm-firth is a mode of the logistic test: give --glm "
                                                         "--glm-logistic"),
            (base[:4] + ["--glm-logistic", "--glm-firth", "always"], "--glm-logistic is a mode of --glm"),
            (base + ["--glm", "--glm-logistic", "--glm-firth", "sometimes"],
             "--glm-firth takes fallback or always, not 'sometimes'")):
        with pytest.raises(ValueError, match=what):
            variants_pca.main(argv)
    with pytest.raises(ValueError, match="--glm-firth is a mode of the logistic test"):
        variants_pca.main(["--bed-path", prefix, "--grm", "--glm-firth", "always"])


# ---- output ------------------------------------------------------------------------------------------------------------
def test_write_format():
    b = plink.BimRecord("3", "rs9", 77, "T", "C")
    st = np.array([[10, 0.15, 0.5, 0.2, 2.5, 0.012419330651552318], [40, 0.25, np.nan, np.nan, np.nan, np.nan]])
    import io
    import os
    import tempfile
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "x.glm.logistic.hybrid")
        variants_pca.write_glm_logistic(path, [b, b], 1, st, np.array([0, 6]), np.array([1, 0], np.uint8))
        lines = io.open(path).read().splitlines()
    assert lines[0] == "#CHROM\tPOS\tID\tREF\tALT\tA1\tA1_FREQ\tFIRTH?\tTEST\tOBS_CT\tOR\tLOG(OR)_SE\tZ_STAT\tP\tERRCODE"
    assert lines[1] == f"3\t77\trs9\tC\tT\tT\t0.15\tY\tADD\t10\t{float(np.exp(0.5))!r}\t0.2\t2.5\t0.012419330651552318\t."
    assert lines[2] == "3\t77\trs9\tC\tT\tT\t0.25\tN\tADD\t40\tNA\tNA\tNA\tNA\tFIRTH_CONVERGE_FAIL"
    assert native.GLM_ERRCODES[6] == "FIRTH_CONVERGE_FAIL" and ref.ERRCODES == native.GLM_ERRCODES


def _numbers(rows, off):
    x = np.array([[np.nan if v == "NA" else float(v) for v in (r[8 + off], r[6], r[9 + off], r[10 + off], r[11 + off],
                                                                r[12 + off])] for r in rows])
    x[:, 2] = np.log(x[:, 2])
    return x


def _check_file(path, want, werr, wfirth, bim, hybrid):
    header, got = _read(path)
    off = 1 if hybrid else 0
    assert header[7] == ("FIRTH?" if hybrid else "TEST")
    assert [r[:6] for r in got] == [[b.contig, str(b.position), b.id, b.a2, b.a1, b.a1] for b in bim]
    if hybrid:
        assert [r[7] for r in got] == ["Y" if f else "N" for f in wfirth]
    assert [r[13 + off] for r in got] == [ref.ERRCODES[e] for e in werr]
    x = _numbers(got, off)
    assert np.array_equal(x[:, [0, 1, 3, 4, 5]], want[:, [0, 1, 3, 4, 5]], equal_nan=True)
    assert np.allclose(x[:, 2], want[:, 2], rtol=1e-13, atol=1e-15, equal_nan=True)


def _rare_fileset(tmp_path, cc, seed=1, n_rare=12):
    """_fileset with rows 100 .. 100 + n_rare replaced by rare variants carried by cases (and a few controls)."""
    prefix, fam, _ = _fileset(tmp_path)
    bed = plink.BedFile(prefix)
    code = codes(bed.rows(0, bed.n_variants), len(fam))
    rng = np.random.default_rng(seed)
    cases, ctrl = np.flatnonzero(cc == 2.0), np.flatnonzero(cc == 1.0)
    for r in range(n_rare):
        code[100 + r] = 3
        code[100 + r, rng.choice(cases, 1 + r % 3, replace=False)] = 2
        if r % 4 == 3:
            code[100 + r, rng.choice(ctrl, 1, replace=False)] = 2
    d = np.where(code == 0, 2, np.where(code == 2, 1, np.where(code == 3, 0, -1))).T
    bim = plink.read_bim(prefix)
    plink.write_fileset(prefix, d, fam=fam, positions=[b.position for b in bim])
    return prefix, fam, code


@pytest.mark.parametrize("mode", ["fallback", "always"])
def test_grm_run_end_to_end(tmp_path, capsys, double, mode):
    _, fam, _ = _fileset(tmp_path)
    cc = _cc(fam, rate=0.3)
    prefix, fam, code = _rare_fileset(tmp_path, cc)
    ph = _pheno_file(tmp_path, fam, cc)
    P = str(tmp_path / "P")
    variants_pca.main(["--bed-path", prefix, "--grm", "--num-pc", "2", "--glm", "--glm-logistic", "--glm-firth", mode,
                       "--pheno", ph, "--output-path", P])
    out = capsys.readouterr().out
    ev = np.array([[float(x) for x in ln.split("\t")[2:]] for ln in open(P + ".eigenvec").read().splitlines()[1:]])
    y = np.where(cc == 2.0, 1.0, 0.0)
    m = ref.FALLBACK if mode == "fallback" else ref.ALWAYS
    want, werr, _, wfirth = ref.mirror(grm_ref.pack(code), len(fam), y, ev, mode=m)
    hybrid = mode == "fallback"
    _check_file(P + (".T.glm.logistic.hybrid" if hybrid else ".T.glm.firth"), want, werr, wfirth,
                plink.read_bim(prefix), hybrid)
    cases = int(np.count_nonzero(y == 1))
    lam = variants_pca.lambda_gc(want, werr)
    head = "GLM logistic" if hybrid else "GLM Firth"
    fitted = f", {int(wfirth.sum())} fitted by Firth regression" if hybrid else ""
    assert (f"{head}: T on {len(fam)} of {len(fam)} samples ({cases} cases, {len(fam) - cases} controls, 0 without a "
            f"phenotype or covariate), 3 covariates (intercept, 2 PCs); 120 variants tested, "
            f"{int(np.count_nonzero(werr))} with an ERRCODE{fitted}; lambda_GC = {lam!r}.") in out
    assert double[-1].firth_modes == [mode]
    if hybrid:
        assert wfirth.sum() >= 8


def test_fallback_rows_match_a_plain_run(tmp_path, capsys, double):
    """The FIRTH? N rows of the .hybrid file are the text of the .glm.logistic rows of a run without --glm-firth."""
    _, fam, _ = _fileset(tmp_path)
    cc = _cc(fam, rate=0.3)
    prefix, fam, _ = _rare_fileset(tmp_path, cc)
    ph = _pheno_file(tmp_path, fam, cc)
    argv = ["--bed-path", prefix, "--grm", "--num-pc", "2", "--glm", "--glm-logistic", "--pheno", ph]
    variants_pca.main(argv + ["--output-path", str(tmp_path / "A")])
    variants_pca.main(argv + ["--glm-firth", "fallback", "--output-path", str(tmp_path / "B")])
    plain = open(str(tmp_path / "A") + ".T.glm.logistic").read().splitlines()
    hyb = open(str(tmp_path / "B") + ".T.glm.logistic.hybrid").read().splitlines()
    assert len(plain) == len(hyb)
    n_rows = 0
    for a, b in zip(plain[1:], hyb[1:]):
        f = b.split("\t")
        if f[7] == "N":
            assert "\t".join(f[:7] + f[8:]) == a
            n_rows += 1
        else:
            assert a.split("\t")[13] == "LOGISTIC_CONVERGE_FAIL"
    assert 100 <= n_rows < 120
    assert not (tmp_path / "B.T.glm.logistic").exists()


def test_projection_run(tmp_path, capsys, double):
    prefix, fam, _ = _fileset(tmp_path)
    npz = str(tmp_path / "r.npz")
    variants_pca.main(["--bed-path", prefix, "--grm", "--num-pc", "2", "--save-grm-loadings", npz])
    study, fam2, _ = _fileset(tmp_path / ".." / tmp_path.name, n=30, seed=3)
    cc = _cc(fam2, seed=5, rate=0.4)
    P = str(tmp_path / "Q")
    variants_pca.main(["--bed-path", study, "--project-loadings", npz, "--glm", "--glm-logistic", "--glm-firth",
                       "always", "--pheno", _pheno_file(tmp_path, fam2, cc, "Z"), "--output-path", P])
    out = capsys.readouterr().out
    ev = np.array([[float(x) for x in ln.split("\t")[2:]] for ln in open(P + ".eigenvec").read().splitlines()[1:]])
    want, werr, _, wfirth = ref.mirror(plink.BedFile(study).rows(0, 120), 30, (cc == 2.0).astype(float), ev)
    _check_file(P + ".Z.glm.firth", want, werr, wfirth, plink.read_bim(study), False)
    assert "GLM Firth: Z on 30 of 30 samples" in out and "3 covariates (intercept, 2 PCs); 120 variants tested" in out


def test_king_cutoff_run_end_to_end(tmp_path, capsys, monkeypatch):
    made = []

    def _native(self, n):
        if self._nat is None:
            self._nat = KingFirthDouble(n)
            made.append(self._nat)
        return self._nat
    monkeypatch.setattr(VariantsPcaDriver, "_native", _native)
    _, fam, _ = _fileset(tmp_path)
    cc = _cc(fam, seed=2, rate=0.4)
    prefix, fam, code = _rare_fileset(tmp_path, cc)
    cc[4] = np.nan
    P = str(tmp_path / "P")
    variants_pca.main(["--bed-path", prefix, "--king-cutoff", "0.177", "--num-pc", "3", "--glm", "--glm-logistic",
                       "--glm-firth", "fallback", "--pheno", _pheno_file(tmp_path, fam, cc, missing={4}),
                       "--output-path", P])
    nat = made[0]
    y = np.where(cc == 2.0, 1.0, np.where(cc == 1.0, 0.0, np.nan))
    want, werr, _, wfirth = ref.mirror(grm_ref.pack(code), len(fam), y, nat.vecs, mode=ref.FALLBACK)
    _check_file(P + ".T.glm.logistic.hybrid", want, werr, wfirth, plink.read_bim(prefix), True)
    out = capsys.readouterr().out
    assert f"GLM logistic: T on {len(fam) - 1} of {len(fam)} samples" in out
    assert f", {int(wfirth.sum())} fitted by Firth regression; lambda_GC" in out
