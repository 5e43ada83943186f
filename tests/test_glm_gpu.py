"""Linear association tests on the GPU (vpca_glm_begin / vpca_glm_linear_bed; DESIGN.md 15): BETA, SE and T_STAT against
per-variant lstsq on the complete cases over sample counts at the kernels' tile edges, covariate counts from 1 to 32 and
missing rates up to 95 %, OBS_CT, A1_FREQ and ERRCODE exactly, P against scipy at the kernel's own T and df, the bits
across calls, chunk caps, strides, runs and counted alleles, the state rules and refusals, and the driver end to end."""
import re

import numpy as np
import pytest
import scipy.stats

import glm_ref
import grm_ref
from qc_ref import counts as qc_counts
from spark_examples_b200 import native, plink, variants_pca

pytestmark = pytest.mark.gpu

VIF_OK = 1e3   # BETA, SE and T_STAT are compared where the dosage's variance inflation factor is below this


def _bits(a):
    return np.ascontiguousarray(a, np.float64).view(np.int64)


def _cohort(seed, n, nv, q, miss, excluded=0.05):
    """(rows, pheno, covar): Balding-Nichols codes with per-row missing rates `miss` (a list cycled over the rows), a
    monomorphic, an all-missing and a one-called row at the front; q - 1 covariates (the first two PC-like, the rest
    noise), NaN phenotypes for `excluded` of the samples; row 3 is the dosage of covariate 1 when q > 1."""
    rng = np.random.default_rng(seed)
    code = grm_ref.balding_nichols(rng, n, nv)
    for v in range(nv):
        rate = miss[v % len(miss)]
        if rate:
            code[v, rng.random(n) < rate] = 1
    code[0] = 0
    code[1] = 1
    code[2] = 1
    code[2, 0] = 2
    pop = np.repeat(np.arange(3), _pop_sizes(n))
    pheno = np.array([0.0, 0.5, 1.0])[pop] + rng.normal(size=n)
    pheno[rng.random(n) < excluded] = np.nan
    covar = rng.normal(size=(n, q - 1))
    if q > 1 and nv > 3 and n >= 40:
        code[3, code[3] == 1] = 2   # row 3 fully called, and its dosage is covariate 1
        covar[:, 0] = glm_ref.dosages(grm_ref.pack(code[3:4]), n)[0][0]
    return grm_ref.pack(code), pheno, covar


def _pop_sizes(n, pops=3):
    share = 1.12 ** np.arange(pops)
    sizes = np.floor(n * share / share.sum()).astype(np.int64)
    sizes[np.argsort(-(n * share / share.sum() - sizes))[: n - sizes.sum()]] += 1
    return sizes


def _vif(rows, n, pheno, covar, counted=1):
    """VIF of the dosage over each variant's complete cases (inf where undefined)."""
    g, called = glm_ref.dosages(rows, n, counted)
    reg = glm_ref.regression_samples(pheno, covar)
    C = np.concatenate([np.ones((n, 1)), covar], axis=1)
    out = np.full(g.shape[0], np.inf)
    for v in range(g.shape[0]):
        A = reg & called[v]
        if A.sum() <= C.shape[1] + 1:
            continue
        ga = g[v, A]
        css = ((ga - ga.mean()) ** 2).sum()
        s = ((ga - C[A] @ np.linalg.lstsq(C[A], ga, rcond=None)[0]) ** 2).sum()
        out[v] = css / s if s > 0 else np.inf
    return out


def check(got, gerr, want, werr, vif, note=""):
    assert np.array_equal(gerr, werr), (note, np.flatnonzero(gerr != werr), gerr[gerr != werr], werr[gerr != werr])
    assert np.array_equal(got[:, 0], want[:, 0]), note
    assert np.array_equal(np.isnan(got[:, 1]), np.isnan(want[:, 1])), note
    assert np.array_equal(_bits(got[~np.isnan(got[:, 1]), 1]), _bits(want[~np.isnan(want[:, 1]), 1])), note
    ok = werr == 0
    assert np.all(np.isnan(got[~ok, 2:])), note
    assert np.all(np.isfinite(got[ok, 2:])), note
    assert np.all(np.isfinite(got[:, 0])) and np.all(np.isfinite(got[got[:, 0] > 0, 1])), note
    cmp = ok & (vif < VIF_OK)
    b, se, t = got[cmp, 2], got[cmp, 3], got[cmp, 4]
    wb, wse, wt = want[cmp, 2], want[cmp, 3], want[cmp, 4]
    # BETA's error scales with its standard error (beta near 0 carries no relative precision), T_STAT's with max(|T|, 1)
    assert np.all(np.abs(b - wb) <= 1e-9 * np.maximum(np.abs(wb), wse)), (note, np.max(np.abs(b - wb) / wse))
    assert np.all(np.abs(se - wse) <= 1e-9 * wse), (note, np.max(np.abs(se - wse) / wse))
    assert np.all(np.abs(t - wt) <= 1e-9 * np.maximum(np.abs(wt), 1.0)), note


def check_p_df(stats, q, note=""):
    """P within 1e-10 relative of 2 t.sf(|T_STAT|, df) at the kernel's own T_STAT and df = OBS_CT - q - 1, for P >= 1e-300."""
    df = stats[:, 0] - q - 1
    want = 2.0 * scipy.stats.t.sf(np.abs(stats[:, 4]), df)
    big = want >= 1e-300
    assert np.all(np.abs(stats[big, 5] - want[big]) <= 1e-10 * want[big]), \
        (note, np.max(np.abs(stats[big, 5] - want[big]) / want[big]))
    assert np.all(stats[~big, 5] <= 1e-290), note


CASES = [   # (n, q, missing rates)
    (3, 1, [0.0]), (4, 2, [0.0]), (13, 11, [0.0]), (34, 32, [0.0]), (40, 17, [0.0, 0.01]),
    (127, 2, [0.0, 0.01, 0.3, 0.95]), (128, 11, [0.0, 0.01, 0.3, 0.95]), (129, 17, [0.0, 0.01, 0.3, 0.95]),
    (255, 32, [0.01, 0.3]), (256, 1, [0.0, 0.3]), (257, 11, [0.01, 0.95]),
    (511, 2, [0.3]), (513, 32, [0.0, 0.01]), (2504, 11, [0.0, 0.01, 0.3, 0.95]), (2504, 32, [0.01]),
]


@pytest.mark.parametrize("n,q,miss", CASES)
def test_against_lstsq(n, q, miss):
    nv = 257 if n < 1000 else 300   # one more than a 256-variant CTA of the sums
    rows, pheno, covar = _cohort(n * 100 + q, n, nv, q, miss, excluded=0.0 if n < q + 8 else 0.05)
    with native.NativePca(max(n, 2), device=0) as nat:
        used = nat.glmBegin(pheno, covar)
        got, gerr = nat.glmLinearBed(rows)
    want, werr = glm_ref.linear(rows, n, pheno, covar)
    assert used == int(glm_ref.regression_samples(pheno, covar).sum())
    check(got, gerr, want, werr, _vif(rows, n, pheno, covar), f"n={n} q={q}")
    check_p_df(got[gerr == 0], q, f"n={n} q={q}")
    assert gerr[0] == 2 and gerr[1] == 1                     # monomorphic, all missing
    if q > 1 and n >= 40:
        assert gerr[3] == 3                                  # the dosage is a covariate
    if n == q + 2:
        assert np.any((gerr == 0) & (got[:, 0] == q + 2))    # df = 1 is tested


def test_large_cohort_p_values():
    n, q = 21845, 11
    rows, pheno, covar = _cohort(5, n, 40, q, [0.0, 0.01, 0.3])
    with native.NativePca(n, device=0) as nat:
        nat.glmBegin(pheno, covar)
        got, gerr = nat.glmLinearBed(rows)
    want, werr = glm_ref.linear(rows, n, pheno, covar)
    check(got, gerr, want, werr, _vif(rows, n, pheno, covar), "n=21845")
    check_p_df(got[gerr == 0], q, "n=21845")


def test_p_values_over_df_and_t():
    """A phenotype equal to a dosage plus a little noise drives T_STAT far out; df from 1 up."""
    rng = np.random.default_rng(3)
    for n, noise in ((4, 1.0), (10, 0.5), (200, 0.05), (3000, 0.02), (3000, 1.0)):
        code = grm_ref.balding_nichols(rng, n, 64)
        rows = grm_ref.pack(code)
        g, _ = glm_ref.dosages(rows, n)
        pheno = g[5] + noise * rng.normal(size=n)
        with native.NativePca(n, device=0) as nat:
            nat.glmBegin(pheno)
            got, gerr = nat.glmLinearBed(rows)
        want, werr = glm_ref.linear(rows, n, pheno)
        assert np.array_equal(gerr, werr)
        check_p_df(got[gerr == 0], 1, f"n={n}")
        assert np.allclose(got[gerr == 0, 4], want[werr == 0, 4], rtol=1e-8)


def test_p_values_at_small_t_and_large_df():
    """|T_STAT| from 1e-3 down to 1e-6 at df near 21 845: there 1 - x = T^2 / (df + T^2) is below 1e-12, so computing it
    as 1 - x by subtraction would move P by more than 1e-9 relative.  The phenotype of each call is noise with its
    component along one variant's dosage (after the covariates) replaced by a tiny multiple of it."""
    n, q = 21845, 3
    rng = np.random.default_rng(17)
    code = grm_ref.balding_nichols(rng, n, 8)
    rows = grm_ref.pack(code)
    g, _ = glm_ref.dosages(rows, n)
    C = np.concatenate([np.ones((n, 1)), rng.normal(size=(n, q - 1))], axis=1)
    y0 = rng.normal(size=n)
    with native.NativePca(n, device=0) as nat:
        for j, target in enumerate((1e-3, 1e-4, 1e-5, 1e-6)):
            gt = g[j] - C @ np.linalg.lstsq(C, g[j], rcond=None)[0]
            y = y0 - (y0 @ gt) / (gt @ gt) * gt + target / np.sqrt(gt @ gt) * gt
            nat.glmBegin(y, C[:, 1:])
            got, gerr = nat.glmLinearBed(rows)
            assert gerr[j] == 0 and abs(got[j, 4]) < 10 * target and got[j, 0] - q - 1 > 21000, (j, got[j])
            check_p_df(got[gerr == 0], q, f"T near {target}")


def test_covariates_collinear_over_the_called_samples():
    """A covariate that is an indicator of three samples is collinear with the intercept at a variant where those three
    are not called: VIF_INFINITE there (a Cholesky pivot of Q_A^T Q_A below 1e-10), as in the reference; a fit
    elsewhere."""
    n = 200
    rows, pheno, covar = _cohort(21, n, 60, 3, [0.0], excluded=0.0)
    code = np.stack([(rows[:, i // 4] >> (2 * (i % 4))) & 3 for i in range(n)], axis=1)
    covar[:, 0] = 0.0
    covar[[10, 20, 30], 0] = 1.0
    code[6:12, [10, 20, 30]] = 1                             # rows 6 .. 11: the indicator's samples missing
    rows = grm_ref.pack(code)
    with native.NativePca(n, device=0) as nat:
        nat.glmBegin(pheno, covar)
        got, gerr = nat.glmLinearBed(rows)
    want, werr = glm_ref.linear(rows, n, pheno, covar)
    check(got, gerr, want, werr, _vif(rows, n, pheno, covar), "indicator")
    assert np.all(gerr[6:12] == 3)
    assert np.all(gerr[12:] != 3)


def test_bits_across_calls_strides_chunks_and_runs():
    n, q = 301, 5
    rows, pheno, covar = _cohort(7, n, 700, q, [0.0, 0.01, 0.3])
    rng = np.random.default_rng(8)
    wide = rng.integers(0, 256, (rows.shape[0], rows.shape[1] + 13), dtype=np.uint8)
    wide[:, :rows.shape[1]] = rows
    wide[:, rows.shape[1] - 1] |= np.uint8(0b11111100)   # garbage in the padding bits of the last byte (n % 4 = 1)
    with native.NativePca(n, device=0) as nat:
        nat.glmBegin(pheno, covar)
        whole, e0 = nat.glmLinearBed(rows)
        again, e1 = nat.glmLinearBed(rows)
        strided, e2 = nat.glmLinearBed(wide)
        pieces = [nat.glmLinearBed(rows[a:b]) for a, b in ((0, 1), (1, 2), (2, 255), (255, 699), (699, 700))]
        a2, e3 = nat.glmLinearBed(rows, counted=2)
    for got, err in ((again, e1), (strided, e2), (np.concatenate([p[0] for p in pieces]),
                                                   np.concatenate([p[1] for p in pieces]))):
        assert np.array_equal(_bits(got), _bits(whole)) and np.array_equal(err, e0)
    ok = e0 == 0
    assert np.array_equal(e3, e0)
    assert np.array_equal(a2[:, 0], whole[:, 0])
    assert np.allclose(a2[:, 1], 1.0 - whole[:, 1], rtol=0, atol=1e-15, equal_nan=True)
    assert np.allclose(a2[ok, 2], -whole[ok, 2], rtol=1e-10)
    assert np.allclose(a2[ok, 3], whole[ok, 3], rtol=1e-10)
    assert np.allclose(a2[ok, 4], -whole[ok, 4], rtol=1e-10)
    assert np.allclose(a2[ok, 5], whole[ok, 5], rtol=1e-8)


def test_chunk_cap():
    """More rows than one 2^20-row chunk: the same bits as the rows split into two calls elsewhere."""
    n = 9
    rng = np.random.default_rng(11)
    nv = (1 << 20) + 37
    code = rng.integers(0, 4, (nv, n), dtype=np.uint8)
    rows = grm_ref.pack(code)
    pheno = rng.normal(size=n)
    with native.NativePca(n, device=0) as nat:
        nat.glmBegin(pheno, rng.normal(size=(n, 2)))
        whole, e0 = nat.glmLinearBed(rows)
        a, ea = nat.glmLinearBed(rows[:1000])
        b, eb = nat.glmLinearBed(rows[1000:])
    assert np.array_equal(_bits(whole), _bits(np.concatenate([a, b])))
    assert np.array_equal(e0, np.concatenate([ea, eb]))


def test_state_and_refusals():
    n = 50
    rows, pheno, covar = _cohort(9, n, 20, 3, [0.0])
    with native.NativePca(n, device=0) as nat:
        with pytest.raises(native.VpcaError) as e:
            nat.glmLinearBed(rows)
        assert e.value.code == native.VPCA_ERR_STATE
        for y, c, what in ((np.where(np.arange(n) == 3, np.inf, pheno), covar, "infinite"),
                           (pheno, np.where(np.arange(n)[:, None] == 4, -np.inf, covar), "infinite"),
                           (pheno, np.zeros((n, 32)), "exceed"),
                           (np.where(np.arange(n) < 4, 1.0, np.nan), covar, "regression samples"),
                           (np.ones(n), covar, "constant"),
                           (pheno, np.stack([covar[:, 0], 2.0 * covar[:, 0] + 1.0], axis=1), "covariate 2 is collinear")):
            with pytest.raises(native.VpcaError, match=what) as e:
                nat.glmBegin(y, c)
            assert e.value.code == native.VPCA_ERR_BAD_ARG
            with pytest.raises(native.VpcaError) as e:   # a refused begin leaves no state
                nat.glmLinearBed(rows)
            assert e.value.code == native.VPCA_ERR_STATE
        nat.glmBegin(pheno, covar)
        nat.glmLinearBed(rows)
        with pytest.raises(native.VpcaError) as e:
            nat.glmLinearBed(rows, counted=3)
        assert e.value.code == native.VPCA_ERR_BAD_ARG
        nat.reset()
        with pytest.raises(native.VpcaError) as e:
            nat.glmLinearBed(rows)
        assert e.value.code == native.VPCA_ERR_STATE


def test_leaves_the_grm_pca_and_loadings_alone():
    n, nv = 120, 400
    code = grm_ref.balding_nichols(np.random.default_rng(12), n, nv, miss=0.02)
    rows = grm_ref.pack(code)
    pheno = np.random.default_rng(13).normal(size=n)

    def run(with_glm):
        with native.NativePca(n, device=0) as nat:
            nat.grmBed(rows)
            nat.grmFinalize()
            if with_glm:
                nat.glmBegin(pheno)
                nat.glmLinearBed(rows)
            G = nat.getGrm()
            vecs, evals = nat.computePcaGrm(3)
            w, tab = nat.grmLoadingsBed(3, rows)
            return G, vecs, evals, w, tab
    for a, b in zip(run(False), run(True)):
        assert np.array_equal(_bits(a), _bits(b))


# ---- the driver end to end -----------------------------------------------------------------------------------------------
def _driver_cohort(tmp_path, n=600, nv=4000):
    """The seeded stratified cohort: 3 populations, phenotype mean (0, 0.5, 1) plus N(0, 1) noise, no causal variant."""
    rng = np.random.default_rng(7)
    code = grm_ref.balding_nichols(rng, n, nv, pops=3, miss=0.01)
    d = np.where(code == 0, 2, np.where(code == 2, 1, np.where(code == 3, 0, -1))).T
    prefix = str(tmp_path / "c")
    plink.write_fileset(prefix, d, positions=1000 * np.arange(nv) + 1)
    pop = np.repeat(np.arange(3), _pop_sizes(n))
    y = np.array([0.0, 0.5, 1.0])[pop] + rng.normal(size=n)
    fam = plink.read_fam_ids(prefix)
    (tmp_path / "p.txt").write_text("#FID IID T\n" + "".join(f"{f} {i} {float(v)!r}\n" for (f, i), v in zip(fam, y)))
    return prefix, str(tmp_path / "p.txt"), y


def _read_glm(path):
    lines = open(path).read().splitlines()
    head = lines[0].split("\t")
    rows = [ln.split("\t") for ln in lines[1:]]
    return head, rows


@pytest.mark.parametrize("mode", ["grm", "carrier", "king"])
def test_driver_end_to_end(tmp_path, capsys, mode):
    prefix, pheno_file, y = _driver_cohort(tmp_path)
    P = str(tmp_path / "P")
    argv = ["--bed-path", prefix, "--maf", "0.01", "--ld-prune", "0.2", "--num-pc", "2", "--pheno", pheno_file, "--glm",
            "--output-path", P]
    if mode == "grm":
        argv.append("--grm")
    elif mode == "king":
        argv += ["--king-cutoff", "0.177"]
    variants_pca.main(argv)
    out = capsys.readouterr().out
    m = re.search(r"GLM linear: T on (\d+) of (\d+) samples .* (\d+) variants tested, (\d+) with an ERRCODE; "
                  r"lambda_GC = ([0-9.]+)\.", out)
    assert m, out
    lam = float(m.group(5))
    assert lam <= 1.1
    head, rows = _read_glm(P + ".T.glm.linear")
    assert head == ["#CHROM", "POS", "ID", "REF", "ALT", "A1", "A1_FREQ", "TEST", "OBS_CT", "BETA", "SE", "T_STAT", "P",
                    "ERRCODE"]
    # the reference with P.eigenvec as the covariates, over the variants that pass --maf (not only the pruned ones)
    bed = plink.BedFile(prefix)
    allrows = bed.rows(0, bed.n_variants)
    keep, _ = variants_pca.variant_qc_keep(qc_counts(allrows, len(y)), None, 0.01, None, None)
    assert len(rows) == int(keep.sum())
    bim = [b for b, k in zip(plink.read_bim(prefix), keep) if k]
    assert [r[2] for r in rows] == [b.id for b in bim]
    if mode == "grm":
        ev = [ln.split("\t") for ln in open(P + ".eigenvec").read().splitlines()[1:]]
        vecs = np.array([[float(x) for x in r[2:]] for r in ev])
        want, werr = glm_ref.linear(allrows[keep], len(y), y, vecs)
        got = np.array([[float("nan") if x == "NA" else float(x) for x in (r[8], r[6], r[9], r[10], r[11], r[12])]
                        for r in rows])
        gerr = np.array([glm_ref.ERRCODES.index(r[13]) for r in rows])
        check(got, gerr, want, werr, np.zeros(len(gerr)), "driver")
        assert abs(lam - glm_ref.lambda_gc(want, werr)) <= 1e-6
