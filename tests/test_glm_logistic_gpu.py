"""Logistic association tests on the GPU (vpca_glm_logistic_begin / vpca_glm_logistic_bed; DESIGN.md 16): BETA, SE and Z
against the fully converged per-variant fit on the complete cases, over sample counts at the kernel's tile and warp
edges, covariate counts from 1 to 32, missing rates up to 95 % and case rates of 50, 10 and 1 %; OBS_CT, A1_FREQ,
ERRCODE and the pass count exactly against the mirror of the kernel's iteration; separated and near-fixed variants; P
against scipy; the counted-allele symmetry and the bits across calls, chunk caps, strides, runs and neighbours; the
state rules and refusals; and the driver end to end."""
import re

import numpy as np
import pytest
import scipy.stats

import glm_logistic_ref as ref
import glm_ref
import grm_ref
from qc_ref import counts as qc_counts
from spark_examples_b200 import native, plink, variants_pca
from test_glm_gpu import _pop_sizes, _vif

pytestmark = pytest.mark.gpu

VIF_OK = 1e3      # BETA, SE and Z are compared where the dosage's variance inflation factor is below this
PASSES_OK = 20    # ... and the mirror converges within this many passes


def _bits(a):
    return np.ascontiguousarray(a, np.float64).view(np.int64)


def _cohort(seed, n, nv, q, miss, rate, excluded=0.05):
    """(rows, pheno 0/1/NaN, covar): Balding-Nichols codes with per-row missing rates `miss` (cycled over the rows), a
    monomorphic and an all-missing row at the front; q - 1 N(0, 1) covariates; a case probability of about `rate`,
    raised in the third population and by covariate 1 and the dosage of row 5; NaN phenotypes for `excluded` of the
    samples."""
    rng = np.random.default_rng(seed)
    code = grm_ref.balding_nichols(rng, n, nv)
    for v in range(nv):
        r = miss[v % len(miss)]
        if r:
            code[v, rng.random(n) < r] = 1
    code[0] = 0
    code[1] = 1
    pop = np.repeat(np.arange(3), _pop_sizes(n))
    covar = rng.normal(size=(n, q - 1))
    g5 = np.where(code[5 % nv] == 0, 2.0, np.where(code[5 % nv] == 2, 1.0, 0.0))
    eta = np.log(rate / (1 - rate)) + 0.4 * (pop == 2) + 0.3 * g5 + (0.3 * covar[:, 0] if q > 1 else 0.0)
    pheno = (rng.random(n) < 1 / (1 + np.exp(-eta))).astype(float)
    pheno[:2] = [0.0, 1.0]                                     # both classes present
    pheno[2:][rng.random(n - 2) < excluded] = np.nan
    return grm_ref.pack(code), pheno, covar


def check(got, gerr, gpass, rows, n, pheno, covar, counted=1, note=""):
    """ERRCODE, passes, OBS_CT and A1_FREQ exactly against the mirror; BETA, SE and Z against the converged fit where
    the VIF is below VIF_OK and the mirror converged within PASSES_OK passes; P against scipy at the kernel's Z."""
    want, werr, wpass = ref.mirror(rows, n, pheno, covar, counted=counted)
    assert np.array_equal(gerr, werr), (note, np.flatnonzero(gerr != werr), gerr[gerr != werr], werr[gerr != werr])
    assert np.array_equal(gpass, wpass), (note, np.flatnonzero(gpass != wpass), gpass[gpass != wpass],
                                          wpass[gpass != wpass])
    assert np.array_equal(got[:, 0], want[:, 0]), note
    assert np.array_equal(np.isnan(got[:, 1]), np.isnan(want[:, 1])), note
    assert np.array_equal(_bits(got[~np.isnan(got[:, 1]), 1]), _bits(want[~np.isnan(want[:, 1]), 1])), note
    ok = gerr == 0
    assert np.all(np.isnan(got[~ok, 2:])), note
    assert np.all(np.isfinite(got[ok, 2:])), note
    vif = _vif(rows, n, pheno, covar, counted)
    cmp = np.flatnonzero(ok & (vif < VIF_OK) & (wpass <= PASSES_OK))
    conv = ref.converged(rows, n, pheno, covar, counted, variants=cmp)
    b, se, z = got[cmp, 2], got[cmp, 3], got[cmp, 4]
    wb, wse, wz = conv[cmp, 2], conv[cmp, 3], conv[cmp, 4]
    assert np.all(np.isfinite(wb)), note
    assert np.all(np.abs(b - wb) <= 1e-7 * np.maximum(np.abs(wb), wse)), (note, np.max(np.abs(b - wb) / wse))
    assert np.all(np.abs(se - wse) <= 1e-7 * wse), (note, np.max(np.abs(se - wse) / wse))
    assert np.all(np.abs(z - wz) <= 1e-7 * np.maximum(np.abs(wz), 1.0)), note
    check_p(got[ok], note)
    return cmp.size


def check_p(stats, note=""):
    """P within 1e-12 relative of 2 norm.sf(|Z|) at the kernel's own Z for P >= 1e-300, and 0 past |Z| = 38.5."""
    want = 2.0 * scipy.stats.norm.sf(np.abs(stats[:, 4]))
    big = want >= 1e-300
    assert np.all(np.abs(stats[big, 5] - want[big]) <= 1e-12 * want[big]), \
        (note, np.max(np.abs(stats[big, 5] - want[big]) / want[big]))
    assert np.all(stats[~big, 5] <= 1e-290), note
    assert np.all(stats[np.abs(stats[:, 4]) > 38.5, 5] == 0.0), note


CASES = [   # (n, q, missing rates, case rate): sample counts at the 32-sample tile edges; q covers every KMAX
    (8, 1, [0.0], 0.5), (31, 2, [0.0, 0.3], 0.5), (32, 3, [0.0], 0.5), (33, 4, [0.01], 0.5), (63, 5, [0.0, 0.3], 0.5),
    (64, 8, [0.0], 0.5), (65, 9, [0.01, 0.3], 0.5), (127, 16, [0.0, 0.3], 0.5), (128, 17, [0.0], 0.5),
    (255, 11, [0.0, 0.01, 0.3, 0.95], 0.5), (256, 32, [0.0, 0.01], 0.5), (257, 1, [0.0, 0.3, 0.95], 0.1),
    (511, 11, [0.01, 0.3], 0.1), (1000, 2, [0.0, 0.01], 0.1), (2504, 11, [0.0, 0.01, 0.3, 0.95], 0.1),
    (2504, 32, [0.01], 0.5), (2504, 3, [0.0, 0.3], 0.01), (2504, 16, [0.01], 0.01),
]


@pytest.mark.parametrize("n,q,miss,rate", CASES)
def test_against_the_converged_fit(n, q, miss, rate):
    nv = 97   # three CTAs of 32 variants and one more
    rows, pheno, covar = _cohort(n * 100 + q, n, nv, q, miss, rate, excluded=0.0 if n < q + 20 else 0.05)
    with native.NativePca(n, device=0) as nat:
        used = nat.glmLogisticBegin(pheno, covar)
        got, gerr, gpass = nat.glmLogisticBed(rows)
    assert used == int(glm_ref.regression_samples(pheno, covar).sum())
    compared = check(got, gerr, gpass, rows, n, pheno, covar, note=f"n={n} q={q} rate={rate}")
    assert gerr[0] == 2 and gerr[1] == 1                       # monomorphic, all missing
    if n >= 255:
        assert compared >= 20, compared


def test_separated_variants():
    """Carriers only among the cases (1, 2, 3 and 10 of them), only among the controls, and a variant whose called
    samples are all cases: LOGISTIC_CONVERGE_FAIL, after 25 passes or (no control among the called) before any."""
    n, q = 400, 3
    rng = np.random.default_rng(31)
    covar = rng.normal(size=(n, q - 1))
    pheno = (rng.random(n) < 0.3).astype(float)
    cases, ctrl = np.flatnonzero(pheno == 1), np.flatnonzero(pheno == 0)
    code = np.full((8, n), 3, np.uint8)
    for r, k in enumerate((1, 2, 3, 10)):
        code[r, rng.choice(cases, k, replace=False)] = 2
    code[4, rng.choice(ctrl, 1, replace=False)] = 2
    code[5, rng.choice(ctrl, 6, replace=False)] = 0
    code[6] = 1
    code[6, cases] = rng.integers(2, 4, len(cases))            # only the cases are called
    code[7] = grm_ref.balding_nichols(rng, n, 1)[0]            # an ordinary variant
    rows = grm_ref.pack(code)
    with native.NativePca(n, device=0) as nat:
        nat.glmLogisticBegin(pheno, covar)
        got, gerr, gpass = nat.glmLogisticBed(rows)
    check(got, gerr, gpass, rows, n, pheno, covar, note="separated")
    assert np.all(gerr[:7] == 5) and gerr[7] == 0
    assert np.all(gpass[:6] == 25) and gpass[6] == 0


@pytest.mark.parametrize("n", [2504, 65537, 1000003])
def test_near_fixed_alleles(n):
    rng = np.random.default_rng(n)
    q = 3
    code = np.concatenate([glm_ref.near_fixed_codes(rng, n), grm_ref.balding_nichols(rng, n, 3, miss=0.01)])
    rows = grm_ref.pack(code)
    covar = rng.normal(size=(n, q - 1))
    pheno = (rng.random(n) < 0.3).astype(float)
    # past 65 535 samples a context holds a one-row Gram band instead of the whole Gram
    with native.NativePca(n, device=0, gram_band=(0, 1) if n > 65535 else None) as nat:
        nat.glmLogisticBegin(pheno, covar)
        got, gerr, gpass = nat.glmLogisticBed(rows)
        a2, e2, p2 = nat.glmLogisticBed(rows, counted=2)
    check(got, gerr, gpass, rows, n, pheno, covar, note=f"near-fixed n={n}")
    check(a2, e2, p2, rows, n, pheno, covar, counted=2, note=f"near-fixed A2 n={n}")
    _symmetric(got, gerr, gpass, a2, e2, p2)


def _symmetric(a1, e1, p1, a2, e2, p2):
    """Counting A2: the same ERRCODE, passes, OBS_CT, SE and P bits, and BETA and Z negated bit for bit."""
    assert np.array_equal(e1, e2) and np.array_equal(p1, p2)
    ok = e1 == 0
    assert np.array_equal(_bits(a1[:, 0]), _bits(a2[:, 0]))
    assert np.array_equal(_bits(a1[ok, 2]), _bits(-a2[ok, 2]))
    assert np.array_equal(_bits(a1[ok, 3]), _bits(a2[ok, 3]))
    assert np.array_equal(_bits(a1[ok, 4]), _bits(-a2[ok, 4]))
    assert np.array_equal(_bits(a1[ok, 5]), _bits(a2[ok, 5]))


def test_p_values_far_out():
    """Dosage effects from weak to overwhelming at 21 845 samples: |Z| from below 1 to past 38.5, where P is 0."""
    n = 21845
    rng = np.random.default_rng(41)
    code = grm_ref.balding_nichols(rng, n, 48)
    rows = grm_ref.pack(code)
    g, _ = glm_ref.dosages(rows, n)
    eta = -1.0 + sum(b * (g[j] - g[j].mean()) for j, b in ((3, 0.05), (9, 0.5), (17, 1.5), (30, 3.0), (40, 6.0)))
    pheno = (rng.random(n) < 1 / (1 + np.exp(-eta))).astype(float)
    covar = np.zeros((n, 0))                                   # the intercept alone
    with native.NativePca(n, device=0) as nat:
        nat.glmLogisticBegin(pheno, covar)
        got, gerr, gpass = nat.glmLogisticBed(rows)
    check(got, gerr, gpass, rows, n, pheno, covar, note="far out")
    z = np.abs(got[gerr == 0, 4])
    assert z.min() < 1.0 and z.max() > 38.5, (z.min(), z.max())


def test_bits_across_calls_strides_chunks_runs_and_neighbours():
    """One-row calls, a split at every CTA edge, strides with noisy padding and a second run give the bits of one call;
    a row keeps its bits among neighbours that converge at other pass counts, in any order."""
    n, q = 301, 5
    rows, pheno, covar = _cohort(7, n, 200, q, [0.0, 0.01, 0.3], 0.3)
    rng = np.random.default_rng(8)
    cases = np.flatnonzero(pheno == 1)
    sep = np.full((3, n), 3, np.uint8)                        # separated rows: 25 passes each
    for r in range(3):
        sep[r, rng.choice(cases, r + 1, replace=False)] = 2
    rows = np.concatenate([rows, grm_ref.pack(sep)])
    nv = rows.shape[0]
    wide = rng.integers(0, 256, (nv, rows.shape[1] + 13), dtype=np.uint8)
    wide[:, :rows.shape[1]] = rows
    wide[:, rows.shape[1] - 1] |= np.uint8(0b11111100)        # garbage in the padding bits (n % 4 = 1)
    order = rng.permutation(nv)
    with native.NativePca(n, device=0) as nat:
        nat.glmLogisticBegin(pheno, covar)
        whole = nat.glmLogisticBed(rows)
        again = nat.glmLogisticBed(rows)
        strided = nat.glmLogisticBed(wide)
        ones = [nat.glmLogisticBed(rows[v:v + 1]) for v in range(0, nv, 7)]
        pieces = [nat.glmLogisticBed(rows[a:b]) for a, b in ((0, 31), (31, 33), (33, 64), (64, 190), (190, nv))]
        shuffled = nat.glmLogisticBed(rows[order])
        a2 = nat.glmLogisticBed(rows, counted=2)
    with native.NativePca(n, device=0) as nat:
        nat.glmLogisticBegin(pheno, covar)
        run2 = nat.glmLogisticBed(rows)
    assert len(set(whole[2].tolist())) >= 4                     # neighbours converge at different pass counts
    joined = tuple(np.concatenate([p[i] for p in pieces]) for i in range(3))
    for other in (again, strided, joined, run2):
        assert np.array_equal(_bits(other[0]), _bits(whole[0]))
        assert np.array_equal(other[1], whole[1]) and np.array_equal(other[2], whole[2])
    for k, v in enumerate(range(0, nv, 7)):
        assert np.array_equal(_bits(ones[k][0]), _bits(whole[0][v:v + 1])) and ones[k][2][0] == whole[2][v]
    assert np.array_equal(_bits(shuffled[0]), _bits(whole[0][order])) and np.array_equal(shuffled[2], whole[2][order])
    _symmetric(*whole, *a2)


def test_chunk_cap():
    """More rows than one 2^20-row chunk: the same bits as the rows split into two calls elsewhere."""
    n = 12
    rng = np.random.default_rng(11)
    nv = (1 << 20) + 37
    code = rng.integers(0, 4, (nv, n), dtype=np.uint8)
    rows = grm_ref.pack(code)
    pheno = np.array([0.0, 1.0] * 6)
    with native.NativePca(n, device=0) as nat:
        nat.glmLogisticBegin(pheno, rng.normal(size=(n, 1)))
        whole = nat.glmLogisticBed(rows)
        a = nat.glmLogisticBed(rows[:1000])
        b = nat.glmLogisticBed(rows[1000:])
    for i in range(3):
        assert np.array_equal(_bits(whole[i]) if i == 0 else whole[i], _bits(np.concatenate([a[i], b[i]])) if i == 0
                              else np.concatenate([a[i], b[i]]))
    assert np.count_nonzero(whole[1] == 0) > 1000


def test_state_and_refusals():
    n = 50
    rows, pheno, covar = _cohort(9, n, 20, 3, [0.0], 0.4)
    with native.NativePca(n, device=0) as nat:
        with pytest.raises(native.VpcaError) as e:
            nat.glmLogisticBed(rows)
        assert e.value.code == native.VPCA_ERR_STATE
        sep = covar.copy()
        sep[:, 1] = np.where(pheno == 1, 1.0, -1.0) + 0.01 * covar[:, 1]   # a covariate that separates the classes
        sep[np.isnan(pheno), 1] = 0.0
        for y, c, what in ((np.where(np.arange(n) == 3, np.inf, pheno), covar, "infinite"),
                           (pheno, np.where(np.arange(n)[:, None] == 4, -np.inf, covar), "infinite"),
                           (pheno, np.zeros((n, 32)), "exceed"),
                           (np.where(np.arange(n) < 4, 1.0, np.nan), covar, "regression samples"),
                           (np.where(np.arange(n) == 7, 2.0, pheno), covar, "phenotype of sample 7 is 2, not 0"),
                           (np.where(np.isnan(pheno), np.nan, 0.0), covar, "0 cases and"),
                           (np.where(np.isnan(pheno), np.nan, 1.0), covar, "controls among"),
                           (pheno, np.stack([covar[:, 0], 2.0 * covar[:, 0] + 1.0], axis=1), "covariate 2 is collinear"),
                           (pheno, sep, "null model .* does not converge")):
            with pytest.raises(native.VpcaError, match=what) as e:
                nat.glmLogisticBegin(y, c)
            assert e.value.code == native.VPCA_ERR_BAD_ARG
            with pytest.raises(native.VpcaError) as e:         # a refused begin leaves no state
                nat.glmLogisticBed(rows)
            assert e.value.code == native.VPCA_ERR_STATE
        nat.glmLogisticBegin(pheno, covar)
        nat.glmLogisticBed(rows)
        with pytest.raises(native.VpcaError) as e:             # a linear test on the logistic state
            nat.glmLinearBed(rows)
        assert e.value.code == native.VPCA_ERR_STATE
        with pytest.raises(native.VpcaError) as e:
            nat.glmLogisticBed(rows, counted=3)
        assert e.value.code == native.VPCA_ERR_BAD_ARG
        nat.glmBegin(np.where(np.isnan(pheno), np.nan, pheno + covar[:, 0]), covar)
        nat.glmLinearBed(rows)
        with pytest.raises(native.VpcaError) as e:             # a logistic test on the linear state
            nat.glmLogisticBed(rows)
        assert e.value.code == native.VPCA_ERR_STATE
        nat.glmLogisticBegin(pheno, covar)
        nat.reset()
        with pytest.raises(native.VpcaError) as e:
            nat.glmLogisticBed(rows)
        assert e.value.code == native.VPCA_ERR_STATE


def test_leaves_the_grm_pca_and_loadings_alone():
    n, nv = 120, 400
    code = grm_ref.balding_nichols(np.random.default_rng(12), n, nv, miss=0.02)
    rows = grm_ref.pack(code)
    pheno = (np.random.default_rng(13).random(n) < 0.4).astype(float)

    def run(with_glm):
        with native.NativePca(n, device=0) as nat:
            nat.grmBed(rows)
            nat.grmFinalize()
            if with_glm:
                nat.glmLogisticBegin(pheno)
                nat.glmLogisticBed(rows)
            G = nat.getGrm()
            vecs, evals = nat.computePcaGrm(3)
            w, tab = nat.grmLoadingsBed(3, rows)
            return G, vecs, evals, w, tab
    for a, b in zip(run(False), run(True)):
        assert np.array_equal(_bits(a), _bits(b))


def test_leaves_the_gram_alone():
    n, nv = 200, 300
    code = grm_ref.balding_nichols(np.random.default_rng(14), n, nv, miss=0.02)
    rows = grm_ref.pack(code)
    pheno = (np.random.default_rng(15).random(n) < 0.4).astype(float)

    def run(with_glm):
        with native.NativePca(n, device=0) as nat:
            if with_glm:
                nat.glmLogisticBegin(pheno)
                nat.glmLogisticBed(rows)
            nat.accumulateBed(0, rows, 1)
            nat.commit(0)
            nat.finalizeGram()
            return nat.getGram()
    assert np.array_equal(run(False), run(True))


# ---- the driver end to end -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", ["grm", "carrier", "king"])
def test_driver_end_to_end(tmp_path, capsys, mode):
    n, nv = 600, 4000
    rng = np.random.default_rng(7)
    code = grm_ref.balding_nichols(rng, n, nv, pops=3, miss=0.01)
    d = np.where(code == 0, 2, np.where(code == 2, 1, np.where(code == 3, 0, -1))).T
    prefix = str(tmp_path / "c")
    plink.write_fileset(prefix, d, positions=1000 * np.arange(nv) + 1)
    pop = np.repeat(np.arange(3), _pop_sizes(n))
    y = np.where(rng.random(n) < np.array([0.2, 0.35, 0.5])[pop], 2.0, 1.0)
    y[:5] = 0.0                                                # missing by code
    fam = plink.read_fam_ids(prefix)
    (tmp_path / "p.txt").write_text("#FID IID D\n" + "".join(f"{f} {i} {float(v)!r}\n" for (f, i), v in zip(fam, y)))
    P = str(tmp_path / "P")
    argv = ["--bed-path", prefix, "--maf", "0.01", "--ld-prune", "0.2", "--num-pc", "2", "--pheno",
            str(tmp_path / "p.txt"), "--glm", "--glm-logistic", "--output-path", P]
    if mode == "grm":
        argv.append("--grm")
    elif mode == "king":
        argv += ["--king-cutoff", "0.177"]
    variants_pca.main(argv)
    out = capsys.readouterr().out
    m = re.search(r"GLM logistic: D on (\d+) of (\d+) samples \((\d+) cases, (\d+) controls, 5 without a phenotype or "
                  r"covariate\), 3 covariates \(intercept, 2 PCs\); (\d+) variants tested, (\d+) with an ERRCODE; "
                  r"lambda_GC = ([0-9.]+)\.", out)
    assert m, out
    lam = float(m.group(7))
    assert 0.9 <= lam <= 1.1
    lines = open(P + ".D.glm.logistic").read().splitlines()
    assert lines[0].split("\t") == ["#CHROM", "POS", "ID", "REF", "ALT", "A1", "A1_FREQ", "TEST", "OBS_CT", "OR",
                                    "LOG(OR)_SE", "Z_STAT", "P", "ERRCODE"]
    rows = [ln.split("\t") for ln in lines[1:]]
    bed = plink.BedFile(prefix)
    allrows = bed.rows(0, bed.n_variants)
    keep, _ = variants_pca.variant_qc_keep(qc_counts(allrows, n), None, 0.01, None, None)
    assert len(rows) == int(keep.sum()) == int(m.group(5))
    if mode == "grm":
        ev = [ln.split("\t") for ln in open(P + ".eigenvec").read().splitlines()[1:]]
        vecs = np.array([[float(x) for x in r[2:]] for r in ev])
        yy = np.where(y == 2.0, 1.0, np.where(y == 1.0, 0.0, np.nan))
        got = np.array([[float("nan") if x == "NA" else float(x) for x in (r[8], r[6], r[9], r[10], r[11], r[12])]
                        for r in rows])
        got[:, 2] = np.log(got[:, 2])
        gerr = np.array([ref.ERRCODES.index(r[13]) for r in rows])
        want, werr, _ = ref.mirror(allrows[keep], n, yy, vecs)
        assert np.array_equal(gerr, werr)
        ok = werr == 0
        assert np.allclose(got[ok, 2], want[ok, 2], rtol=1e-6, atol=1e-9 * np.max(want[ok, 3]))
        assert np.allclose(got[ok, 3:5], want[ok, 3:5], rtol=1e-6)
        assert abs(lam - variants_pca.lambda_gc(want, werr)) <= 1e-6
