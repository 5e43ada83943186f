"""Firth-penalized logistic tests on the GPU (vpca_glm_firth_bed; DESIGN.md 17): ERRCODE, passes and the Firth flags
exactly against the mirror of the kernel's iteration and BETA, SE and Z against the converged Firth fit, over the
logistic test's grid, in both modes; separated rows and the 2 x 2 closed form; near-fixed alleles up to a million
samples; fallback's maximum-likelihood rows against vpca_glm_logistic_bed and its Firth rows against `always`, bit for
bit; the bits across calls, CTA edges, strides, runs, neighbours and the chunk cap; the counted-allele symmetry; the state
and mode refusals; and the driver end to end."""
import re

import numpy as np
import pytest

import glm_firth_ref as ref
import glm_ref
import grm_ref
from spark_examples_b200 import native, plink, variants_pca
from test_glm_gpu import _pop_sizes, _vif
from test_glm_logistic_gpu import CASES, _cohort, _symmetric, check_p

pytestmark = pytest.mark.gpu

VIF_OK = 1e3      # BETA, SE and Z are compared where the dosage's variance inflation factor is below this


def _bits(a):
    return np.ascontiguousarray(a, np.float64).view(np.int64)


def check(res, rows, n, pheno, covar, mode, counted=1, note=""):
    """ERRCODE, passes, Firth flags, OBS_CT and A1_FREQ exactly against the mirror; BETA, SE and Z of the Firth rows to
    1e-7 against the converged Firth fit where the VIF is below VIF_OK; P against scipy at the kernel's Z."""
    got, gerr, gpass, gfirth = res
    want, werr, wpass, wfirth = ref.mirror(rows, n, pheno, covar, counted=counted,
                                           mode=ref.FALLBACK if mode == "fallback" else ref.ALWAYS)
    bad = np.flatnonzero((gerr != werr) | (gpass != wpass))
    assert bad.size == 0, (note, bad, gerr[bad], werr[bad], gpass[bad], wpass[bad])
    assert np.array_equal(gfirth, wfirth), note
    assert np.array_equal(got[:, 0], want[:, 0]), note
    assert np.array_equal(_bits(got[~np.isnan(got[:, 1]), 1]), _bits(want[~np.isnan(want[:, 1]), 1])), note
    ok = gerr == 0
    assert np.all(np.isnan(got[~ok, 2:])) and np.all(np.isfinite(got[ok, 2:])), note
    vif = _vif(rows, n, pheno, covar, counted)
    cmp = np.flatnonzero(ok & (gfirth == 1) & (vif < VIF_OK))
    conv = ref.converged(rows, n, pheno, covar, counted, variants=cmp)
    b, se, z = got[cmp, 2], got[cmp, 3], got[cmp, 4]
    wb, wse, wz = conv[cmp, 2], conv[cmp, 3], conv[cmp, 4]
    assert np.all(np.isfinite(wb)), note
    assert np.all(np.abs(b - wb) <= 1e-7 * np.maximum(np.abs(wb), wse)), (note, np.max(np.abs(b - wb) / wse))
    assert np.all(np.abs(se - wse) <= 1e-7 * wse), (note, np.max(np.abs(se - wse) / wse))
    assert np.all(np.abs(z - wz) <= 1e-7 * np.maximum(np.abs(wz), 1.0)), note
    check_p(got[ok], note)
    return cmp.size


def _rare(rng, pheno, n, base):
    """Rows of A2 carriers on an A1 background: 0 to 3 carriers among the cases and 0 to 3 among the controls."""
    cases, ctrl = np.flatnonzero(pheno == 1), np.flatnonzero(pheno == 0)
    out = []
    for a in range(min(4, len(cases) + 1)):
        for b in range(min(4, len(ctrl) + 1)):
            c = base.copy()
            c[np.concatenate([rng.choice(cases, a, replace=False), rng.choice(ctrl, b, replace=False)])] = 2
            out.append(c)
    return np.array(out, np.uint8)


@pytest.mark.parametrize("n,q,miss,rate", CASES)
def test_against_the_converged_fit(n, q, miss, rate):
    nv = 81
    rows, pheno, covar = _cohort(n * 100 + q, n, nv, q, miss, rate, excluded=0.0 if n < q + 20 else 0.05)
    rng = np.random.default_rng(n + q)
    rows = np.concatenate([rows, grm_ref.pack(_rare(rng, pheno, n, np.full(n, 3, np.uint8)))])
    with native.NativePca(n, device=0) as nat:
        nat.glmLogisticBegin(pheno, covar)
        fb = nat.glmFirthBed(rows, mode="fallback")
        al = nat.glmFirthBed(rows, mode="always")
    note = f"n={n} q={q} rate={rate}"
    check(fb, rows, n, pheno, covar, "fallback", note=note + " fallback")
    compared = check(al, rows, n, pheno, covar, "always", note=note + " always")
    if n >= 255:
        assert compared >= 20, compared
    f = fb[3] == 1                                             # the same bits in both modes
    assert np.array_equal(_bits(fb[0][f]), _bits(al[0][f])) and np.array_equal(fb[2][f], al[2][f])


def test_separated_variants():
    """Carriers only among the cases (1, 2, 3 and 10 of them) and only among the controls: finite in both modes, and at
    q = 1 the closed form of the 2 x 2 table with 1/2 added to each cell."""
    for q in (3, 1):
        n = 400
        rng = np.random.default_rng(31)
        covar = rng.normal(size=(n, q - 1))
        pheno = (rng.random(n) < 0.3).astype(float)
        cases, ctrl = np.flatnonzero(pheno == 1), np.flatnonzero(pheno == 0)
        code = np.full((6, n), 3, np.uint8)
        for r, k in enumerate((1, 2, 3, 10)):
            code[r, rng.choice(cases, k, replace=False)] = 2
        code[4, rng.choice(ctrl, 1, replace=False)] = 2
        code[5, rng.choice(ctrl, 6, replace=False)] = 2
        rows = grm_ref.pack(code)
        with native.NativePca(n, device=0) as nat:
            nat.glmLogisticBegin(pheno, covar)
            ml = nat.glmLogisticBed(rows)
            fb = nat.glmFirthBed(rows, mode="fallback")
            al = nat.glmFirthBed(rows, mode="always")
        assert np.all(ml[1] == ref.CONVERGE_FAIL)
        for res, mode in ((fb, "fallback"), (al, "always")):
            assert np.all(res[1] == 0) and np.all(res[3] == 1) and np.all(np.isfinite(res[0][:, 2:]))
            check(res, rows, n, pheno, covar, mode, note=f"separated q={q} {mode}")
        assert np.array_equal(_bits(fb[0]), _bits(al[0]))
        if q == 1:
            g, _ = glm_ref.dosages(rows, n)
            for v in range(len(code)):
                a, b = np.sum(g[v][cases] != 0), np.sum(g[v][ctrl] != 0)
                c, d = len(cases) - a, len(ctrl) - b
                want = np.log((a + 0.5) * (d + 0.5) / ((b + 0.5) * (c + 0.5)))
                assert abs(al[0][v, 2] - want) <= 1e-7 * max(abs(want), al[0][v, 3]), (v, al[0][v, 2], want)


@pytest.mark.parametrize("n", [2504, 65537, 1000003])
def test_near_fixed_alleles(n):
    rng = np.random.default_rng(n)
    q = 3
    code = np.concatenate([glm_ref.near_fixed_codes(rng, n), grm_ref.balding_nichols(rng, n, 2, miss=0.01)])
    rows = grm_ref.pack(code)
    covar = rng.normal(size=(n, q - 1))
    pheno = (rng.random(n) < 0.3).astype(float)
    with native.NativePca(n, device=0, gram_band=(0, 1) if n > 65535 else None) as nat:
        nat.glmLogisticBegin(pheno, covar)
        a1 = nat.glmFirthBed(rows, mode="always")
        a2 = nat.glmFirthBed(rows, counted=2, mode="always")
    check(a1, rows, n, pheno, covar, "always", note=f"near-fixed n={n}")
    _symmetric(*a1[:3], *a2[:3])
    assert np.array_equal(a1[3], a2[3])


def test_fallback_bits_against_logistic_and_always():
    """fallback's maximum-likelihood rows are vpca_glm_logistic_bed's bits, its Firth rows `always`'s bits."""
    n, q = 600, 4
    rows, pheno, covar = _cohort(5, n, 150, q, [0.0, 0.01, 0.3], 0.1)
    rng = np.random.default_rng(6)
    rows = np.concatenate([rows, grm_ref.pack(_rare(rng, pheno, n, np.full(n, 3, np.uint8)))])
    with native.NativePca(n, device=0) as nat:
        nat.glmLogisticBegin(pheno, covar)
        ml = nat.glmLogisticBed(rows)
        fb = nat.glmFirthBed(rows, mode="fallback")
        al = nat.glmFirthBed(rows, mode="always")
    f = fb[3] == 1
    assert f.sum() >= 5 and (~f).sum() >= 100
    assert np.array_equal(f, (ml[1] == ref.CONVERGE_FAIL) & (ml[2] > 0))
    assert np.array_equal(_bits(fb[0][~f]), _bits(ml[0][~f]))
    assert np.array_equal(fb[1][~f], ml[1][~f]) and np.array_equal(fb[2][~f], ml[2][~f])
    assert np.array_equal(_bits(fb[0][f]), _bits(al[0][f]))
    assert np.array_equal(fb[1][f], al[1][f]) and np.array_equal(fb[2][f], al[2][f])


def test_bits_across_calls_strides_chunks_runs_and_neighbours():
    n, q = 301, 5
    rows, pheno, covar = _cohort(7, n, 120, q, [0.0, 0.01, 0.3], 0.3)
    rng = np.random.default_rng(8)
    rows = np.concatenate([rows, grm_ref.pack(_rare(rng, pheno, n, np.full(n, 3, np.uint8)))])
    nv = rows.shape[0]
    wide = rng.integers(0, 256, (nv, rows.shape[1] + 13), dtype=np.uint8)
    wide[:, :rows.shape[1]] = rows
    wide[:, rows.shape[1] - 1] |= np.uint8(0b11111100)        # garbage in the padding bits (n % 4 = 1)
    order = rng.permutation(nv)
    res = {}
    with native.NativePca(n, device=0) as nat:
        nat.glmLogisticBegin(pheno, covar)
        for mode in ("always", "fallback"):
            whole = nat.glmFirthBed(rows, mode=mode)
            again = nat.glmFirthBed(rows, mode=mode)
            strided = nat.glmFirthBed(wide, mode=mode)
            ones = [nat.glmFirthBed(rows[v:v + 1], mode=mode) for v in range(0, nv, 5)]
            pieces = [nat.glmFirthBed(rows[a:b], mode=mode) for a, b in ((0, 31), (31, 33), (33, 64), (64, 100),
                                                                          (100, nv))]
            shuffled = nat.glmFirthBed(rows[order], mode=mode)
            a2 = nat.glmFirthBed(rows, counted=2, mode=mode)
            res[mode] = whole
            assert len(set(whole[2][whole[3] == 1].tolist())) >= 4, mode   # neighbours at other pass counts
            joined = tuple(np.concatenate([p[i] for p in pieces]) for i in range(4))
            for other in (again, strided, joined):
                assert np.array_equal(_bits(other[0]), _bits(whole[0])), mode
                for i in (1, 2, 3):
                    assert np.array_equal(other[i], whole[i]), mode
            for k, v in enumerate(range(0, nv, 5)):
                assert np.array_equal(_bits(ones[k][0]), _bits(whole[0][v:v + 1])) and ones[k][2][0] == whole[2][v]
            assert np.array_equal(_bits(shuffled[0]), _bits(whole[0][order]))
            assert np.array_equal(shuffled[2], whole[2][order]) and np.array_equal(shuffled[3], whole[3][order])
            _symmetric(*whole[:3], *a2[:3])
    with native.NativePca(n, device=0) as nat:
        nat.glmLogisticBegin(pheno, covar)
        for mode in ("always", "fallback"):
            run2 = nat.glmFirthBed(rows, mode=mode)
            assert np.array_equal(_bits(run2[0]), _bits(res[mode][0]))
            assert all(np.array_equal(run2[i], res[mode][i]) for i in (1, 2, 3))


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
        for mode in ("fallback", "always"):
            whole = nat.glmFirthBed(rows, mode=mode)
            a = nat.glmFirthBed(rows[:1000], mode=mode)
            b = nat.glmFirthBed(rows[(1 << 20) - 5:], mode=mode)
            mid = nat.glmFirthBed(rows[1000:(1 << 20) - 5], mode=mode)
            assert np.array_equal(_bits(whole[0]), _bits(np.concatenate([a[0], mid[0], b[0]])))
            for i in (1, 2, 3):
                assert np.array_equal(whole[i], np.concatenate([a[i], mid[i], b[i]]))
            assert np.count_nonzero(whole[3]) > 1000, mode


def test_state_and_refusals():
    n = 50
    rows, pheno, covar = _cohort(9, n, 20, 3, [0.0], 0.4)
    with native.NativePca(n, device=0) as nat:
        with pytest.raises(native.VpcaError) as e:
            nat.glmFirthBed(rows)
        assert e.value.code == native.VPCA_ERR_STATE
        nat.glmBegin(np.where(np.isnan(pheno), np.nan, pheno + covar[:, 0]), covar)
        with pytest.raises(native.VpcaError, match="the GLM state is linear") as e:
            nat.glmFirthBed(rows, mode="always")
        assert e.value.code == native.VPCA_ERR_STATE
        nat.glmLogisticBegin(pheno, covar)
        nat.glmFirthBed(rows)
        lib, h = nat._lib, nat._h
        out = np.zeros((20, 6))
        err = np.zeros(20, np.int32)
        for mode in (0, 3, -1):
            rc = lib.vpca_glm_firth_bed(h, rows.ctypes.data, 20, rows.shape[1], 1, mode, out.ctypes.data,
                                        err.ctypes.data, None, None)
            assert rc == native.VPCA_ERR_BAD_ARG, mode
        with pytest.raises(native.VpcaError) as e:
            nat.glmFirthBed(rows, mode="sometimes")
        assert e.value.code == native.VPCA_ERR_BAD_ARG
        with pytest.raises(native.VpcaError) as e:
            nat.glmFirthBed(rows, counted=3)
        assert e.value.code == native.VPCA_ERR_BAD_ARG
        # out_passes and out_firth may be NULL
        rc = lib.vpca_glm_firth_bed(h, rows.ctypes.data, 20, rows.shape[1], 1, 2, out.ctypes.data, err.ctypes.data,
                                    None, None)
        assert rc == 0
        full = nat.glmFirthBed(rows, mode="always")
        assert np.array_equal(_bits(out), _bits(full[0])) and np.array_equal(err, full[1])
        nat.reset()
        with pytest.raises(native.VpcaError) as e:
            nat.glmFirthBed(rows)
        assert e.value.code == native.VPCA_ERR_STATE


# ---- the driver end to end -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", ["fallback", "always"])
def test_driver_end_to_end(tmp_path, capsys, mode):
    n, nv = 600, 3000
    rng = np.random.default_rng(7)
    code = grm_ref.balding_nichols(rng, n, nv, pops=3, miss=0.01)
    pop = np.repeat(np.arange(3), _pop_sizes(n))
    y = np.where(rng.random(n) < np.array([0.05, 0.1, 0.15])[pop], 2.0, 1.0)
    y[:5] = 0.0                                                # missing by code
    cases = np.flatnonzero(y == 2.0)
    for r in range(10, 2000, 97):                              # rare variants, some carried by cases alone
        code[r] = 3
        code[r, rng.choice(cases, 1 + r % 3, replace=False)] = 2
    d = np.where(code == 0, 2, np.where(code == 2, 1, np.where(code == 3, 0, -1))).T
    prefix = str(tmp_path / "c")
    plink.write_fileset(prefix, d, positions=1000 * np.arange(nv) + 1)
    fam = plink.read_fam_ids(prefix)
    (tmp_path / "p.txt").write_text("#FID IID D\n" + "".join(f"{f} {i} {float(v)!r}\n" for (f, i), v in zip(fam, y)))
    P = str(tmp_path / "P")
    variants_pca.main(["--bed-path", prefix, "--ld-prune", "0.2", "--num-pc", "2", "--grm", "--pheno",
                       str(tmp_path / "p.txt"), "--glm", "--glm-logistic", "--glm-firth", mode, "--output-path", P])
    out = capsys.readouterr().out
    ev = [ln.split("\t") for ln in open(P + ".eigenvec").read().splitlines()[1:]]
    vecs = np.array([[float(x) for x in r[2:]] for r in ev])
    yy = np.where(y == 2.0, 1.0, np.where(y == 1.0, 0.0, np.nan))
    bed = plink.BedFile(prefix)
    allrows = bed.rows(0, bed.n_variants)
    want, werr, _, wfirth = ref.mirror(allrows, n, yy, vecs, mode=ref.FALLBACK if mode == "fallback" else ref.ALWAYS)
    head = "GLM logistic" if mode == "fallback" else "GLM Firth"
    fitted = f", {int(wfirth.sum())} fitted by Firth regression" if mode == "fallback" else ""
    m = re.search(head + r": D on \d+ of 600 samples \(\d+ cases, \d+ controls, 5 without a phenotype or covariate\), 3 "
                  r"covariates \(intercept, 2 PCs\); 3000 variants tested, (\d+) with an ERRCODE" + re.escape(fitted) +
                  r"; lambda_GC = ([0-9.]+)\.", out)
    assert m, out
    path = P + (".D.glm.logistic.hybrid" if mode == "fallback" else ".D.glm.firth")
    lines = open(path).read().splitlines()
    rows = [ln.split("\t") for ln in lines[1:]]
    off = 1 if mode == "fallback" else 0
    if off:
        assert lines[0].split("\t")[7] == "FIRTH?"
        assert [r[7] for r in rows] == ["Y" if f else "N" for f in wfirth]
    gerr = np.array([ref.ERRCODES.index(r[13 + off]) for r in rows])
    assert np.array_equal(gerr, werr)
    got = np.array([[float("nan") if x == "NA" else float(x) for x in (r[9 + off], r[10 + off])] for r in rows])
    ok = werr == 0
    assert np.allclose(np.log(got[ok, 0]), want[ok, 2], rtol=1e-6, atol=1e-9 * np.max(want[ok, 3]))
    assert np.allclose(got[ok, 1], want[ok, 3], rtol=1e-6)
    assert wfirth.sum() >= 10
