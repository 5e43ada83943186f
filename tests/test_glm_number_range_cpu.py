"""The linear tests' reference (tests/glm_ref.py) at a million samples, and why the kernels centre the dosage (DESIGN.md
15).  The reference must not cancel where the kernel could: at near-fixed alleles, with a covariate far from 0 and with
a phenotype of any scale, it gives the same BETA, SE, T_STAT and P to 1e-12 as the forms that are exact in real
arithmetic.  A numpy restatement of the kernels' sums (one FMA chain per column in sample order, which np.cumsum
reproduces exactly because g q is exact for an integer g of at most 2 in magnitude) shows the Schur term
s = sum g^2 - u^T u losing seven digits to cancellation at 10^5 samples when g is the raw dosage of an almost fixed
allele, and none when g is centred on the integer nearest its mean."""
import numpy as np
import pytest

import glm_ref
import grm_ref

TOL = 1e-12


def _agree(got, gerr, want, werr, sign=1.0, scale=1.0, note=""):
    """BETA, SE, T_STAT and P of `got` (BETA and T_STAT times `sign`, BETA and SE over `scale`) against `want`."""
    assert np.array_equal(gerr, werr) and np.array_equal(got[:, 0], want[:, 0]), note
    ok = werr == 0
    b, se, t, p = sign * got[ok, 2] / scale, got[ok, 3] / scale, sign * got[ok, 4], got[ok, 5]
    wb, wse, wt, wp = (want[ok, i] for i in range(2, 6))
    assert np.all(np.abs(b - wb) <= TOL * np.maximum(np.abs(wb), wse)), (note, np.max(np.abs(b - wb) / wse))
    assert np.all(np.abs(se - wse) <= TOL * wse), (note, np.max(np.abs(se - wse) / wse))
    assert np.all(np.abs(t - wt) <= TOL * np.maximum(np.abs(wt), 1.0)), (note, np.max(np.abs(t - wt)))
    assert np.all(np.abs(p - wp) <= TOL * wp), (note, np.max(np.abs(p - wp) / wp))


def test_reference_at_a_million_samples():
    n = 10 ** 6
    rng = np.random.default_rng(1)
    code = np.concatenate([glm_ref.near_fixed_codes(rng, n), grm_ref.balding_nichols(rng, n, 2)])
    code[:, rng.random(n) < 0.01] = 1
    rows = grm_ref.pack(code)
    covar = rng.normal(size=(n, 3))
    y = rng.normal(size=n) + 0.2 * covar[:, 0]
    y[:5] = np.nan
    want, werr = glm_ref.linear(rows, n, y, covar)
    assert np.all(werr == 0)
    m, merr = glm_ref.linear(glm_ref.mirror(rows), n, y, covar)
    _agree(m, merr, want, werr, sign=-1.0, note="mirrored")
    assert np.all(np.abs(m[:, 1] + want[:, 1] - 1.0) <= np.spacing(1.0))
    _agree(*glm_ref.linear(rows, n, y, covar, counted=2), want, werr, sign=-1.0, note="counted=2")
    _agree(*glm_ref.linear(rows, n, y, covar, centre=False), want, werr, note="not centred")
    shifted = covar.copy()
    shifted[:, 1] += 1e4
    _agree(*glm_ref.linear(rows, n, y, shifted), want, werr, note="covariate + 1e4")
    for scale in (1e6, 1e-6):
        _agree(*glm_ref.linear(rows, n, scale * y, covar), want, werr, scale=scale, note=f"phenotype x {scale}")


def test_mirror_swaps_the_homozygous_codes():
    code = np.array([[0, 1, 2, 3, 3, 2, 1, 0, 0]], np.uint8)
    want = np.array([[3, 1, 2, 0, 0, 2, 1, 3, 3]], np.uint8)
    assert np.array_equal(glm_ref.codes(glm_ref.mirror(grm_ref.pack(code)), 9), want)
    g1, c1 = glm_ref.dosages(glm_ref.mirror(grm_ref.pack(code)), 9)
    g2, c2 = glm_ref.dosages(grm_ref.pack(code), 9, counted=2)
    assert np.array_equal(g1, g2) and np.array_equal(c1, c2)


@pytest.mark.parametrize("s,obs,c", [(0, 1, 0), (0, 10, 0), (4, 10, 0), (5, 10, 1), (15, 10, 1), (16, 10, 2), (20, 10, 2),
                                     (1, 1, 1), (3, 2, 1)])
def test_nearest_integer_mean(s, obs, c):
    assert glm_ref.nearest_integer_mean(s, obs) == c
    assert glm_ref.nearest_integer_mean(2 * obs - s, obs) == 2 - c   # the centre of 2 - g
    assert abs(s / obs - c) <= 0.5


# ---- the kernels' arithmetic in numpy --------------------------------------------------------------------------------------
def _chain(a):
    """a[0] + a[1] + ... in order, rounding after every addition."""
    return float(np.cumsum(a)[-1])


def _mgs(C):
    """vpca_glm_begin's Q: the columns of C orthonormalised in order by modified Gram-Schmidt applied twice."""
    Q = np.zeros_like(C)
    for c in range(C.shape[1]):
        col = C[:, c].copy()
        for _ in range(2):
            for k in range(c):
                col -= _chain(Q[:, k] * col) * Q[:, k]
        Q[:, c] = col / np.sqrt(_chain(col * col))
    return Q


def _kernel_schur(g, Q):
    """s = sum g^2 - u^T u, u = L^-1 Q^T g, P = Q^T Q = L L^T, with b = Q^T g as glm_sums_kernel sums it."""
    b = np.array([_chain(g * Q[:, c]) for c in range(Q.shape[1])])
    u = np.linalg.solve(np.linalg.cholesky(Q.T @ Q), b)
    return float(g @ g) - float(u @ u)


def test_the_schur_term_cancels_unless_the_dosage_is_centred():
    n = 100_000
    rng = np.random.default_rng(4)
    C = np.concatenate([np.ones((n, 1)), rng.normal(size=(n, 2))], axis=1)
    Q = _mgs(C)
    cases = {"A1 fixed but one het": np.where(np.arange(n) == 7, 1.0, 2.0),
             "all het but one hom": np.where(np.arange(n) == 7, 2.0, 1.0),
             "A1 frequency 0.999": rng.binomial(2, 0.999, n).astype(np.float64)}
    raw = {}
    for name, g in cases.items():
        c = glm_ref.nearest_integer_mean(g.sum(), n)
        Cc = C - np.concatenate([[0.0], C[:, 1:].mean(axis=0)])
        r = (g - c) - Cc @ np.linalg.lstsq(Cc, g - c, rcond=None)[0]
        want = float(r @ r)
        raw[name] = abs(_kernel_schur(g, Q) - want) / want
        centred = abs(_kernel_schur(g - c, Q) - want) / want
        assert centred <= 1e-14, (name, centred)
    assert raw["A1 fixed but one het"] > 1e-7, raw
    assert raw["all het but one hom"] > 1e-8, raw
