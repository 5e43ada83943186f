"""Host reference of the linear association tests (DESIGN.md 15): per variant, np.linalg.lstsq on the complete cases with
an intercept and the covariates, scipy.stats.t.sf for P, and the ERRCODE rules of include/vpca.h.  Also a numpy double
of NativePca.glmBegin / glmLinearBed for the driver tests, and the genomic inflation factor."""
import numpy as np
import scipy.stats

from qc_ref import codes

ERRCODES = (".", "TOO_FEW_OBS", "CONST_ALLELE", "VIF_INFINITE", "NO_RESIDUAL")
LAMBDA_DENOM = 0.45493642311957283   # the median of chi-square with 1 degree of freedom


def dosages(rows, n, counted=1):
    """(nv, stride) .bed rows -> (g (nv, n) float64 count of the counted allele, 0 for a missing call; called (nv, n))."""
    c = codes(np.asarray(rows), n)
    g = np.select([c == 0, c == 2, c == 3], [2.0, 1.0, 0.0], 0.0) if counted == 1 else \
        np.select([c == 0, c == 2, c == 3], [0.0, 1.0, 2.0], 0.0)
    return g, c != 1


def regression_samples(pheno, covar):
    ok = np.isfinite(pheno)
    if covar is not None and covar.shape[1]:
        ok &= np.isfinite(covar).all(axis=1)
    return ok


def linear(rows, n, pheno, covar=None, counted=1, centre=True):
    """-> (stats (nv, 6): OBS_CT, A1_FREQ, BETA, SE, T_STAT, P with NaN where undefined; err (nv,) int).  Per variant,
    over the called regression samples A, the residuals of g - c and of the phenotype after [1, covar - its mean] by
    lstsq, c the integer nearest the mean of g over A (with centre=False, of g after [1, covar]).  The intercept absorbs
    both shifts, so BETA, SE and the residuals are those of [1, covar, g]; but the residual of a dosage that is almost constant, such as 2 at all but a few samples, is then
    computed from values of size at most 2 around a mean within 1/2 of 0, not as a difference of sums of size 4 OBS_CT,
    and a covariate far from 0 is not nearly collinear with the intercept."""
    pheno = np.asarray(pheno, np.float64)
    covar = np.zeros((n, 0)) if covar is None else np.asarray(covar, np.float64).reshape(n, -1)
    reg = regression_samples(pheno, covar)
    q = covar.shape[1] + 1
    g, called = dosages(rows, n, counted)
    nv = g.shape[0]
    out = np.full((nv, 6), np.nan)
    err = np.zeros(nv, np.int32)
    C = np.concatenate([np.ones((n, 1)), covar], axis=1)
    yt = np.zeros(n)   # the residual phenotype y~ = y - C (C^T C)^-1 C^T y over all regression samples
    yt[reg] = pheno[reg] - C[reg] @ np.linalg.lstsq(C[reg], pheno[reg], rcond=None)[0]
    Q = np.zeros((n, q))   # an orthonormal basis of C over the regression samples (zero elsewhere)
    Q[reg] = np.linalg.qr(C[reg])[0]
    for v in range(nv):
        A = reg & called[v]
        obs = int(A.sum())
        out[v, 0] = obs
        ga, ya, Ca = g[v, A], pheno[A], C[A]
        if obs:
            out[v, 1] = ga.sum() / (2.0 * obs)
        df = obs - q - 1
        if df < 1:
            err[v] = 1
            continue
        if np.all(ga == ga[0]):
            err[v] = 2
            continue
        if centre:
            ga = ga - nearest_integer_mean(ga.sum(), obs)
            Ca = Ca - np.concatenate([[0.0], Ca[:, 1:].mean(axis=0)])
        # the dosage's residual sum of squares after the covariates against its centred one
        gr = ga - Ca @ np.linalg.lstsq(Ca, ga, rcond=None)[0]
        s = float(gr @ gr)
        css = float(((ga - ga.mean()) ** 2).sum())
        if collinear(Q[A]) or s <= 1e-10 * css:
            err[v] = 3
            continue
        # BETA and the residuals from the two residuals after the covariates (Frisch-Waugh-Lovell): no solve with the
        # dosage beside the intercept, whose condition would be squared into BETA
        yr = ya - Ca @ np.linalg.lstsq(Ca, ya, rcond=None)[0]
        beta = float(gr @ yr) / s
        res = yr - beta * gr
        rss = float(res @ res)
        if rss <= 1e-12 * float((yt[A] ** 2).sum()):
            err[v] = 4
            continue
        se = np.sqrt(rss / df / s)
        t = beta / se
        out[v, 2:] = beta, se, t, 2.0 * scipy.stats.t.sf(abs(t), df)
    return out, err


def nearest_integer_mean(sum_g, obs):
    """The integer in {0, 1, 2} nearest the mean dosage sum_g / obs > 0, a tie going to 1, in integers as glm.cu has it.
    The tie rule makes the centre of 2 - g exactly 2 minus the centre of g, so the two centred dosages are negatives."""
    sum_g, obs = int(sum_g), int(obs)
    return 0 if 2 * sum_g < obs else 2 if 2 * sum_g > 3 * obs else 1


def mirror(rows):
    """.bed rows with codes 00 (HOM_A1) and 11 (HOM_A2) swapped: counting A1 in them counts A2 in `rows`."""
    rows = np.asarray(rows, np.uint8)
    lo, hi = rows & 0x55, (rows >> 1) & 0x55
    hom = ~(lo ^ hi) & 0x55   # 00 or 11
    return rows ^ (hom * 3).astype(np.uint8)


def near_fixed_codes(rng, n, kinds=None):
    """Codes (k, n) of variants whose counted allele A1 is almost fixed or whose dosage is almost constant: A1 fixed but
    1, 2, 3 or 10 hets; A1 fixed but one HOM_A2; all het but one or two homs; A1 frequency 0.999 and 0.99.  The carriers
    of the rarer genotypes sit at random samples, at least one of them.  kinds: a subset of KINDS by name."""
    out = []
    for kind in KINDS if kinds is None else kinds:
        c = np.zeros(n, np.uint8)
        if kind.startswith("het"):
            c[rng.choice(n, int(kind[3:]), replace=False)] = 2
        elif kind == "hom2":
            c[rng.integers(n)] = 3
        elif kind.startswith("allhet"):
            c[:] = 2
            c[rng.choice(n, int(kind[6:]), replace=False)] = [0, 3][: int(kind[6:])]
        else:
            a1 = rng.binomial(2, float(kind[1:]), n)
            if np.all(a1 == 2):
                a1[rng.integers(n)] = 1
            c = np.select([a1 == 2, a1 == 1], [0, 2], 3).astype(np.uint8)
        out.append(c)
    return np.stack(out)


KINDS = ("het1", "het2", "het3", "het10", "hom2", "allhet1", "allhet2", "f0.999", "f0.99")


def collinear(QA, pivot_min=1e-10):
    """The covariates are collinear over A: a Cholesky pivot of P = Q_A^T Q_A (eigenvalues in [0, 1]) is <= pivot_min.
    This is the kernel's rule; it holds, among others, wherever C_A is rank-deficient."""
    P = QA.T @ QA
    d = np.zeros(len(P))
    L = np.zeros_like(P)
    for j in range(len(P)):
        d[j] = P[j, j] - L[j, :j] @ L[j, :j]
        if not d[j] > pivot_min:
            return True
        L[j, j] = np.sqrt(d[j])
        L[j + 1:, j] = (P[j + 1:, j] - L[j + 1:, :j] @ L[j, :j]) / L[j, j]
    return False


def lambda_gc(stats, err):
    """median T_STAT^2 over the `.` variants / the median of chi-square(1)."""
    t = stats[err == 0, 4]
    return float(np.median(t * t) / LAMBDA_DENOM) if len(t) else float("nan")


class GlmDouble:
    """NativePca.glmBegin / glmLinearBed in numpy (the per-variant lstsq above), with the refusals of vpca_glm_begin."""

    def glmBegin(self, pheno, covar=None):
        from spark_examples_b200 import native
        y = np.asarray(pheno, np.float64)
        c = np.zeros((self.n, 0)) if covar is None else np.asarray(covar, np.float64).reshape(self.n, -1)
        if np.isinf(y).any() or np.isinf(c).any() or c.shape[1] + 1 > 32:
            raise native.VpcaError(native.VPCA_ERR_BAD_ARG, "bad GLM input")
        reg = regression_samples(y, c)
        if reg.sum() < c.shape[1] + 3 or np.all(y[reg] == y[reg][0]):
            raise native.VpcaError(native.VPCA_ERR_BAD_ARG, "bad GLM input")
        self.glm = (y, c)
        self.glm_calls = []
        return int(reg.sum())

    def glmLinearBed(self, rows, counted=1):
        rows = np.asarray(rows)
        self.glm_calls.append(rows.shape[0])
        return linear(rows, self.n, *self.glm, counted=counted)
