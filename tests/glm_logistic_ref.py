"""Host reference of the logistic association tests (DESIGN.md 16), in two parts.

`converged`: per variant, maximum likelihood on the complete cases of logit P(case) = [1, covar, g] theta by Newton with
step halving, iterated until the step is below 1e-14 (relative to max(1, |theta|)) or at its rounding floor; BETA, SE = sqrt([H^-1]_gg), Z and
P = 2 scipy.stats.norm.sf(|Z|).  The design is centred as glm_ref.linear centres it (the dosage on its nearest integer
mean, the covariates on their means): the intercept absorbs both shifts, so the fit is that of [1, covar, g], but a
dosage that is almost constant is not almost collinear with the intercept.

`mirror`: the kernel's own iteration in numpy: the orthonormal basis Q of [1, covar] over the regression samples
(modified Gram-Schmidt applied twice, as vpca_glm_logistic_begin), the null fit on Q, the centred dosage, the start
(theta_null, 0), the Newton-decrement rule, the halving, the pivot rules and the pass cap.  It gives the ERRCODE and the
pass count of every variant (and BETA / SE at its own stopping point).

Also a numpy double of NativePca.glmLogisticBegin / glmLogisticBed for the driver tests."""
import numpy as np
import scipy.stats

from glm_ref import dosages, nearest_integer_mean, regression_samples

ERRCODES = (".", "TOO_FEW_OBS", "CONST_ALLELE", "VIF_INFINITE", "NO_RESIDUAL", "LOGISTIC_CONVERGE_FAIL")
OK, TOO_FEW_OBS, CONST_ALLELE, VIF_INFINITE, CONVERGE_FAIL = 0, 1, 2, 3, 5
MAX_PASS, MAX_HALVE, DELTA2, FALL, PIVOT_MIN = 25, 8, 1e-18, 1e-10, 1e-10


def evaluate(X, y, theta):
    """l, grad l and H = X^T W X of the logistic likelihood at theta."""
    eta = X @ theta
    e = np.exp(-np.abs(eta))
    rd = 1.0 / (1.0 + e)
    mu = np.where(eta >= 0.0, rd, e * rd)
    w = e * rd * rd
    m = np.where(y != 0.0, -eta, eta)
    l = -float(np.sum(np.maximum(m, 0.0) + np.log1p(e)))
    return l, X.T @ (y - mu), X.T @ (w[:, None] * X)


def cholesky(H, first):
    """(L with the pivots' square roots on the diagonal, code): code VIF_INFINITE for a pivot <= PIVOT_MIN H_jj on the first
    pass, CONVERGE_FAIL for a pivot <= 0 later, else OK."""
    p = len(H)
    L = np.zeros_like(H)
    for j in range(p):
        d = H[j, j] - L[j, :j] @ L[j, :j]
        if not (d > PIVOT_MIN * H[j, j] if first else d > 0.0):
            return None, VIF_INFINITE if first else CONVERGE_FAIL
        L[j, j] = np.sqrt(d)
        L[j + 1:, j] = (H[j + 1:, j] - L[j + 1:, :j] @ L[j, :j]) / L[j, j]
    return L, OK


def newton(X, y, theta0, pivot_rule=True, halvings=None):
    """The kernel's passes from theta0 -> (code, passes, theta + the last step, the last L).  pivot_rule: the first
    pass's VIF rule (the null fit has only the pivot > 0 rule).  halvings: a list the number of halved steps is
    appended to."""
    out = _newton(X, y, theta0, pivot_rule)
    if halvings is not None:
        halvings.append(out[4])
    return out[:4]


def _newton(X, y, theta0, pivot_rule):
    import scipy.linalg
    th = np.array(theta0, np.float64)
    thp, dl, lp, halv, total = th.copy(), np.zeros_like(th), 0.0, 0, 0
    for k in range(1, MAX_PASS + 1):
        l, g, H = evaluate(X, y, th)
        if not np.isfinite(l):
            return CONVERGE_FAIL, k, None, None, total
        if k > 1 and l < lp - FALL * abs(lp):
            if halv == MAX_HALVE or k == MAX_PASS:
                return CONVERGE_FAIL, k, None, None, total
            halv += 1
            total += 1
            dl = 0.5 * dl
            th = thp + dl
            continue
        L, code = cholesky(H, k == 1 and pivot_rule)
        if code:
            return code, k, None, None, total
        z = scipy.linalg.solve_triangular(L, g, lower=True)
        dd = float(z @ z)
        dl = scipy.linalg.solve_triangular(L.T, z, lower=False)
        if not np.isfinite(dd):
            return CONVERGE_FAIL, k, None, None, total
        if dd <= DELTA2:
            return OK, k, th + dl, L, total
        if k == MAX_PASS:
            return CONVERGE_FAIL, k, None, None, total
        lp, halv, thp, th = l, 0, th, th + dl
    return CONVERGE_FAIL, MAX_PASS, None, None, total


def basis(C):
    """The columns of C orthonormalised in order, modified Gram-Schmidt applied twice (vpca_glm_begin's basis)."""
    Q = np.array(C, np.float64)
    for c in range(Q.shape[1]):
        for _ in range(2):
            for k in range(c):
                Q[:, c] -= (Q[:, k] @ Q[:, c]) * Q[:, k]
        Q[:, c] /= np.sqrt(Q[:, c] @ Q[:, c])
    return Q


def _setup(n, pheno, covar):
    pheno = np.asarray(pheno, np.float64)
    covar = np.zeros((n, 0)) if covar is None else np.asarray(covar, np.float64).reshape(n, -1)
    reg = regression_samples(pheno, covar)
    return pheno, covar, reg, covar.shape[1] + 1


def null_fit(Q, y):
    """theta_null of Q over all regression samples, or None when the null model does not converge."""
    code, _, th, _ = newton(Q, y, np.zeros(Q.shape[1]), pivot_rule=False)
    return th if code == OK else None


def _flag(obs, ga, ya, q):
    if obs - q - 1 < 1:
        return TOO_FEW_OBS
    if np.all(ga == ga[0]):
        return CONST_ALLELE
    if np.all(ya == 0.0) or np.all(ya == 1.0):
        return CONVERGE_FAIL
    return OK


def mirror(rows, n, pheno, covar=None, counted=1, halvings=None):
    """-> (stats (nv, 6): OBS_CT, A1_FREQ, BETA, SE, Z, P at the kernel's stopping rule, NaN where undefined; err (nv,);
    passes (nv,)).  halvings: a list each fitted variant's number of halved steps is appended to."""
    pheno, covar, reg, q = _setup(n, pheno, covar)
    g, called = dosages(rows, n, counted)
    Q = np.zeros((n, q))
    Q[reg] = basis(np.concatenate([np.ones((int(reg.sum()), 1)), covar[reg]], axis=1))
    th0 = null_fit(Q[reg], pheno[reg])
    assert th0 is not None, "the null model does not converge"
    nv = g.shape[0]
    out = np.full((nv, 6), np.nan)
    err = np.zeros(nv, np.int32)
    passes = np.zeros(nv, np.int32)
    for v in range(nv):
        A = reg & called[v]
        obs = int(A.sum())
        out[v, 0] = obs
        ga, ya = g[v, A], pheno[A]
        if obs:
            out[v, 1] = ga.sum() / (2.0 * obs)
        err[v] = _flag(obs, ga, ya, q)
        if err[v]:
            continue
        X = np.concatenate([Q[A], (ga - nearest_integer_mean(ga.sum(), obs))[:, None]], axis=1)
        code, k, th, L = newton(X, ya, np.append(th0, 0.0), halvings=halvings)
        err[v], passes[v] = code, k
        if code == OK:
            beta, se = th[-1], 1.0 / L[-1, -1]
            out[v, 2:] = beta, se, beta / se, 2.0 * scipy.stats.norm.sf(abs(beta / se))
    return out, err, passes


def fit_full(X, y, tol=1e-14, max_iter=200):
    """Newton with step halving on the log-likelihood, until every step entry is <= tol max(1, |theta|), or the step
    is at the rounding floor of the N-term gradient (<= 1e-12 max(1, |theta|) and no longer halving from one step to
    the next; about 2e-14 at 21 845 samples) -> (theta, H, iterations) or None when it does not get there."""
    th = np.zeros(X.shape[1])
    l, g, H = evaluate(X, y, th)
    last = np.inf
    for it in range(1, max_iter + 1):
        step = np.linalg.solve(H, g)
        t = 1.0
        for _ in range(60):
            l2, g2, H2 = evaluate(X, y, th + t * step)
            if l2 >= l - 1e-12 * abs(l):
                break
            t *= 0.5
        th = th + t * step
        l, g, H = l2, g2, H2
        rel = float(np.max(np.abs(t * step) / np.maximum(1.0, np.abs(th))))
        if rel <= tol or (rel <= 1e-12 and rel > 0.5 * last):
            return th, H, it
        last = rel
    return None


def converged(rows, n, pheno, covar=None, counted=1, variants=None):
    """-> stats (nv, 6): OBS_CT, A1_FREQ, BETA, SE, Z, P of the fully converged fit (NaN where it is undefined or does
    not converge).  variants: fit only these (the others stay NaN past A1_FREQ)."""
    pheno, covar, reg, q = _setup(n, pheno, covar)
    g, called = dosages(rows, n, counted)
    nv = g.shape[0]
    out = np.full((nv, 6), np.nan)
    for v in range(nv) if variants is None else variants:
        A = reg & called[v]
        obs = int(A.sum())
        out[v, 0] = obs
        ga, ya, Ca = g[v, A], pheno[A], covar[A]
        if obs:
            out[v, 1] = ga.sum() / (2.0 * obs)
        if _flag(obs, ga, ya, q):
            continue
        X = np.concatenate([np.ones((obs, 1)), Ca - Ca.mean(axis=0),
                            (ga - nearest_integer_mean(ga.sum(), obs))[:, None]], axis=1)
        r = fit_full(X, ya)
        if r is None:
            continue
        th, H, _ = r
        se = float(np.sqrt(np.linalg.inv(H)[-1, -1]))
        z = th[-1] / se
        out[v, 2:] = th[-1], se, z, 2.0 * scipy.stats.norm.sf(abs(z))
    return out


class LogisticDouble:
    """NativePca.glmLogisticBegin / glmLogisticBed in numpy (mirror above), with the refusals of
    vpca_glm_logistic_begin."""

    def glmLogisticBegin(self, pheno, covar=None):
        from spark_examples_b200 import native
        y = np.asarray(pheno, np.float64)
        c = np.zeros((self.n, 0)) if covar is None else np.asarray(covar, np.float64).reshape(self.n, -1)
        bad = native.VpcaError(native.VPCA_ERR_BAD_ARG, "bad GLM input")
        if np.isinf(y).any() or np.isinf(c).any() or c.shape[1] + 1 > 32:
            raise bad
        f = y[np.isfinite(y)]
        if np.any((f != 0.0) & (f != 1.0)):
            raise bad
        reg = regression_samples(y, c)
        if reg.sum() < c.shape[1] + 3 or np.all(y[reg] == y[reg][0]):
            raise bad
        self.glm_logistic = (y, c)
        self.glm_calls = []
        return int(reg.sum())

    def glmLogisticBed(self, rows, counted=1):
        rows = np.asarray(rows)
        self.glm_calls.append(rows.shape[0])
        return mirror(rows, self.n, *self.glm_logistic, counted=counted)
