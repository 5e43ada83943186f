"""Host reference of the Firth-penalized logistic tests (DESIGN.md 17), in two parts.

`mirror`: the kernel's iteration in numpy, on the basis of glm_logistic_ref.mirror (Q, the null fit, the centred
dosage, the start (theta_null, 0)).  Each pass evaluates l and H = X^T W X at the trial point, factors H = L L^T and
takes the penalized log-likelihood l* = l + sum log L_jj (walk A), then the Firth score
U* = sum x_i (y_i - mu_i + h_i (1/2 - mu_i)) with h_i = w_i ||L^-1 x_i||^2 (walk B).  The step rule:
  - a trial point theta_prev + t Delta is backtracked by t <- t / 2 when l is not finite, a pivot of H is <= 0 or l* fell
    by more than 1e-10 |l*_prev|; else by the secant t <- t s0 / (s0 - s1) when s1 = U*^T Delta < -0.45 s0,
    s0 = delta^2_prev (the directional derivative of l* along Delta crossed zero well before t);
  - an accepted point takes z = L^-1 U*, delta^2 = z^T z, Delta = L^-T z, and stops at delta^2 <= 1e-18, reporting
    BETA = beta + Delta_g and SE = 1 / L_gg; otherwise the next trial point is at t = min(1, MAX_DELTA / delta);
  - at most MAX_BACKTRACK backtracks in a row and MAX_PASS passes (backtracked ones included).
It gives the ERRCODE and the pass count of every variant, and in `fallback` mode which variants the Firth fit replaces.

`converged`: the same penalized fit on the centred raw design [1, covar - mean, g'] of glm_logistic_ref.converged,
iterated until the step is at its rounding floor; BETA, SE = sqrt([H^-1]_gg) of the unpenalized information at the
fit, Z and P = 2 norm.sf(|Z|).  test_glm_firth_cpu checks both against scipy.optimize on -l*.

Also a numpy double of NativePca.glmFirthBed for the driver tests."""
import numpy as np
import scipy.linalg
import scipy.stats

import glm_logistic_ref as lref
from glm_ref import dosages, nearest_integer_mean

OK, VIF_INFINITE, CONVERGE_FAIL, FIRTH_FAIL = 0, 3, 5, 6
ERRCODES = lref.ERRCODES + ("FIRTH_CONVERGE_FAIL",)
FALLBACK, ALWAYS = 1, 2
MAX_PASS, MAX_BACKTRACK, DELTA2, FALL, PIVOT_MIN, MAX_DELTA, SECANT = 100, 30, 1e-18, 1e-10, 1e-10, 5.0, 0.45


def walk_a(X, y, theta, first):
    """l, the factor L of H (None when a pivot fails) and l* at theta.  first: the first pass's VIF rule (a pivot
    <= PIVOT_MIN H_jj is VIF_INFINITE) -> (l, L, lstar, code)."""
    l, _, H = lref.evaluate(X, y, theta)
    if not np.isfinite(l):
        return l, None, None, FIRTH_FAIL
    L, code = lref.cholesky(H, first)
    if code:
        return l, None, None, code if first else FIRTH_FAIL
    return l, L, l + float(np.sum(np.log(np.diag(L)))), OK


def walk_b(X, y, theta, L):
    """The Firth score U* at theta, with h_i = w_i ||L^-1 x_i||^2 through the explicit inverse of L."""
    eta = X @ theta
    e = np.exp(-np.abs(eta))
    rd = 1.0 / (1.0 + e)
    mu = np.where(eta >= 0.0, rd, e * rd)
    w = e * rd * rd
    Li = scipy.linalg.solve_triangular(L, np.eye(len(L)), lower=True)
    h = w * np.sum((X @ Li.T) ** 2, axis=1)
    return X.T @ (y - mu + h * (0.5 - mu))


def firth(X, y, theta0, max_pass=MAX_PASS, max_backtrack=MAX_BACKTRACK, delta2=DELTA2, stats=None):
    """The kernel's passes from theta0 -> (code, passes, theta + the last step, the last L).  stats: a dict that counts
    the backtracks by kind ('halve', 'secant') and keeps 'margin', the least |s1 / s0 + SECANT| of the fit."""
    th = np.array(theta0, np.float64)
    thp = dl = None
    lsp = s0 = 0.0
    t, bt = 1.0, 0
    for k in range(1, max_pass + 1):
        l, L, ls, code = walk_a(X, y, th, k == 1)
        if k == 1 and code:
            return code, k, None, None
        kind = None
        if k > 1 and (code or ls < lsp - FALL * abs(lsp)):
            kind = "halve"
        else:
            us = walk_b(X, y, th, L)
            if k > 1:
                s1 = float(us @ dl)
                if stats is not None:
                    stats["margin"] = min(stats.get("margin", np.inf), abs(s1 / s0 + SECANT))
                if s1 < -SECANT * s0:
                    kind = "secant"
        if kind is not None:
            if bt == max_backtrack or k == max_pass:
                return FIRTH_FAIL, k, None, None
            bt += 1
            t = 0.5 * t if kind == "halve" else t * s0 / (s0 - s1)
            th = thp + t * dl
            if stats is not None:
                stats[kind] = stats.get(kind, 0) + 1
            continue
        z = scipy.linalg.solve_triangular(L, us, lower=True)
        dd = float(z @ z)
        step = scipy.linalg.solve_triangular(L.T, z, lower=False)
        if not np.isfinite(dd):
            return FIRTH_FAIL, k, None, None
        if dd <= delta2:
            return OK, k, th + step, L
        if k == max_pass:
            return FIRTH_FAIL, k, None, None
        t = MAX_DELTA / np.sqrt(dd) if dd > MAX_DELTA * MAX_DELTA else 1.0
        lsp, s0, thp, dl, bt = ls, dd, th, step, 0
        th = thp + t * dl
    return FIRTH_FAIL, max_pass, None, None


def _design(Q, A, ga, obs):
    return np.concatenate([Q[A], (ga - nearest_integer_mean(ga.sum(), obs))[:, None]], axis=1)


def mirror(rows, n, pheno, covar=None, counted=1, mode=ALWAYS, stats=None):
    """-> (stats (nv, 6): OBS_CT, A1_FREQ, BETA, SE, Z, P at the kernels' stopping rules, NaN where undefined; err (nv,);
    passes (nv,) of the fit reported; firth (nv,) uint8, 1 where the Firth fit ran).  mode FALLBACK: the maximum-likelihood
    mirror of glm_logistic_ref, and the Firth fit for the variants it ends with LOGISTIC_CONVERGE_FAIL after at least one
    pass; ALWAYS: the Firth fit for every variant that passes the ERRCODE checks before the first pass."""
    pheno, covar, reg, q = lref._setup(n, pheno, covar)
    g, called = dosages(rows, n, counted)
    Q = np.zeros((n, q))
    Q[reg] = lref.basis(np.concatenate([np.ones((int(reg.sum()), 1)), covar[reg]], axis=1))
    th0 = lref.null_fit(Q[reg], pheno[reg])
    assert th0 is not None, "the null model does not converge"
    if mode == FALLBACK:
        out, err, passes = lref.mirror(rows, n, pheno, covar, counted=counted)
        todo = np.flatnonzero((err == CONVERGE_FAIL) & (passes > 0))
    else:
        nv = g.shape[0]
        out = np.full((nv, 6), np.nan)
        err = np.zeros(nv, np.int32)
        passes = np.zeros(nv, np.int32)
        todo = []
        for v in range(nv):
            A = reg & called[v]
            obs = int(A.sum())
            out[v, 0] = obs
            if obs:
                out[v, 1] = g[v, A].sum() / (2.0 * obs)
            err[v] = lref._flag(obs, g[v, A], pheno[A], q)
            if err[v] == OK:
                todo.append(v)
    firth_flag = np.zeros(len(err), np.uint8)
    for v in todo:
        A = reg & called[v]
        ga = g[v, A]
        code, k, th, L = firth(_design(Q, A, ga, int(A.sum())), pheno[A], np.append(th0, 0.0), stats=stats)
        err[v], passes[v], firth_flag[v] = code, k, 1
        out[v, 2:] = np.nan
        if code == OK:
            beta, se = th[-1], 1.0 / L[-1, -1]
            out[v, 2:] = beta, se, beta / se, 2.0 * scipy.stats.norm.sf(abs(beta / se))
    return out, err, passes, firth_flag


def converged(rows, n, pheno, covar=None, counted=1, variants=None):
    """-> stats (nv, 6): OBS_CT, A1_FREQ, BETA, SE, Z, P of the fully converged Firth fit on [1, covar - mean, g'] (NaN
    where undefined or where it does not get there).  variants: fit only these."""
    pheno, covar, reg, q = lref._setup(n, pheno, covar)
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
        if lref._flag(obs, ga, ya, q):
            continue
        X = np.concatenate([np.ones((obs, 1)), Ca - Ca.mean(axis=0),
                            (ga - nearest_integer_mean(ga.sum(), obs))[:, None]], axis=1)
        th = fit_full(X, ya)
        if th is None:
            continue
        _, _, H = lref.evaluate(X, ya, th)
        se = float(np.sqrt(np.linalg.inv(H)[-1, -1]))
        z = th[-1] / se
        out[v, 2:] = th[-1], se, z, 2.0 * scipy.stats.norm.sf(abs(z))
    return out


def fit_full(X, y, max_iter=400):
    """The penalized maximum from 0 by the mirror's rule, to a Newton decrement of 1e-12 (six orders below the mirror's,
    above the rounding floor of about sqrt(N) u) -> theta, or None."""
    code, _, th, _ = firth(X, y, np.zeros(X.shape[1]), max_pass=max_iter, max_backtrack=60, delta2=1e-24)
    return th if code == OK else None


def penalized(X, y, theta):
    """-l*(theta) and -U*(theta) of the raw design, for scipy.optimize."""
    _, L, ls, code = walk_a(X, y, theta, False)
    if code:
        return np.inf, np.zeros_like(theta)
    return -ls, -walk_b(X, y, theta, L)


class FirthDouble:
    """NativePca.glmFirthBed in numpy (mirror above), on the state of glm_logistic_ref.LogisticDouble."""

    def glmFirthBed(self, rows, counted=1, mode="fallback"):
        rows = np.asarray(rows)
        self.glm_calls.append(rows.shape[0])
        self.firth_modes = getattr(self, "firth_modes", []) + [mode]
        return mirror(rows, self.n, *self.glm_logistic, counted=counted,
                      mode={"fallback": FALLBACK, "always": ALWAYS}[mode])
