"""Host reference of the variance-standardized relationship matrix (DESIGN.md 13): the z table of each variant restated
in Python floats with the operations of csrc/grm.cu in the same order (so the bits must match), the same table in exact
rationals rounded once per step, and the GRM itself in numpy FP64.  Its top eigenpairs from the small eigh of Z^T Z
(Pcs), which never reads the device's GRM, and the checks a GRM solve must pass against them (check_grm_pairs).  Also
the .bed helpers and the Balding-Nichols cohorts the GRM tests share."""
from fractions import Fraction
import math

import numpy as np

from qc_ref import codes, counts

def z_table(h1, het, h2):
    """-> None for a skipped variant, else the four z values indexed by the .bed code (00, 01, 10, 11)."""
    n, a = h1 + het + h2, 2 * h1 + het
    if not 0 < a < 2 * n:
        return None
    a1 = a <= 2 * n - a
    r = a if a1 else 2 * n - a
    mu = r / n
    q = r / (2 * n)
    s = 1.0 / math.sqrt(mu * (1.0 - q))
    d_hom1, d_hom2 = (2.0, 0.0) if a1 else (0.0, 2.0)
    return ((d_hom1 - mu) * s, 0.0, (1.0 - mu) * s, (d_hom2 - mu) * s)


def _rn(x: Fraction) -> float:
    return float(x)   # Fraction -> float rounds to nearest even once


def _sqrt_rn(x: float) -> float:
    """The correctly rounded square root, by exact comparison of the neighbours of math.sqrt's candidate."""
    fx = Fraction(x)
    best = None
    c = math.sqrt(x)
    for cand in (math.nextafter(c, 0.0), c, math.nextafter(c, math.inf)):
        err = abs(Fraction(cand) ** 2 - fx)
        if best is None or err < best[0]:
            best = (err, cand)
    return best[1]


def z_table_exact(h1, het, h2):
    """z_table with every step an exact rational rounded once to a double."""
    n, a = h1 + het + h2, 2 * h1 + het
    if not 0 < a < 2 * n:
        return None
    a1 = a <= 2 * n - a
    r = a if a1 else 2 * n - a
    mu = _rn(Fraction(r, n))
    q = _rn(Fraction(r, 2 * n))
    one_q = _rn(1 - Fraction(q))
    prod = _rn(Fraction(mu) * Fraction(one_q))
    s = _rn(1 / Fraction(_sqrt_rn(prod)))
    d_hom1, d_hom2 = (2, 0) if a1 else (0, 2)
    z = lambda d: _rn(Fraction(_rn(d - Fraction(mu))) * Fraction(s))
    return (z(d_hom1), 0.0, z(1), z(d_hom2))


def z_tables(c):
    """z_table of (nv, 4) counts, vectorised with the same numpy float64 operations -> (tab (nv, 4), used (nv,) bool)."""
    c = np.asarray(c, np.int64)
    n, a = c[:, 0] + c[:, 1] + c[:, 2], 2 * c[:, 0] + c[:, 1]
    used = (a > 0) & (a < 2 * n)
    a1 = a <= 2 * n - a
    r = np.where(a1, a, 2 * n - a).astype(np.float64)
    nn = np.where(used, n, 1).astype(np.float64)
    mu = r / nn
    q = r / (2.0 * nn)
    with np.errstate(divide="ignore", invalid="ignore"):   # unused variants: overwritten with 0 below
        s = 1.0 / np.sqrt(mu * (1.0 - q))
        tab = np.stack([(np.where(a1, 2.0, 0.0) - mu) * s, np.zeros_like(mu), (1.0 - mu) * s,
                        (np.where(a1, 0.0, 2.0) - mu) * s], axis=1)
    tab[~used] = 0.0
    return tab, used


def z_matrix(rows, n):
    """(nv, stride) .bed rows -> (Z (n, M) float64 of the used variants in row order, used (nv,) bool)."""
    tab, used = z_tables(counts(rows, n))
    code = codes(rows, n).astype(np.int64)
    Z = np.take_along_axis(tab, code, axis=1)[used].T
    return np.ascontiguousarray(Z), used


def grm(rows, n):
    """-> (G (n, n) float64 = Z Z^T / M in numpy FP64, M, Z)."""
    Z, used = z_matrix(rows, n)
    M = Z.shape[1]
    return (Z @ Z.T) / M if M else np.zeros((n, n)), M, Z


def tolerance(Z, panel=1024):
    """Cellwise bound on |G_device - G_numpy| (DESIGN.md 13): (|Z| |Z|^T / M) times the summation depth of both sums in
    units of the double rounding error, plus one rounding of the division."""
    n, M = Z.shape
    A = np.abs(Z)
    return depth(M, panel) * 2.0 ** -53 * (A @ A.T) / max(M, 1)


def depth(M, panel=1024):
    """The summation depth of tolerance(), in units of the double rounding error."""
    return panel + -(-M // panel) + 2 * (256 + -(-M // 256)) + 4


class Pcs:
    """FP64 top-k eigenpairs of G = Z Z^T / M that never read the device's GRM: the small eigh of Z^T Z / M (M x M), or
    of Z Z^T / M when N < M, then u = Z w / sqrt(M lambda).  Z is (N, M) numpy, or a torch float64 tensor (on the GPU
    for large N).  Residuals G u - lambda u = Z (Z^T u) / M - lambda u cost O(N M) without forming G.

    lam: the top k eigenvalues (zeros past min(N, M)); rank: how many of them are nonzero (above 1e-9 lam[0]); U: (N, rank)
    numpy, their unit eigenvectors."""

    def __init__(self, Z, k):
        self.Z = Z
        self.n, self.M = n, M = Z.shape
        small = (Z.T @ Z if n >= M else Z @ Z.T) / M
        if isinstance(Z, np.ndarray):
            import scipy.linalg
            self._np = lambda a: a
            d = small.shape[0]
            w, W = scipy.linalg.eigh(small, subset_by_index=[max(0, d - k), d - 1])
        else:
            import torch
            self._np = lambda a: a.cpu().numpy()
            w, W = map(self._np, torch.linalg.eigh(small))
        del small
        order = np.argsort(-w, kind="stable")[:k]
        self.lam = np.zeros(k)
        self.lam[:len(order)] = w[order]
        self.rank = int((self.lam > 1e-9 * self.lam[0]).sum())
        W = W[:, order[:self.rank]]
        self.U = self._np(Z @ self._like(W)) / np.sqrt(M * self.lam[:self.rank])[None, :] if n >= M else W
        self.fro2 = float((Z * Z).sum())

    def _like(self, a):
        """numpy -> Z's kind (and device)"""
        a = np.ascontiguousarray(a, np.float64)
        if isinstance(self.Z, np.ndarray):
            return a
        import torch
        return torch.from_numpy(a).to(self.Z.device)

    def gaps_allow(self, k):
        """the top k + 1 eigenvalues are far enough apart for two solvers' vectors to agree to 1e-8"""
        return k >= len(self.lam) or np.min(np.abs(np.diff(self.lam[: k + 1]))) / self.lam[0] > 1e-4

    def residuals(self, vecs, evals):
        """||G u - lambda u|| / lambda_1 per column, G u = Z (Z^T u) / M"""
        u = self._like(vecs)
        r = self._np(self.Z @ (self.Z.T @ u) / self.M - u * self._like(evals)[None, :])
        return np.linalg.norm(r, axis=0) / self.lam[0]

    def residual_bound(self):
        """1e-11 plus the device GRM's own cellwise error (tolerance()) in Frobenius norm, || |Z| |Z|^T ||_F <= ||Z||_F^2,
        relative to lambda_1"""
        return 1e-11 + depth(self.M) * 2.0 ** -53 * self.fro2 / (self.M * self.lam[0])


def check_grm_pairs(ref, vecs, evals, k, note=""):
    """The assertions every GRM solve must meet against the Z^T Z reference.  Pairs past ref.rank belong to a zero
    eigenvalue: |lambda| <= 1e-12 lambda_1 and the vector orthogonal to every nonzero pair's."""
    from oracle import oracle
    r = min(ref.rank, k)
    assert vecs.shape == (ref.n, k) and evals.shape == (k,), note
    assert np.all(np.isfinite(vecs)) and np.all(np.isfinite(evals)), note
    assert np.allclose(evals[:r], ref.lam[:r], rtol=1e-10, atol=0), (note, evals, ref.lam[:k])
    assert np.all(np.abs(evals[r:]) <= 1e-12 * ref.lam[0]), (note, evals, ref.lam[:k])
    if r:
        err = oracle.eigvec_rel_err(vecs[:, :r], ref.U[:, :r])
        assert np.all(err <= 1e-6), (note, err)
    if r < k:
        leak = np.abs(ref.U.T @ vecs[:, r:])
        assert leak.max() <= 1e-8, (note, leak.max())
    res = ref.residuals(vecs, evals)
    assert np.all(res <= ref.residual_bound()), (note, res, ref.residual_bound())
    assert np.abs(vecs.T @ vecs - np.eye(k)).max() <= 1e-10, note
    assert np.allclose(np.linalg.norm(vecs, axis=0), 1.0, rtol=0, atol=1e-12), note
    for c in range(k):
        assert vecs[np.argmax(np.abs(vecs[:, c])), c] > 0, (note, c)   # sign rule: largest-|.| entry (lowest index) positive


class Solve:
    """computePcaGrm(k) on a context, with the path it took: eig_method (1 direct, 2 Lanczos, 3 Lanczos gave up and the
    direct reduction ran), eig_iterations and the kernel_launches delta of the call."""

    def __init__(self, nat, k):
        before = nat.stats()
        self.vecs, self.evals = nat.computePcaGrm(k)
        after = nat.stats()
        self.method = after["eig_method"]
        self.iters = after["eig_iterations"]
        self.launches = after["kernel_launches"] - before["kernel_launches"]

    def __repr__(self):
        return f"Solve(method={self.method}, iters={self.iters}, launches={self.launches})"


def assert_path(s, method, n):
    """The solve took the path claimed.  Band Lanczos (2): norm, scale, tile, reduce, combine and two lz_dots / lz_update
    pairs, nine launches per step.  Direct (1): ceil(n / 64) replays of the 64-step graph (one launch per step up to
    n = 3072, two above), then bisection, inverse iteration and the back-transformation; a GRM needs no centring."""
    assert s.method == method, s
    if method == 2:
        assert 16 <= s.iters <= 320 and s.launches >= 9 * s.iters, s
    elif method == 1:
        assert s.iters == 0 and s.launches == (1 if n <= 3072 else 2) * 64 * -(-n // 64) + 3, s


def pack(code):
    """(nv, n) 2-bit codes -> (nv, ceil(n / 4)) .bed rows, padding bits 0."""
    code = np.asarray(code, dtype=np.uint8)
    nv, n = code.shape
    pad = (-n) % 4
    c = np.concatenate([code, np.zeros((nv, pad), np.uint8)], axis=1).reshape(nv, -1, 4)
    return (c[..., 0] | (c[..., 1] << 2) | (c[..., 2] << 4) | (c[..., 3] << 6)).astype(np.uint8)


def dosage_codes(d, missing=None):
    """A1 dosages (2, 1, 0) -> .bed codes (00, 10, 11); missing calls (mask) -> 01."""
    code = np.where(d == 2, 0, np.where(d == 1, 2, 3)).astype(np.uint8)
    if missing is not None:
        code[missing] = 1
    return code


def balding_nichols(rng, n, nv, pops=3, miss=0.0):
    """(nv, n) .bed codes of `pops` populations under the Balding-Nichols model, as tests/eig_ref.structured_cells draws
    them: ancestral frequency p = 0.05 + 0.45 u, population i's frequency from Beta(p (1 - F) / F, (1 - p) (1 - F) / F)
    with F running linearly from 0.20 down to 0.04, a share of the samples proportional to 1.12^i (so the top eigenvalues
    stand apart), A1 dosages ~ Binomial(2, p_i); `miss` of the calls missing at random."""
    share = 1.12 ** np.arange(pops)
    sizes = np.floor(n * share / share.sum()).astype(np.int64)
    sizes[np.argsort(-(n * share / share.sum() - sizes))[: n - sizes.sum()]] += 1
    anc = 0.05 + 0.45 * rng.random(nv)
    d = np.empty((nv, n), np.uint8)
    col = 0
    for i, fst in enumerate(np.linspace(0.20, 0.04, pops)):
        q = (1.0 - fst) / fst
        p = rng.beta(anc * q, (1.0 - anc) * q)
        d[:, col:col + sizes[i]] = rng.binomial(2, p[:, None], (nv, sizes[i]))
        col += sizes[i]
    return dosage_codes(d, rng.random((nv, n)) < miss if miss > 0 else None)
