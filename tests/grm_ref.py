"""Host reference of the variance-standardized relationship matrix (DESIGN.md 13): the z table of each variant restated
in Python floats with the operations of csrc/grm.cu in the same order (so the bits must match), the same table in exact
rationals rounded once per step, and the GRM itself in numpy FP64.  Also the .bed helpers and the Balding-Nichols
cohorts the GRM tests share."""
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
    u = 2.0 ** -53
    depth = panel + -(-M // panel) + 2 * (256 + -(-M // 256)) + 4
    return depth * u * (A @ A.T) / max(M, 1)


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
