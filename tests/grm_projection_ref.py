"""Host reference of the GRM loadings and projection (DESIGN.md 14) in numpy FP64, with the error bounds the tests use:
a recursive sum of m products has error at most (m + 1) u sum |products| (u = 2^-53), counted once for the device and
once for the reference."""
import numpy as np

from grm_ref import z_tables
from qc_ref import codes, counts

U_RND = 2.0 ** -53


def z_full(rows, n, tab=None):
    """(n, nv) z values of every row (unused variants and missing calls 0), through `tab` or the rows' own tables."""
    if tab is None:
        tab, _ = z_tables(counts(rows, n))
    code = codes(rows, n).astype(np.int64)
    return np.ascontiguousarray(np.take_along_axis(np.asarray(tab, np.float64), code, axis=1).T)


def loadings(rows, n, U):
    """-> (W = Z^T U (nv, k), tab (nv, 4), bound (nv, k) on |W_device - W|)."""
    tab, _ = z_tables(counts(rows, n))
    Z = z_full(rows, n, tab)
    W = Z.T @ U
    bound = 2.0 * (n + 1) * U_RND * (np.abs(Z).T @ np.abs(U))
    return W, tab, bound


def projection(rows, n, tab, W):
    """Raw sums Y W (n, k) of rows (nv, stride) of n samples through the reference tables, and the bound on the device's
    raw sums."""
    Y = z_full(rows, n, tab)
    nv = Y.shape[1]
    return Y @ W, 2.0 * (nv + 1) * U_RND * (np.abs(Y) @ np.abs(W))


def round_trip_bound(Z, U, evals, M):
    """Bound on |p - u| for the reference's own samples projected with loadings computed on the device: the residual
    |G u - lambda u| / lambda (G = Z Z^T / M, formed without G), plus the summation error of the loadings carried through
    the projection and of the projection itself."""
    A = np.abs(Z)
    res = np.abs(Z @ (Z.T @ U) / M - U * evals[None, :]) / evals[None, :]
    n, nv = Z.shape
    summ = 2.0 * (n + nv + 2) * U_RND * (A @ (A.T @ np.abs(U))) / (M * evals[None, :])
    return res.max(axis=0) + summ
