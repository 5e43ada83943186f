"""numpy restatement of variant loadings and projection (DESIGN.md 6), shared by the projection tests.

loadings:   W = X^T U (variants x k), count = column sums of X
projection: P = (Y - count / n_ref) W / lambda  (Y: new samples x the same variants)
"""
import numpy as np


def np_loadings(X, U):
    """X: (N samples, V variants) small integers; U: (N, k).  -> (W (V, k) float64, count (V,) int32)."""
    X64 = np.asarray(X, np.float64)
    return X64.T @ np.asarray(U, np.float64), np.asarray(X, np.int64).sum(axis=0).astype(np.int32)


def np_project(Y, W, count, n_ref, evals):
    """Y: (M, V) cells of the new samples, aligned with the rows of W (V, k) and count (V,). -> (M, k)."""
    mean = np.asarray(count, np.float64) / float(n_ref)
    return ((np.asarray(Y, np.float64) - mean[None, :]) @ np.asarray(W, np.float64)) / np.asarray(evals, np.float64)[None, :]


def dense_to_csr(X):
    """(N, V) multiplicities -> CSR rows (offsets int64, sample indices int32), a sample listed m times for m."""
    Xt = np.asarray(X, np.int64).T
    counts = Xt.sum(axis=1)
    off = np.zeros(Xt.shape[0] + 1, np.int64)
    np.cumsum(counts, out=off[1:])
    idx = []
    for v in range(Xt.shape[0]):
        nz = np.nonzero(Xt[v])[0]
        idx.append(np.repeat(nz, Xt[v, nz]))
    return off, (np.concatenate(idx) if idx else np.zeros(0, np.int64)).astype(np.int32)
