"""numpy restatement of LD pruning (vpca_ld_prune_bed, DESIGN.md 9) for the tests: .bed rows decoded to A1 counts, the
six exact sums of every pair by integer matrix products, r2 with the library's three rounded double operations, the
window starts from contig and position, and the keep-first sweep."""
import numpy as np

MISSING = 1                                   # .bed code 01


def decode(rows: np.ndarray, n: int):
    """(nv, stride) uint8 .bed rows -> D (nv, n) int64 A1 counts (00 -> 2, 10 -> 1, 11 -> 0; 0 when missing) and
    M (nv, n) int64, 1 where called."""
    rows = np.asarray(rows, np.uint8)
    codes = np.stack([(rows >> s) & 3 for s in (0, 2, 4, 6)], axis=-1).reshape(rows.shape[0], -1)[:, :n]
    D = np.choose(codes, [2, 0, 1, 0]).astype(np.int64)
    M = (codes != MISSING).astype(np.int64)
    return D, M


def _imatmul(a: np.ndarray, b: np.ndarray) -> np.ndarray:
    """Exact integer product a @ b.T of small non-negative integer matrices, through float64 BLAS: every entry is at
    most 4 n < 2^53, so each partial sum is an exact integer and the result is the integer product."""
    return np.rint(a.astype(np.float64) @ b.astype(np.float64).T).astype(np.int64)


def sums(D: np.ndarray, M: np.ndarray, rows_i, rows_j):
    """The six sums of the pairs (i, j) for i in rows_i, j in rows_j: (n, Sx, Sy, Sxx, Syy, Sxy), each (|i|, |j|) int64,
    x the counts of i, y those of j, over the samples called at both."""
    Di, Mi, Dj, Mj = D[rows_i], M[rows_i], D[rows_j], M[rows_j]
    return (_imatmul(Mi, Mj), _imatmul(Di, Mj), _imatmul(Mi, Dj), _imatmul(Di * Di, Mj), _imatmul(Mi, Dj * Dj),
            _imatmul(Di, Dj))


def r2_of(n, sx, sy, sxx, syy, sxy):
    """-> (r2 float64, defined bool): cov^2 / (vx vy) from exact int64, each double operation rounded once; defined where
    both variances are positive (r2 is 0 elsewhere)."""
    n, sx, sy, sxx, syy, sxy = (np.asarray(v, np.int64) for v in (n, sx, sy, sxx, syy, sxy))
    cov = n * sxy - sx * sy
    vx = n * sxx - sx * sx
    vy = n * syy - sy * sy
    ok = (vx > 0) & (vy > 0)
    c = cov.astype(np.float64)
    with np.errstate(divide="ignore", invalid="ignore"):
        r2 = (c * c) / (vx.astype(np.float64) * vy.astype(np.float64))
    return np.where(ok, r2, 0.0), ok


def r2_matrix(D, M):
    """(nv, nv) r2 of every pair and where it is defined (entry [i, j]: x = variant i)."""
    idx = np.arange(D.shape[0])
    return r2_of(*sums(D, M, idx, idx))


def window_starts(contigs, positions, kb: float) -> np.ndarray:
    """window_lo[j]: the first i <= j on j's contig with pos_j - pos_i <= kb * 1000 (a plain scan; assumes sorted input)."""
    v = len(positions)
    lo = np.zeros(v, np.int64)
    for j in range(v):
        i = j
        while i > 0 and contigs[i - 1] == contigs[j] and positions[j] - positions[i - 1] <= kb * 1000:
            i -= 1
        lo[j] = i
    return lo


def ld_pairs(D, M, window_lo, r2_max: float, block: int = 256):
    """Every in-LD pair (i, j), window_lo[j] <= i < j, in order of j then i -> (pairs (P, 2) int64, r2 (P,))."""
    v = D.shape[0]
    out_p, out_r = [], []
    for j0 in range(0, v, block):
        j1 = min(v, j0 + block)
        lo = int(np.min(window_lo[j0:j1])) if j1 > j0 else j0
        ii = np.arange(lo, j1)
        jj = np.arange(j0, j1)
        r2, ok = r2_of(*sums(D, M, ii, jj))
        sel = ok & (r2 > r2_max) & (ii[:, None] < jj[None, :]) & (ii[:, None] >= np.asarray(window_lo)[jj][None, :])
        js, is_ = np.nonzero(sel.T)                    # by j, then i
        out_p.append(np.stack([ii[is_], jj[js]], axis=1))
        out_r.append(r2.T[js, is_])
    if not out_p:
        return np.zeros((0, 2), np.int64), np.zeros(0)
    return np.concatenate(out_p).astype(np.int64), np.concatenate(out_r)


def sweep(v: int, pairs) -> np.ndarray:
    """Keep-first: in order, j is kept iff no kept i among its in-LD partners (i < j, in j's window)."""
    partners = [[] for _ in range(v)]
    for i, j in np.asarray(pairs, np.int64).reshape(-1, 2).tolist():
        partners[j].append(i)
    keep = np.zeros(v, bool)
    for j in range(v):
        keep[j] = not any(keep[i] for i in partners[j])
    return keep


def prune(rows, n: int, window_lo, r2_max: float):
    """The whole pipeline -> (keep, pairs, r2) as vpca_ld_prune_bed computes them."""
    D, M = decode(rows, n)
    pairs, r2 = ld_pairs(D, M, np.asarray(window_lo, np.int64), r2_max)
    return sweep(D.shape[0], pairs), pairs, r2
