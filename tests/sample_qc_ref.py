"""numpy restatement of the sample QC calls (vpca_sample_missing_bed, vpca_subset_bed_samples) for the tests: the missing
calls of every sample over PLINK .bed rows, and the rows repacked to a subset of their samples with zero padding bits."""
import numpy as np

MISSING = 1   # .bed code 01


def _codes(rows: np.ndarray, n: int) -> np.ndarray:
    """(nv, stride) uint8 .bed rows -> (nv, n) codes (low bits first); bytes past ceil(n / 4) are not read."""
    rows = np.asarray(rows, np.uint8)[:, : (n + 3) // 4]
    return np.stack([(rows >> s) & 3 for s in (0, 2, 4, 6)], axis=-1).reshape(rows.shape[0], -1)[:, :n]


def _pack(codes: np.ndarray) -> np.ndarray:
    """(nv, m) codes -> (nv, ceil(m / 4)) .bed rows, padding codes 00 as PLINK writes them."""
    codes = np.asarray(codes, np.uint8)
    nv, m = codes.shape
    pad = (-m) % 4
    if pad:
        codes = np.concatenate([codes, np.zeros((nv, pad), np.uint8)], axis=1)
    c4 = codes.reshape(nv, -1, 4)
    return (c4[:, :, 0] | (c4[:, :, 1] << 2) | (c4[:, :, 2] << 4) | (c4[:, :, 3] << 6)).astype(np.uint8)


def missing_counts(rows: np.ndarray, n: int, block: int = 256) -> np.ndarray:
    """(n,) int64: rows where each sample has code 01."""
    rows = np.asarray(rows, np.uint8)
    out = np.zeros(n, np.int64)
    for v0 in range(0, rows.shape[0], block):
        out += (_codes(rows[v0:v0 + block], n) == MISSING).sum(axis=0)
    return out


def subset_rows(rows: np.ndarray, n: int, keep_idx, block: int = 256) -> np.ndarray:
    """(nv, ceil(m / 4)) uint8: each row with the codes of samples keep_idx, in that order, packed."""
    rows = np.asarray(rows, np.uint8)
    idx = np.asarray(keep_idx, np.int64)
    out = np.empty((rows.shape[0], (len(idx) + 3) // 4), np.uint8)
    for v0 in range(0, rows.shape[0], block):
        out[v0:v0 + block] = _pack(_codes(rows[v0:v0 + block], n)[:, idx])
    return out
