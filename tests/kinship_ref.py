"""numpy restatement of KING-robust kinship (Manichaikul et al., Bioinformatics 26:2867, 2010; PLINK 2's
--make-king-table) for the tests: integer counts per sample pair from PLINK .bed rows, then one double division."""
import numpy as np

HET, HOM_A1, HOM_A2, MISSING = 2, 0, 3, 1     # .bed 2-bit codes


def bed_codes(rows: np.ndarray, n: int) -> np.ndarray:
    """(nv, stride) uint8 .bed rows -> (nv, n) codes (low bits first)."""
    rows = np.asarray(rows, np.uint8)
    return np.stack([(rows >> s) & 3 for s in (0, 2, 4, 6)], axis=-1).reshape(rows.shape[0], -1)[:, :n]


def pack_codes(codes: np.ndarray) -> np.ndarray:
    """(nv, n) codes -> (nv, ceil(n / 4)) .bed rows, padding samples 00 like PLINK."""
    codes = np.asarray(codes, np.uint8)
    nv, n = codes.shape
    pad = (-n) % 4
    if pad:
        codes = np.concatenate([codes, np.zeros((nv, pad), np.uint8)], axis=1)
    c4 = codes.reshape(nv, -1, 4)
    return (c4[:, :, 0] | (c4[:, :, 1] << 2) | (c4[:, :, 2] << 4) | (c4[:, :, 3] << 6)).astype(np.uint8)


def dosage_codes(dosage_a1: np.ndarray) -> np.ndarray:
    """(n, nv) A1 allele counts in {0, 1, 2}, -1 missing -> (nv, n) .bed codes."""
    d = np.asarray(dosage_a1).T
    c = np.full(d.shape, MISSING, np.uint8)
    c[d == 2] = HOM_A1
    c[d == 1] = HET
    c[d == 0] = HOM_A2
    return c


def count_matrices(codes: np.ndarray):
    """(nv, n) codes -> n x n int64 matrices (entry [a, b]): NSNP, HETHET, IBS0, HET1_HOM2 (a het, b hom)."""
    c = np.asarray(codes).T
    H = (c == HET).astype(np.float64)
    P1 = (c == HOM_A1).astype(np.float64)
    P2 = (c == HOM_A2).astype(np.float64)
    called = H + P1 + P2
    as_int = lambda m: np.rint(m).astype(np.int64)      # float64 products of 0/1 matrices below 2^53 are exact
    nsnp = as_int(called @ called.T)
    hethet = as_int(H @ H.T)
    ibs0 = as_int(P1 @ P2.T + P2 @ P1.T)
    het1_hom2 = as_int(H @ (P1 + P2).T)
    return nsnp, hethet, ibs0, het1_hom2


def kinship_value(hethet, ibs0, het1, het2):
    """(HETHET - 2 IBS0) / (2 HETHET + HET1_HOM2 + HET2_HOM1) from exact int64, NaN where the denominator is 0."""
    num = np.asarray(hethet, np.int64) - 2 * np.asarray(ibs0, np.int64)
    den = 2 * np.asarray(hethet, np.int64) + np.asarray(het1, np.int64) + np.asarray(het2, np.int64)
    with np.errstate(divide="ignore", invalid="ignore"):
        k = num.astype(np.float64) / den.astype(np.float64)
    return np.where(den == 0, np.nan, k)


def king_pairs(codes: np.ndarray, min_kinship: float = -np.inf):
    """Every pair a < b ordered by b, then a -> (ids (P, 2), counts (P, 5) NSNP, HETHET, IBS0, HET1_HOM2, HET2_HOM1,
    kinship (P,)), filtered like vpca_kinship_pairs (-inf: all pairs, NaN included; else KINSHIP >= min, NaN never)."""
    n = np.asarray(codes).shape[1]
    nsnp, hethet, ibs0, h1 = count_matrices(codes)
    b, a = np.tril_indices(n, -1)                      # row-major lower triangle: by b, then a
    counts = np.stack([nsnp[a, b], hethet[a, b], ibs0[a, b], h1[a, b], h1[b, a]], axis=1)
    kin = kinship_value(counts[:, 1], counts[:, 2], counts[:, 3], counts[:, 4])
    keep = np.ones(len(kin), bool) if np.isneginf(min_kinship) else (kin >= min_kinship)
    ids = np.stack([a, b], axis=1)
    return ids[keep].astype(np.int32), counts[keep].astype(np.int32), kin[keep]


def pair_counts(codes: np.ndarray, a: int, b: int):
    """The five counts of one pair straight from the two sample columns."""
    ca, cb = np.asarray(codes)[:, a], np.asarray(codes)[:, b]
    both = (ca != MISSING) & (cb != MISSING)
    hethet = int(np.sum((ca == HET) & (cb == HET)))
    ibs0 = int(np.sum(((ca == HOM_A1) & (cb == HOM_A2)) | ((ca == HOM_A2) & (cb == HOM_A1))))
    het1 = int(np.sum((ca == HET) & both & (cb != HET)))
    het2 = int(np.sum((cb == HET) & both & (ca != HET)))
    return int(both.sum()), hethet, ibs0, het1, het2
