"""Host references of variant QC (DESIGN.md 10): the four genotype counts of .bed rows in numpy, the exact HWE p-value
restated in Python floats with the operations of csrc/qc.cu in the same order (so the bits must match), and the same
p-value as an exact rational from big-integer weights."""
from fractions import Fraction
from math import comb

import numpy as np

HOM_A1, HET, HOM_A2, MISSING = 0, 1, 2, 3
TIE = 1.0 + 2.0 ** -40


def codes(rows, n):
    """(nv, stride) .bed rows -> (nv, n) 2-bit codes, the extraction of plink.decode_rows (bytes past ceil(n / 4) and
    the padding samples dropped)."""
    rows = np.asarray(rows, dtype=np.uint8)
    return np.stack([(rows >> s) & 3 for s in (0, 2, 4, 6)], axis=-1).reshape(rows.shape[0], -1)[:, :n]


_PER_BYTE = np.stack([(codes(np.arange(256, dtype=np.uint8)[:, None], 4) == k).sum(1) for k in (0, 2, 3, 1)],
                     axis=1).astype(np.uint8)   # [byte, HOM_A1 / HET / HOM_A2 / MISSING]: its four samples' codes


def counts(rows, n):
    """(nv, 4) int32 HOM_A1 (code 00), HET (10), HOM_A2 (11), MISSING (01): whole bytes through a table of the four codes
    of every byte value, then the samples of a last partial byte."""
    rows = np.asarray(rows, dtype=np.uint8)
    full = n // 4
    out = np.stack([_PER_BYTE[:, k][rows[:, :full]].sum(axis=1, dtype=np.int64) for k in range(4)], axis=1)
    if n % 4:
        c = codes(rows[:, full:full + 1], n % 4)
        out += np.stack([(c == k).sum(1) for k in (0, 2, 3, 1)], axis=1)
    return out.astype(np.int32)


def _start(a, het, b):
    n = a + het + b
    r = 2 * min(a, b) + het
    m = r * (2 * n - r) // (2 * n)
    if (m ^ r) & 1:
        m += 1
    return n, r, m


def _walk(n, r, m, het, thr):
    """qc.cu hwe_walk: (sum of the t <= thr, the mode first, then downward, then upward; t(het) or 0)."""
    total = 1.0 if 1.0 <= thr else 0.0
    t_obs = 1.0 if m == het else 0.0
    homr0 = (r - m) // 2
    homc0 = n - m - homr0
    t, h, homr, homc = 1.0, m, homr0, homc0
    while h >= 2:
        t = ((t * float(h)) * float(h - 1)) / ((4.0 * float(homr + 1)) * float(homc + 1))
        h, homr, homc = h - 2, homr + 1, homc + 1
        if t == 0.0:
            break
        if h == het:
            t_obs = t
        if t <= thr:
            total = total + t
    t, h, homr, homc = 1.0, m, homr0, homc0
    while h + 2 <= r:
        t = (((t * 4.0) * float(homr)) * float(homc)) / (float(h + 2) * float(h + 1))
        h, homr, homc = h + 2, homr - 1, homc - 1
        if t == 0.0:
            break
        if h == het:
            t_obs = t
        if t <= thr:
            total = total + t
    return total, t_obs


def hwe_p(a, het, b):
    """The p-value of vpca_hwe_exact for HOM_A1 = a, HET = het, HOM_A2 = b, in Python floats (no contraction)."""
    a, het, b = int(a), int(het), int(b)
    if 2 * min(a, b) + het == 0:
        return 1.0
    n, r, m = _start(a, het, b)
    total, t_obs = _walk(n, r, m, het, float("inf"))
    tail, _ = _walk(n, r, m, het, t_obs * TIE)
    return min(tail / total, 1.0)


def hwe_p_many(c):
    return np.array([hwe_p(x[0], x[1], x[2]) for x in np.asarray(c).reshape(-1, 4).tolist()], np.float64)


def hwe_weights(a, het, b):
    """{h: C(n, h) C(n - h, homr) 2^h}: the relative probability of h hets given n and the rare-allele copies r."""
    n = a + het + b
    r = 2 * min(a, b) + het
    return {h: comb(n, h) * comb(n - h, (r - h) // 2) * 2 ** h for h in range(r % 2, r + 1, 2)}


def hwe_p_exact(a, het, b):
    """(exact p as a Fraction, the smallest |w(h) / w(obs) - 1| over h != obs, inf if none): a relative gap below the
    float test's tolerance would make the two definitions differ on a near-tie."""
    a, het, b = int(a), int(het), int(b)
    if 2 * min(a, b) + het == 0:
        return Fraction(1), float("inf")
    w = hwe_weights(a, het, b)
    wo = w[het]
    tail = sum(x for x in w.values() if x <= wo)
    gap = min((abs(Fraction(x, wo) - 1) for h, x in w.items() if h != het), default=float("inf"))
    return min(Fraction(tail, sum(w.values())), Fraction(1)), float(gap)
