"""Linear association tests on the GPU where the counted allele is almost fixed (DESIGN.md 15), from 2504 samples to a
million: A1 fixed but a few hets or one HOM_A2, all het but one or two homs, A1 frequencies 0.999 and 0.99, the same
rows mirrored (00 <-> 11) and ordinary Balding-Nichols rows as a control.  There a raw dosage makes sum g^2 about
4 OBS_CT while the Schur term s = sum g^2 - u^T u is about the number of minor-allele carriers, so s would cancel by a
factor of about 4 OBS_CT / s.  Each cohort runs with no missing call (the sums alone), about 1 % missing (the
missing-set pass), OBS_CT at either side of the switch between the missing-set and called-set passes, and about 60 %
missing (the called-set pass), with a few samples of NaN phenotype whose codes must not matter; at q = 1, 11 and 32
(the sums kernel's KMAX 2, 16 and 32 and VT 2 and 1).  BETA, SE and T_STAT are compared with per-variant lstsq by
test_glm_gpu.check, at its tolerances, for every variant.  Counting A2 must give the bits of counting A1 in the mirrored
rows, and the bits of counting A1 with BETA and T_STAT negated: the dosage is centred on the integer nearest its mean
with a tie going to 1, so the two centred dosages are exact negatives of each other."""
import numpy as np
import pytest

import glm_ref
import grm_ref
from spark_examples_b200 import native
from test_glm_gpu import _bits, check, check_p_df

pytestmark = pytest.mark.gpu

BIG = 1_000_003
SIZES = [(2504, 1), (2504, 11), (2504, 32), (21845, 1), (21845, 11), (21845, 32), (65537, 1), (65537, 11), (65537, 32),
         (BIG, 1), (BIG, 11)]
# the regression samples made missing at each row: none; about 1 %; OBS_CT == n_reg - OBS_CT (the last count that takes
# the missing-set pass, n_reg even); OBS_CT == n_reg - OBS_CT - 1 (the first that takes the called-set pass, n_reg odd);
# about 60 %
PATHS = ("none", "miss1", "half", "half-1", "miss60")
MIRRORED = ("het1", "het10", "hom2", "allhet1", "f0.999")   # the kinds mirrored at a million samples (16 rows a call)


def _missing_count(path, n_reg):
    return {"none": 0, "miss1": round(0.01 * n_reg), "half": n_reg // 2, "half-1": (n_reg + 1) // 2,
            "miss60": round(0.6 * n_reg)}[path]


def _cohort(seed, n, q, path):
    """(rows, pheno, covar, excluded, designed): the near-fixed rows, the same mirrored, ordinary rows (16 rows in all
    at a million samples, 32 below), `path`'s missing calls at every row, 3 or 4 samples of NaN phenotype (the parity
    of the regression samples that `path` needs) with random codes."""
    rng = np.random.default_rng(seed)
    big = n >= BIG
    near = glm_ref.near_fixed_codes(rng, n)
    mirrored = glm_ref.near_fixed_codes(rng, n, MIRRORED if big else glm_ref.KINDS)
    mirrored = np.where(mirrored == 0, 3, np.where(mirrored == 3, 0, mirrored)).astype(np.uint8)
    designed = len(near) + len(mirrored)
    code = np.concatenate([near, mirrored, grm_ref.balding_nichols(rng, n, (16 if big else 32) - designed)])
    k = 3 if path not in ("half", "half-1") or (n - 3) % 2 == (path == "half-1") else 4
    excluded = np.sort(rng.choice(n, k, replace=False))
    reg = np.ones(n, bool)
    reg[excluded] = False
    n_reg = n - k
    m = _missing_count(path, n_reg)
    for v in range(len(code)):
        # the carriers of the rarer genotypes of a near-fixed row stay called, so that it keeps a fit
        vals, cnt = np.unique(code[v, reg], return_counts=True)
        mode = vals[np.argmax(cnt)]
        cand = np.flatnonzero(reg & (code[v] == mode)) if cnt.max() >= 0.9 * n_reg else np.flatnonzero(reg)
        code[v, rng.choice(cand, m, replace=False)] = 1
    code[:, excluded] = rng.integers(0, 4, (len(code), k))
    covar = rng.normal(size=(n, q - 1))
    pheno = rng.normal(size=n) + (0.2 * covar[:, 0] if q > 1 else 0.0)
    pheno[excluded] = np.nan
    return grm_ref.pack(code), pheno, covar, excluded, designed


@pytest.mark.parametrize("path", PATHS)
@pytest.mark.parametrize("n,q", SIZES)
def test_near_fixed_alleles(n, q, path):
    rows, pheno, covar, excluded, designed = _cohort(n + 7 * q + PATHS.index(path), n, q, path)
    n_reg = n - len(excluded)
    recoded = grm_ref.pack(np.where(np.isin(np.arange(n), excluded), (glm_ref.codes(rows, n) + 1) % 4,
                                    glm_ref.codes(rows, n)).astype(np.uint8))
    with native.NativePca(n, device=0, gram_band=(0, 1) if n > 65535 else None) as nat:
        assert nat.glmBegin(pheno, covar) == n_reg
        got, gerr = nat.glmLinearBed(rows)
        a2, e2 = nat.glmLinearBed(rows, counted=2)
        mir, emir = nat.glmLinearBed(glm_ref.mirror(rows))
        other, eother = nat.glmLinearBed(recoded)
    note = f"n={n} q={q} {path}"
    obs = n_reg - _missing_count(path, n_reg)
    assert np.all(got[:, 0] == obs), note
    assert {"half": 2 * obs == n_reg, "half-1": 2 * obs == n_reg - 1}.get(path, True), note
    want, werr = glm_ref.linear(rows, n, pheno, covar)
    assert np.all(werr[:designed] == 0), (note, werr)
    check(got, gerr, want, werr, np.zeros(len(werr)), note)   # VIF about 1: every variant is compared
    check_p_df(got[gerr == 0], q, note)
    # the codes of samples outside the regression do not matter
    assert np.array_equal(_bits(other), _bits(got)) and np.array_equal(eother, gerr), note
    # counting A2 is counting A1 in the mirrored rows, and negates BETA and T_STAT exactly
    assert np.array_equal(_bits(a2), _bits(mir)) and np.array_equal(e2, emir), note
    assert np.array_equal(e2, gerr) and np.array_equal(a2[:, 0], got[:, 0]), note
    assert np.all(np.abs(a2[:, 1] + got[:, 1] - 1.0) <= np.spacing(1.0)), note
    neg = got[:, 2:] * [-1.0, 1.0, -1.0, 1.0]
    neg[np.isnan(neg)] = np.nan
    assert np.array_equal(_bits(a2[:, 2:]), _bits(neg)), note
