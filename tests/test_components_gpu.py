"""Every eigensolver path along the number of components k: from k = 1 past 16, against the FP64 reference of eig_ref.py.

The generator of synth.cu has five populations, so only its top four components are separated.  The cohorts here come
from `structured_cells` (20 or 40 Balding-Nichols populations), whose top 17 or 34 eigenvalues are apart; each test first
asserts that premise -- a gap above 1e-3 of lambda_1 among the top k + 1 eigenvalues -- so that a drifted cohort fails
as a bad premise, not as a solver bug.

What depends on k (csrc/eig.cu): bisect_kernel<<<k>>>, the Gram-Schmidt over earlier columns in invit_kernel, the max
over k columns in lz_check_kernel, lz_ritz_kernel / lz_ritz_rm_kernel, lz_finish_kernel<<<k>>>, lz_lock_kernel,
backtransform_kernel<<<k>>>, and the deflated verification run that starts at column k (persistent: k .. k + 8, where
k + 8 > 32 reads the locked columns past the kLzVtCols shared-memory mirror from global memory; band solver, also on
one band: k - 1 .. k + 16).  vpca_compute_pca takes 1 <= k <= min(N, max(num_pc, 16)); k > 16 needs num_pc >= k.  Every
case proves its path from eig_method and the call's launch count."""
from types import SimpleNamespace

import numpy as np
import pytest

from eig_ref import (P, Reference, assert_direct, assert_one_band, assert_persistent, band_contexts, check_agree,
                     check_pairs, close_all, compute_pca, compute_pca_bands, gram_context, panel_buffer,
                     structured_cells, synth_cells)

pytestmark = pytest.mark.gpu

COHORT_SEED = 20241015
MIN_GAP = 1e-3


@pytest.fixture(scope="module")
def cohorts():
    """(n, nv, pops) -> (panel buffer on cuda:0, Reference with the top 17 (20 populations) or 34 (40) pairs)"""
    cache = {}

    def get(n, nv, pops):
        if (n, nv, pops) not in cache:
            import torch
            X = structured_cells(n, nv, pops, COHORT_SEED)
            cache[n, nv, pops] = panel_buffer(X), Reference(torch.from_numpy(X).cuda(), 17 if pops <= 20 else 34)
        return cache[n, nv, pops]
    yield get
    cache.clear()


def premise(ref, k):
    gap = ref.min_gap(k)
    assert gap > MIN_GAP, f"premise: the cohort's top {k + 1} eigenvalues are {gap:.2e} lambda_1 apart, not > {MIN_GAP}"


def report(name, s):
    print(f"{name}: {s}")


# ------------------------------------------------------------------------------------------ persistent Lanczos
@pytest.mark.parametrize("n,k", [(2504, 1), (2504, 5), (2504, 8), (2504, 9), (2504, 16), (2503, 16)],
                         ids=["regw-k1", "regw-k5", "regw-k8", "regw-k9", "regw-k16", "scalar-k16"])
def test_persistent_lanczos_along_k(cohorts, n, k):
    """Persistent Lanczos with the regw mat-vec (N = 2504) and the scalar one (N = 2503, N % 4 != 0), num_pc = k."""
    nv = 8192
    buf, ref = cohorts(n, nv, 20)
    premise(ref, k)
    with gram_context(n, buf, nv, k) as nat:
        s = compute_pca(nat, k)
    report(f"persistent n={n} k={k}", s)
    assert_persistent(s)
    check_pairs(ref, s.vecs, s.evals, s.nz, k)


@pytest.mark.parametrize("k", [24, 33])
def test_persistent_lanczos_past_16_components(cohorts, k):
    """Persistent Lanczos with num_pc = 33.  Past 16 components the first 16-step chunks hold fewer steps than pairs
    wanted, and the solver must not test convergence on them: at k = 33 the residuals of the 16- and 32-step tests fed
    the convergence-rate forecast, which gave up at 48 steps and handed over to the direct reduction.  At k = 33 the
    deflated re-run (columns k .. k + 8) also reaches past the 32 mirrored basis columns."""
    n, nv = 3300, 4096
    buf, ref = cohorts(n, nv, 40)
    premise(ref, k)
    with gram_context(n, buf, nv, 33) as nat:
        s = compute_pca(nat, k)
    report(f"persistent n={n} k={k}", s)
    assert_persistent(s)
    check_pairs(ref, s.vecs, s.evals, s.nz, k)


# ------------------------------------------------------------------------------------------- one-band Lanczos
@pytest.mark.parametrize("k,pops", [(16, 20), (33, 40)], ids=["k16", "k33"])
def test_one_band_lanczos_forced_along_k(cohorts, k, pops):
    """One-band Lanczos (the band solver on the whole Gram) forced with VPCA_LZ_PERSIST=0 at N = 2504; its deflated run
    covers columns k - 1 .. k + 16."""
    n, nv = 2504, 8192
    buf, ref = cohorts(n, nv, pops)
    premise(ref, k)
    with gram_context(n, buf, nv, k) as nat:
        s = compute_pca(nat, k, {"VPCA_LZ_PERSIST": "0"})
    report(f"one-band n={n} k={k}", s)
    assert_one_band(s)
    check_pairs(ref, s.vecs, s.evals, s.nz, k)


def test_one_band_lanczos_by_size_16_components(cohorts):
    """One-band Lanczos chosen by the solver (N = 12 000 is past the persistent form's shared-memory fit), k = 16."""
    import torch
    n, nv, k = 12_000, 8192, 16
    free, _ = torch.cuda.mem_get_info()
    if free < 8 * 2 ** 30:
        pytest.skip("needs 8 GB of free HBM")
    buf, ref = cohorts(n, nv, 20)
    premise(ref, k)
    with gram_context(n, buf, nv, k) as nat:
        s = compute_pca(nat, k)
    report(f"one-band n={n} k={k}", s)
    assert_one_band(s)
    check_pairs(ref, s.vecs, s.evals, s.nz, k)


# ------------------------------------------------------------------------------------------------ direct solver
@pytest.mark.parametrize("n,nv,pops,k,fused", [(1092, 8192, 20, 16, True), (3300, 4096, 40, 16, False),
                                               (3300, 4096, 40, 33, False)],
                         ids=["fused-k16", "two-kernel-global-invit-k16", "two-kernel-global-invit-k33"])
def test_direct_solver_along_k(cohorts, n, nv, pops, k, fused):
    """Direct reduction (VPCA_EIG=direct): bisect_kernel<<<k>>>, k inverse iterations each orthogonalised against the
    earlier ones (in global memory above N = 3200), backtransform_kernel<<<k>>>."""
    buf, ref = cohorts(n, nv, pops)
    premise(ref, k)
    with gram_context(n, buf, nv, k) as nat:
        s = compute_pca(nat, k, {"VPCA_EIG": "direct"})
    report(f"direct n={n} k={k}", s)
    assert_direct(s, n, fused)
    check_pairs(ref, s.vecs, s.evals, s.nz, k)


class DenseReference:
    """FP64 eigh of the whole centred Gram C = J X X^T J (every eigenpair, the zero one included)"""

    def __init__(self, X):
        X = np.asarray(X, np.float64)
        self.n = X.shape[0]
        self.nz = int((X.sum(axis=1) > 0).sum())
        J = np.eye(self.n) - 1.0 / self.n
        self.C = J @ (X @ X.T) @ J
        lam, U = np.linalg.eigh(self.C)
        self.lam, self.U = lam[::-1].copy(), U[:, ::-1].copy()

    def residuals(self, vecs, evals):
        return np.linalg.norm(self.C @ vecs - vecs * evals[None, :], axis=0) / self.lam[0]


def test_direct_solver_all_components():
    """k = N = 7 (num_pc = 7): the direct reduction returns every eigenpair, down to the zero eigenvalue of the constant
    vector that the centring leaves."""
    n, k = 7, 7
    X = structured_cells(n, P, 3, COHORT_SEED)
    ref = DenseReference(X)
    assert np.min(np.diff(ref.lam[::-1])) / ref.lam[0] > MIN_GAP, ref.lam             # premise: simple eigenvalues
    with gram_context(n, panel_buffer(X), P, k) as nat:
        s = compute_pca(nat, k)
    report(f"direct n={n} k={k}", s)
    assert_direct(s, n, fused=True)
    check_pairs(ref, s.vecs, s.evals, s.nz, k, eval_atol=1e-12 * ref.lam[0])
    assert abs(s.evals[-1]) <= 1e-12 * ref.lam[0]
    assert np.allclose(s.vecs[:, -1], 1.0 / np.sqrt(n), rtol=0, atol=1e-12)


# ------------------------------------------------------------------------------------------------- band solver
@pytest.mark.parametrize("world", [1, 2, 4])
@pytest.mark.parametrize("k,pops", [(16, 20), (24, 40), (33, 40)], ids=["k16", "k24", "k33"])
def test_band_solver_along_k(cohorts, world, k, pops):
    """Band solver (vpca_compute_pca_bands) on one full context or owner-computes bands of ownerRowBands, num_pc = k."""
    from spark_examples_b200 import native
    n, nv = 2504, 8192
    buf, ref = cohorts(n, nv, pops)
    premise(ref, k)
    if world == 1:
        ctxs = [gram_context(n, buf, nv, k)]
    else:
        ctxs = band_contexts(n, buf, nv, native.ownerRowBands(n, world), k)
    try:
        s = compute_pca_bands(ctxs, k)
    finally:
        close_all(ctxs)
    report(f"bands world={world} n={n} k={k}", s)
    assert s.method == 4 and 16 <= s.iters <= 320, s
    check_pairs(ref, s.vecs, s.evals, s.nz, k)


# ----------------------------------------------------------------------------------------------- bulk components
@pytest.mark.parametrize("k", [8, 16])
def test_bulk_components(k):
    """The generator's five-population cohort: components past the fourth are bulk.  Lanczos converges (eig_method 2)
    or hands over to the direct reduction (3); either way eigenvalues, residuals and orthonormality hold, and the
    vectors match the reference as far as the gaps determine them."""
    from oracle import oracle
    n, nv = 2504, 4096
    buf, X = synth_cells(n, nv)
    ref = Reference(X, k + 1)
    with gram_context(n, buf, nv, k) as nat:
        s = compute_pca(nat, k)
    report(f"bulk n={n} k={k}", s)
    assert s.method in (2, 3), s
    vecs, evals = s.vecs, s.evals
    assert vecs.shape == (n, k) and s.nz == ref.nz
    assert np.allclose(evals, ref.lam[:k], rtol=1e-10, atol=0), (evals, ref.lam[:k])
    assert np.all(ref.residuals(vecs, evals) <= 1e-11)
    assert np.abs(vecs.T @ vecs - np.eye(k)).max() <= 1e-10
    for c in range(k):
        assert vecs[np.argmax(np.abs(vecs[:, c])), c] > 0
    sep = max((j for j in range(1, k + 1) if ref.gaps_allow(j)), default=0)   # the leading columns the gaps determine
    assert sep >= 4, f"premise: the generator's four structured components are apart (only {sep} are)"
    err = oracle.eigvec_rel_err(vecs[:, :sep], ref.U[:, :sep])
    assert np.all(err <= 1e-6), err


# ---------------------------------------------------------------------------------------------- prefix consistency
def test_prefix_consistency(cohorts):
    """computePca(16) and computePca(4) of one Gram: the first four pairs agree."""
    n, nv = 2504, 8192
    buf, ref = cohorts(n, nv, 20)
    premise(ref, 16)
    with gram_context(n, buf, nv, 16) as nat:
        s16 = compute_pca(nat, 16)
        s4 = compute_pca(nat, 4)
    for s, k in ((s16, 16), (s4, 4)):
        assert_persistent(s)
        check_pairs(ref, s.vecs, s.evals, s.nz, k)
    check_agree(SimpleNamespace(vecs=s16.vecs[:, :4], evals=s16.evals[:4]), s4, 4, ref)
