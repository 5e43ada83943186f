"""Every eigensolver path behind vpca_compute_pca, and the band solver's unaligned edges, against an FP64 reference.

`eig_topk` / `lanczos_topk` (csrc/eig.cu) choose a path from N, N mod 4, the SM count and environment switches:

  persistent Lanczos (one cooperative launch per 16-step chunk, reads the int32 Gram S), while its shared memory fits
      mat-vec  regw       N % 4 == 0 and the 512-column segments fill the warps (1092, 2504, 8192, ...)
               task list  N % 4 == 0 otherwise (5632, 10 000, 10 752, ...)
               scalar     N % 4 != 0
      rows of S kept in shared memory as far as they fit, the rest read from L2 (VPCA_LZ_SROWS caps them)
  one-band Lanczos (the band solver of vpca_compute_pca_bands with the whole Gram as its one band, nine kernels per step
      on the int32 S): past that fit (~10 750 on 132 SMs), VPCA_LZ_PERSIST=0
  direct reduction: fused step kernel up to N = 3072, two kernels above (or VPCA_EIG_TWO_KERNELS); inverse iteration
      out of shared memory up to N = 3200, out of global memory above
  Lanczos that gives up hands over to the direct reduction (eig_method 3)

Each test names the path it exercises and proves that it ran: `eig_method`, and -- both Lanczos forms report 2 -- the
`kernel_launches` delta of the call: the persistent form needs fewer launches than steps, the one-band form at least nine
per step, the direct reduction 64 (fused) or 128 (two kernels) per 64-step graph replay.

Reference: the cohort is the synthetic generator's cells X (N x nv, 0/1) and the Gram kernel builds S = X X^T from them
(pinned bit for bit by test_gram_gpu.py).  The centred Gram is C = J S J = (JX)(JX)^T, so its top eigenpairs come from the
small FP64 eigh of (JX)^T (JX): lambda and u = JX v / sqrt(lambda).  Residuals C u - lambda u = JX ((JX)^T u) - lambda u
cost O(N nv) without forming C."""
import numpy as np
import pytest

from eig_ref import (P, Reference, assert_direct, assert_one_band, assert_persistent, band_contexts, bands_from_edges,
                     check_agree, check_pairs, close_all, compute_pca, compute_pca_bands, gram_context, solve,
                     synth_cells)

pytestmark = pytest.mark.gpu

NV = 4096         # variants of every cohort below 65 535 samples
K = 4             # the generator's five populations give four well separated components

# static shared memory of lz_persist_kernel (`ptxas -v`: red, red2, red3); with the device's opt-in limit it decides the
# largest N the persistent form takes.  Update it with the kernel.
LZ_STATIC_SMEM = 9488


def need_free_hbm(gib):
    import torch
    free, _ = torch.cuda.mem_get_info()
    if free < gib * 2 ** 30:
        pytest.skip(f"needs {gib:.0f} GB of free HBM")


def past_fit_gib(n):
    """S (int32) + C (FP64, which eig_alloc allocates whatever the solver) + the Krylov basis + the reference's cells, with
    room to spare"""
    return 1.3 * (12 * n * n + 8 * 400 * n + 24 * n * NV) / 2 ** 30 + 1


def persist_smem(n, sms):
    """dynamic shared memory lz_persist_kernel needs at n on `sms` SMs (base_smem in lanczos_topk, eig.cu)"""
    cap, seg, vt = 384, 512, 32
    rows = -(-n // sms)
    even = lambda x: (x + 1) & ~1
    return 8 * (even(n) + cap + even(rows) + even(rows * -(-n // seg)) + rows * vt + even(n) + vt * vt + cap + even(rows))


def last_persistent_n():
    """the largest N whose persistent-form working set fits one block of this device (10 752 on 132 SMs)"""
    import torch
    props = torch.cuda.get_device_properties(0)
    limit = props.shared_memory_per_block_optin - LZ_STATIC_SMEM
    n = 4096
    while persist_smem(n + 1, props.multi_processor_count) <= limit:
        n += 1
    return n


def resolve(n):
    return {"last_fit": last_persistent_n, "past_fit": lambda: last_persistent_n() + 1}.get(n, lambda: n)()


# ------------------------------------------------------------------------------------------ 1. persistent Lanczos
@pytest.mark.parametrize("n", [1092, 2503, 5632, 8192, 10_000, "last_fit"],
                         ids=["regw-all-rows-smem", "scalar", "tasklist-some-rows-smem", "regw-one-row-smem",
                              "tasklist-rows-from-L2", "tasklist-last-N-that-fits"])
def test_persistent_lanczos_matvec_variants(n):
    """Persistent Lanczos, each mat-vec variant: regw (one w segment in registers per warp) at 1092 with every row of S in
    shared memory and at 8192 with one; the scalar mat-vec at 2503 (N % 4 != 0); the (row, segment) task list at 5632,
    10 000 and the largest N whose shared-memory working set still fits a block, rows mostly or all read from L2."""
    n = resolve(n)
    buf, X = synth_cells(n, NV)
    s = solve(n, buf, NV, K)
    assert_persistent(s)
    check_pairs(Reference(X, K), s.vecs, s.evals, s.nz, K)
    if n == 1092:                        # and the MLlib recipe itself, where it is cheap
        from oracle import oracle
        with gram_context(n, buf, NV, K) as nat:
            S = nat.getGram()
        want, _ = oracle.compute_pca(S, K)
        assert np.all(oracle.eigvec_rel_err(s.vecs, want) <= 1e-6)


@pytest.mark.parametrize("env", [{"VPCA_LZ_SROWS": "0"}, {"VPCA_LZ_SPECULATE": "0"}], ids=["no-rows-in-smem", "no-speculation"])
def test_persistent_lanczos_switches(env):
    """Persistent Lanczos at 2504 with every row of S read from L2 (VPCA_LZ_SROWS=0), and with the verification run
    enqueued only after the host has seen convergence (VPCA_LZ_SPECULATE=0): the same pairs as the default run."""
    n = 2504
    buf, X = synth_cells(n, NV)
    ref = Reference(X, K)
    default, switched = solve(n, buf, NV, K), solve(n, buf, NV, K, env)
    for s in (default, switched):
        assert_persistent(s)
        check_pairs(ref, s.vecs, s.evals, s.nz, K)
    check_agree(switched, default, K, ref)


# ------------------------------------------------------------------------------------------- 2. one-band Lanczos
def assert_same_bits(a, b):
    assert np.array_equal(a.vecs, b.vecs) and np.array_equal(a.evals, b.evals) and a.nz == b.nz, (a, b)


@pytest.mark.parametrize("n", [1092, 2503])
def test_graph_lanczos_forced(n):
    """One-band Lanczos (the band solver on the whole Gram: band_tile_kernel on the int32 S, lz_dots / lz_update,
    lz_ritz_kernel, and the column-major deflated verification run) forced with VPCA_LZ_PERSIST=0: bit for bit
    vpca_compute_pca_bands on the same context, and against the persistent form and the reference."""
    buf, X = synth_cells(n, NV)
    ref = Reference(X, K)
    with gram_context(n, buf, NV, K) as nat:
        one_band = compute_pca(nat, K, {"VPCA_LZ_PERSIST": "0"})
        bands = compute_pca_bands([nat], K)
    persistent = solve(n, buf, NV, K)
    assert_one_band(one_band)
    assert bands.method == 4, bands
    assert_persistent(persistent)
    check_pairs(ref, one_band.vecs, one_band.evals, one_band.nz, K)
    assert_same_bits(one_band, bands)
    check_agree(one_band, persistent, K, ref)


@pytest.mark.parametrize("n", ["past_fit", 12_000, 16_384, 16_385, 20_000])
def test_graph_lanczos_past_the_persistent_fit(n):
    """One-band Lanczos chosen by the solver itself: from the first N whose persistent working set no longer fits a
    block of shared memory (10 753 on 132 SMs) on, where the persistent kernel cannot be launched."""
    n = resolve(n)
    need_free_hbm(past_fit_gib(n))
    buf, X = synth_cells(n, NV)
    s = solve(n, buf, NV, K)
    assert_one_band(s)
    check_pairs(Reference(X, K), s.vecs, s.evals, s.nz, K)


def test_graph_lanczos_at_the_sample_limit():
    """One-band Lanczos at N = 65 535, vpca_compute_pca's limit: S is 17 GB, and C (34 GB) is allocated but not built.
    k = 2 on the structured cohort converges without a hand-over to the direct solver."""
    import torch
    n, nv, k = 65_535, 2048, 2
    need_free_hbm(60)
    buf, X = synth_cells(n, nv)
    with gram_context(n, buf, nv, k) as nat:
        s = compute_pca(nat, k)
    torch.cuda.empty_cache()
    assert_one_band(s)
    check_pairs(Reference(X, k), s.vecs, s.evals, s.nz, k)


# ------------------------------------------------------------------------------------------------ 3. direct solver
@pytest.mark.parametrize("n,fused", [(3072, True), (3073, False), (3200, False), (3201, False), (4096, False)],
                         ids=["fused-smem-invit", "two-kernel-smem-invit", "two-kernel-last-smem-invit",
                              "two-kernel-global-invit", "two-kernel-global-invit-4096"])
def test_direct_solver(n, fused):
    """Direct reduction (VPCA_EIG=direct) on both sides of its switches: the fused step kernel up to N = 3072 and
    tridiag_small + tridiag_big above; inverse iteration with its 8 N doubles in shared memory up to N = 3200
    (invit_kernel<true>) and in global memory above (invit_kernel<false>)."""
    buf, X = synth_cells(n, NV)
    s = solve(n, buf, NV, K, {"VPCA_EIG": "direct"})
    assert_direct(s, n, fused)
    check_pairs(Reference(X, K), s.vecs, s.evals, s.nz, K)


def test_direct_solver_two_kernels_forced():
    """The two-kernel direct reduction forced with VPCA_EIG_TWO_KERNELS=1 at 1092, against the fused form."""
    n = 1092
    buf, X = synth_cells(n, NV)
    ref = Reference(X, K)
    two = solve(n, buf, NV, K, {"VPCA_EIG": "direct", "VPCA_EIG_TWO_KERNELS": "1"})
    fused = solve(n, buf, NV, K, {"VPCA_EIG": "direct"})
    assert_direct(two, n, fused=False)
    assert_direct(fused, n, fused=True)
    for s in (two, fused):
        check_pairs(ref, s.vecs, s.evals, s.nz, K)
    check_agree(two, fused, K, ref)


# ------------------------------------------------------------------------------------------ 4. hand-over above 3072
def test_abandoned_lanczos_hands_over_above_3072():
    """Lanczos that gives up hands over to the two-kernel direct reduction: six components reach into the bulk and need
    more than 32 steps, so with VPCA_EIG_MAXIT=32 the solve falls back -- and then it is the direct solve, bit for bit."""
    n, k = 4000, 6
    buf, X = synth_cells(n, NV)
    cut = solve(n, buf, NV, k, {"VPCA_EIG_MAXIT": "32"})
    direct = solve(n, buf, NV, k, {"VPCA_EIG": "direct"})
    assert cut.method == 3 and cut.iters == 32, cut
    assert_direct(direct, n, fused=False)
    assert cut.launches > direct.launches
    assert np.array_equal(cut.vecs, direct.vecs) and np.array_equal(cut.evals, direct.evals)
    check_pairs(Reference(X, k), cut.vecs, cut.evals, cut.nz, k)


# --------------------------------------------------------------------------------------------------- 5. band solver
@pytest.mark.parametrize("n", [2503, 3001])
def test_band_solver_scalar_loads(n):
    """Band solver on one full context with N % 4 != 0: band_tile_kernel<T, false> (scalar loads, the diagonal clipped
    cell by cell) for both the exact row sums and every mat-vec, against the reference and vpca_compute_pca."""
    buf, X = synth_cells(n, NV)
    ref = Reference(X, K)
    with gram_context(n, buf, NV, K) as nat:
        bands = compute_pca_bands([nat], K)
        full = compute_pca(nat, K)
    assert bands.method == 4 and 16 <= bands.iters <= 320, bands
    assert_persistent(full)
    check_pairs(ref, bands.vecs, bands.evals, bands.nz, K)
    check_agree(bands, full, K, ref)
    assert bands.nz == full.nz


# band bounds off every multiple of 4, 32 and 64, one single-row band, two that straddle a 1024-column tile boundary
UNALIGNED_EDGES = [0, 1, 64, 1064, 2063]


@pytest.mark.parametrize("n", [2503, 2504], ids=["scalar-loads", "vector-loads"])
def test_band_solver_unaligned_bands(n):
    """Band solver on hand-made owner-computes bands [0, 1), [1, 64), [64, 1064), [1064, 2063), [2063, N): the diagonal
    clipping of band_load inside a 4-cell group, with scalar (N % 4 != 0) and int4 loads, and tiles cut by band ends."""
    buf, X = synth_cells(n, NV)
    ref = Reference(X, K)
    ctxs = band_contexts(n, buf, NV, bands_from_edges(UNALIGNED_EDGES + [n]), K)
    try:
        bands = compute_pca_bands(ctxs, K)
    finally:
        close_all(ctxs)
    assert bands.method == 4, bands
    check_pairs(ref, bands.vecs, bands.evals, bands.nz, K)
    full = solve(n, buf, NV, K)
    check_agree(bands, full, K, ref)


def test_band_solver_world_16():
    """Band solver with 16 owner-computes bands (BandEnds' maximum), uneven and unaligned: the rank-order sums of the
    partial products over all 16 slots."""
    n = 3001
    buf, X = synth_cells(n, NV)
    ref = Reference(X, K)
    edges = [round(q * n / 16) + (q % 3 if 0 < q < 16 else 0) for q in range(17)]
    ctxs = band_contexts(n, buf, NV, bands_from_edges(edges), K)
    try:
        bands = compute_pca_bands(ctxs, K)
    finally:
        close_all(ctxs)
    assert bands.method == 4, bands
    check_pairs(ref, bands.vecs, bands.evals, bands.nz, K)
    check_agree(bands, solve(n, buf, NV, K), K, ref)


# ----------------------------------------------------------------- 6. vpca_compute_pca past the fit is the band solver
@pytest.mark.parametrize("n", [12_000, 20_000])
def test_graph_lanczos_and_band_solver_agree(n):
    """Past the persistent fit vpca_compute_pca solves the whole Gram as one band of the band solver: bit for bit what
    vpca_compute_pca_bands (world 1) gives on the same context."""
    need_free_hbm(past_fit_gib(n))
    buf, X = synth_cells(n, NV)
    ref = Reference(X, K)
    with gram_context(n, buf, NV, K) as nat:
        one_band = compute_pca(nat, K)
        bands = compute_pca_bands([nat], K)
    assert_one_band(one_band)
    assert bands.method == 4, bands
    for s in (one_band, bands):
        check_pairs(ref, s.vecs, s.evals, s.nz, K)
    assert_same_bits(one_band, bands)
