"""The solver a GRM feeds (vpca_compute_pca_grm; DESIGN.md 13, "Solve") at the ends of the GRM's size range and where
Lanczos runs out of Krylov space: band Lanczos on FP64 cells at 16 384 and 21 845 samples and at the 65 535-sample
limit, Lanczos and the direct reduction on one GRM, and GRMs whose rank is below k.  The reference never reads the
device's GRM: the small eigh of Z^T Z (grm_ref.Pcs), in torch float64 on the GPU for large N."""
import numpy as np
import pytest

import grm_ref
from spark_examples_b200 import native

pytestmark = pytest.mark.gpu

KC = 1024   # kGrmPanelK: used variants per panel


def _bits(a):
    return np.ascontiguousarray(a, np.float64).view(np.int64)


def _cohort(seed, n, nv, pops, miss=0.01):
    rng = np.random.default_rng(seed)
    return grm_ref.pack(grm_ref.balding_nichols(rng, n, nv, pops=pops, miss=miss))


def need_free_hbm(gib):
    import torch
    free, _ = torch.cuda.mem_get_info()
    if free < gib * 2 ** 30:
        pytest.skip(f"needs {gib:.0f} GiB of free HBM, {free / 2 ** 30:.1f} GiB free")


def mem_available_gib():
    with open("/proc/meminfo") as f:
        for line in f:
            if line.startswith("MemAvailable:"):
                return int(line.split()[1]) / 2 ** 20
    return 0.0


def context_gib(n):
    """a full context at n: S (int32) + d_C (FP64) + the GRM panel and the Krylov basis, with room to spare"""
    return 1.3 * (12 * n * n + 8 * (KC + 400) * n) / 2 ** 30 + 1


def z_torch(rows, n):
    """-> (Z (n, M) float64 on cuda:0, M) from grm_ref's z table"""
    import torch
    tab, used = grm_ref.z_tables(grm_ref.counts(rows, n))
    dev = torch.device("cuda")
    code = torch.from_numpy(np.ascontiguousarray(grm_ref.codes(rows, n))).to(dev).long()
    Zt = torch.gather(torch.from_numpy(tab).to(dev), 1, code)[torch.from_numpy(used).to(dev)]   # (M, n)
    del code
    return Zt.T.contiguous(), int(used.sum())


def _release():
    import torch
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


# ---- 1. large N ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [16384, 21845], ids=["vector-16384", "scalar-21845"])
def test_grm_pcs_at_large_n(n):
    """16 384 samples: vector loads over 16 column tiles; 21 845 (N mod 4 = 1): scalar loads over 22."""
    pytest.importorskip("torch")
    need_free_hbm(context_gib(n) + 2)
    k = 4
    rows = _cohort(n, n, 2000, pops=k + 1)
    with native.NativePca(n, num_pc=k) as nat:
        nat.grmBed(rows)
        m = nat.grmFinalize()
        s = grm_ref.Solve(nat, k)
    grm_ref.assert_path(s, 2, n)
    try:
        Z, M = z_torch(rows, n)
        assert m == M
        grm_ref.check_grm_pairs(grm_ref.Pcs(Z, k), s.vecs, s.evals, k, note=repr(s))
    finally:
        Z = None
        _release()


# ---- 2. the limit: 65 535 samples ---------------------------------------------------------------------------------------
def test_grm_at_the_sample_limit():
    """N = 65 535, the largest grm_check takes (N mod 4 = 3: scalar loads, 64 column tiles): grm_finish_kernel's grid has
    gridDim.y = 65 535, the hardware's cap; the SYRK launches 524 800 CTAs per panel over three panels, the last one
    partial; d_C is 34.4 GB, and each band Lanczos step reads its 17 GB lower triangle.  Lanczos leaves the GRM in place,
    so getGrm after the solve returns it: every cell within grm_ref.tolerance of torch's Z Z^T / M, and G = G^T bit for
    bit, both in blocks of 4096 rows once the context has freed its ~53 GB."""
    torch = pytest.importorskip("torch")
    need_free_hbm(60)
    avail = mem_available_gib()
    if avail < 48:
        pytest.skip(f"the host copy of the 65 535-sample GRM is 34.4 GB: needs 48 GiB of MemAvailable, {avail:.1f} GiB")
    n, k = 65535, 2
    rows = _cohort(65535, n, 2600, pops=k + 1)
    with native.NativePca(n, num_pc=k) as nat:
        nat.grmBed(rows)
        m = nat.grmFinalize()
        s = grm_ref.Solve(nat, k)
        G = nat.getGrm()
    grm_ref.assert_path(s, 2, n)
    Z = Gd = A = want = tol = None
    try:
        Z, M = z_torch(rows, n)
        assert m == M and 2 * KC < M < 3 * KC
        grm_ref.check_grm_pairs(grm_ref.Pcs(Z, k), s.vecs, s.evals, k, note=repr(s))
        Gd = torch.from_numpy(G).to(Z.device)
        G = None
        A = Z.abs()
        scale = grm_ref.depth(M) * 2.0 ** -53 / M
        B = 4096
        for r0 in range(0, n, B):
            r1 = min(n, r0 + B)
            blk = Gd[r0:r1]
            want = (Z[r0:r1] @ Z.T) / M
            tol = scale * (A[r0:r1] @ A.T)
            assert bool(((blk - want).abs() <= tol).all()), f"rows [{r0}, {r1})"
            assert torch.equal(blk, Gd[:, r0:r1].T), f"rows [{r0}, {r1}) against their columns"
    finally:
        Z = Gd = A = want = tol = blk = None
        _release()


# ---- 3. one GRM, both solvers -------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [2503, 2504])
def test_grm_lanczos_twice_then_direct(monkeypatch, n):
    """Band Lanczos on one GRM twice: the same bits (every reduction has a fixed order), and the GRM untouched; then the
    direct reduction on the same context agrees with it (eigenvalues to 1e-11, vectors to 1e-8 where the gaps allow)."""
    from oracle import oracle
    k = 4
    rows = _cohort(n + 1, n, 3000, pops=k + 1)
    monkeypatch.delenv("VPCA_EIG", raising=False)
    monkeypatch.delenv("VPCA_EIG_MAXIT", raising=False)
    with native.NativePca(n, num_pc=k) as nat:
        nat.grmBed(rows)
        nat.grmFinalize()
        G = nat.getGrm()
        a = grm_ref.Solve(nat, k)
        b = grm_ref.Solve(nat, k)
        assert np.array_equal(_bits(nat.getGrm()), _bits(G))
        monkeypatch.setenv("VPCA_EIG", "direct")
        c = grm_ref.Solve(nat, k)
    grm_ref.assert_path(a, 2, n)
    grm_ref.assert_path(b, 2, n)
    grm_ref.assert_path(c, 1, n)
    assert np.array_equal(_bits(a.vecs), _bits(b.vecs)) and np.array_equal(_bits(a.evals), _bits(b.evals))
    Z, _ = grm_ref.z_matrix(rows, n)
    ref = grm_ref.Pcs(Z, k + 1)
    for s in (a, c):
        grm_ref.check_grm_pairs(ref, s.vecs, s.evals, k, note=repr(s))
    assert np.allclose(c.evals, a.evals, rtol=1e-11, atol=0), (c.evals, a.evals)
    if ref.gaps_allow(k):
        err = oracle.eigvec_rel_err(c.vecs, a.vecs)
        assert np.all(err <= 1e-8), err


# ---- 4. rank below k ----------------------------------------------------------------------------------------------------
# A GRM's rank is at most min(M, N - 1) (every z column sums to 0).  With k past it, Lanczos exhausts its Krylov space and
# the pairs past the rank come from a cluster of zero Ritz values: they must still be finite, orthonormal, orthogonal to
# the nonzero pairs and oriented by the sign rule, with |lambda| <= 1e-12 lambda_1.
def _solve_all(n, rows, k):
    with native.NativePca(n, num_pc=k) as nat:
        nat.grmBed(rows)
        m = nat.grmFinalize()
        return grm_ref.Solve(nat, k), m


@pytest.mark.parametrize("env", [{}, {"VPCA_EIG": "direct"}], ids=["default", "direct"])
def test_grm_pcs_past_the_rank_of_three_variants(monkeypatch, env):
    """N = 600, k = 8: three used variants among 40 monomorphic or uncalled rows, so the rank is 3."""
    monkeypatch.delenv("VPCA_EIG", raising=False)
    for key, val in env.items():
        monkeypatch.setenv(key, val)
    n, k = 600, 8
    three = grm_ref.balding_nichols(np.random.default_rng(47), n, 3, pops=3, miss=0.01)
    skip = np.zeros((40, n), np.uint8)
    skip[1::3] = 3
    skip[2::3] = 1
    rows = grm_ref.pack(np.insert(skip, [4, 19, 33], three, axis=0))
    s, m = _solve_all(n, rows, k)
    assert m == 3
    assert s.method in ((1,) if env else (2, 3)), s
    Z, _ = grm_ref.z_matrix(rows, n)
    ref = grm_ref.Pcs(Z, k)
    assert ref.rank == 3
    grm_ref.check_grm_pairs(ref, s.vecs, s.evals, k, note=repr(s))


def test_grm_pcs_of_copies_of_two_variants():
    """N = 1025, k = 4: 2048 rows that are copies of two distinct variants, so M = 2048 (two panels) and the rank is 2:
    k <= M does not make k <= rank."""
    n, k = 1025, 4
    two = grm_ref.balding_nichols(np.random.default_rng(53), n, 2, pops=3, miss=0.01)
    rows = grm_ref.pack(two[np.arange(2 * KC) % 2])
    s, m = _solve_all(n, rows, k)
    assert m == 2 * KC and s.method in (2, 3), s
    Z, _ = grm_ref.z_matrix(rows, n)
    ref = grm_ref.Pcs(Z, k)
    assert ref.rank == 2
    grm_ref.check_grm_pairs(ref, s.vecs, s.evals, k, note=repr(s))
