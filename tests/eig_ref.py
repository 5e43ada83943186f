"""FP64 references and solve helpers shared by the eigensolver tests (test_eig_paths_gpu.py, test_components_gpu.py).

Reference: the cohort's cells X (N x nv, 0/1) reach the Gram kernel, which builds S = X X^T from them (pinned bit for bit
by test_gram_gpu.py).  The centred Gram is C = J S J = (JX)(JX)^T, so its top eigenpairs come from the small FP64 eigh of
(JX)^T (JX): lambda and u = JX v / sqrt(lambda).  Residuals C u - lambda u = JX ((JX)^T u) - lambda u cost O(N nv)
without forming C.

Cohorts: `synth_cells` is the library's own generator (five populations: four separated components, the rest bulk);
`structured_cells` draws many populations in numpy, so that the top 17 or 34 eigenvalues are separated."""
import math
import os
from contextlib import contextmanager

import numpy as np

SEED = 20240901
P = 1024          # variants per panel
LZ_ENV = ("VPCA_EIG", "VPCA_EIG_MAXIT", "VPCA_EIG_TWO_KERNELS", "VPCA_LZ_PERSIST", "VPCA_LZ_SROWS", "VPCA_LZ_SPECULATE")


# ---------------------------------------------------------------------------------------------------- reference helpers
class Reference:
    """FP64 top eigenpairs of the centred Gram of the cells X, from the nv x nv eigh of (JX)^T (JX)"""

    def __init__(self, X, k):
        import torch
        X = X.to(torch.float64)
        self.n = X.shape[0]
        self.nz = int((X.sum(dim=1) > 0).sum())                 # rows of S with a positive sum: samples with a carrier
        self.JX = X - X.mean(dim=0, keepdim=True)
        del X
        lam, V = torch.linalg.eigh(self.JX.t() @ self.JX)
        lam, V = lam.flip(0)[:k], V.flip(1)[:, :k]
        self.U = ((self.JX @ V) / lam.sqrt()).cpu().numpy()
        self.lam = lam.cpu().numpy()

    def residuals(self, vecs, evals):
        """||C u - lambda u|| / lambda_1 per column, C u = JX ((JX)^T u)"""
        import torch
        u = torch.from_numpy(vecs).to(self.JX.device)
        r = self.JX @ (self.JX.t() @ u) - u * torch.from_numpy(evals).to(self.JX.device)[None, :]
        return (torch.linalg.norm(r, dim=0) / float(self.lam[0])).cpu().numpy()

    def gaps_allow(self, k):
        """the top k + 1 eigenvalues are far enough apart for two solvers' vectors to agree to 1e-8"""
        return k >= len(self.lam) or np.min(np.abs(np.diff(self.lam[: k + 1]))) / self.lam[0] > 1e-4

    def min_gap(self, k):
        """smallest gap between neighbours among the top k + 1 eigenvalues, relative to the top one (needs k + 1 pairs)"""
        assert len(self.lam) >= k + 1
        return float(np.min(np.abs(np.diff(self.lam[: k + 1]))) / self.lam[0])


def synth_cells(n, nv):
    """The generator's cells of n samples x nv variants on cuda:0 in panel layout (uint8) and as an (n, nv) int8 view"""
    import torch
    from spark_examples_b200 import native
    assert nv % P == 0
    with native.NativePca(n, max_multiplicity=1, gram_band=(0, min(n, 64))) as gen:   # a generator, not an N x N Gram
        buf = torch.zeros(gen.panelBytes(nv, P), dtype=torch.uint8, device="cuda:0")
        torch.cuda.synchronize()
        gen.synthPanelsDevice(SEED, 0, nv, 0, buf.data_ptr(), P)
        gen.synchronize()
    X = buf.view(torch.int8).view(nv // P, n, P).permute(1, 0, 2).reshape(n, nv)
    return buf, X


def structured_cells(n, nv, pops, seed):
    """(n, nv) int8 carrier cells of `pops` populations under the Balding-Nichols model: ancestral allele frequency
    p = 0.05 + 0.45 u, population i draws its frequency from Beta(p (1 - F) / F, (1 - p) (1 - F) / F) with F_ST = F
    running linearly from 0.20 (i = 0) down to 0.04, holds a share of the samples proportional to 1.12^i, and a sample
    carries the variant when its dosage ~ Binomial(2, p_i) is positive, i.e. with probability 1 - (1 - p_i)^2."""
    rng = np.random.default_rng(seed)
    share = 1.12 ** np.arange(pops)
    sizes = np.floor(n * share / share.sum()).astype(np.int64)
    sizes[np.argsort(-(n * share / share.sum() - sizes))[: n - sizes.sum()]] += 1     # largest remainders
    anc = 0.05 + 0.45 * rng.random(nv)
    X = np.empty((n, nv), np.int8)
    row = 0
    for i, fst in enumerate(np.linspace(0.20, 0.04, pops)):
        q = (1.0 - fst) / fst
        p = rng.beta(anc * q, (1.0 - anc) * q)
        carrier = 1.0 - (1.0 - p) ** 2
        X[row:row + sizes[i]] = rng.random((sizes[i], nv)) < carrier[None, :]
        row += sizes[i]
    return X


def panel_buffer(X):
    """(n, nv) int8 cells (numpy) -> the panel layout of vpca_accumulate_panels on cuda:0, zero cells after nv"""
    import torch
    n, nv = X.shape
    npan = -(-nv // P)
    buf = np.zeros((npan, n, P), np.int8)
    for p in range(npan):
        blk = X[:, p * P:(p + 1) * P]
        buf[p, :, :blk.shape[1]] = blk
    return torch.from_numpy(buf.reshape(-1).view(np.uint8)).to("cuda:0")


def check_pairs(ref, vecs, evals, nz, k, eval_atol=0.0):
    """The assertions every solve below must meet against the FP64 reference"""
    from oracle import oracle
    n = ref.n
    assert vecs.shape == (n, k) and evals.shape == (k,)
    assert nz == ref.nz
    assert np.allclose(evals, ref.lam[:k], rtol=1e-10, atol=eval_atol), (evals, ref.lam[:k])
    err = oracle.eigvec_rel_err(vecs, ref.U[:, :k])
    assert np.all(err <= 1e-6), err
    res = ref.residuals(vecs, evals)
    assert np.all(res <= 1e-11), res
    assert np.abs(vecs.T @ vecs - np.eye(k)).max() <= 1e-10
    assert np.allclose(np.linalg.norm(vecs, axis=0), 1.0, atol=1e-12)
    for c in range(k):
        assert vecs[np.argmax(np.abs(vecs[:, c])), c] > 0               # sign rule: largest-|.| entry positive


def check_agree(a, b, k, ref, vec_tol=1e-8, eval_rtol=1e-11):
    """two solves of the same Gram: eigenvalues to eval_rtol, vectors to vec_tol where the gaps allow"""
    from oracle import oracle
    assert np.allclose(a.evals, b.evals, rtol=eval_rtol, atol=0), (a.evals, b.evals)
    if ref.gaps_allow(k):
        err = oracle.eigvec_rel_err(a.vecs, b.vecs)
        assert np.all(err <= vec_tol), err


# --------------------------------------------------------------------------------------------------------- solve helpers
@contextmanager
def solver_env(env):
    """exactly the given solver switches, whatever the caller's environment holds"""
    saved = {key: os.environ.pop(key, None) for key in LZ_ENV}
    os.environ.update(env or {})
    try:
        yield
    finally:
        for key in LZ_ENV:
            os.environ.pop(key, None)
            if saved[key] is not None:
                os.environ[key] = saved[key]


class Solve:
    def __init__(self, out, before, after):
        self.vecs, self.evals, self.nz = out
        self.method = after["eig_method"]
        self.iters = after["eig_iterations"]
        self.launches = after["kernel_launches"] - before["kernel_launches"]

    def __repr__(self):
        return f"Solve(method={self.method}, iters={self.iters}, launches={self.launches})"


def gram_context(n, buf, nv, k):
    """a fresh full context whose finalized Gram the Gram kernel built from the cells"""
    from spark_examples_b200 import native
    nat = native.NativePca(n, max_multiplicity=1, num_pc=k)
    try:
        nat.accumulatePanels(buf.data_ptr(), nv, P)
        nat.finalizeGram()
    except Exception:
        nat.close()
        raise
    return nat


def compute_pca(nat, k, env=None):
    """vpca_compute_pca under exactly the switches in env (the context must not have solved by Lanczos yet if env sets
    VPCA_LZ_PERSIST: the persistent or one-band form is fixed at a context's first Lanczos solve)"""
    with solver_env(env):
        before = nat.stats()
        out = nat.computePca(k)
        return Solve(out, before, nat.stats())


def solve(n, buf, nv, k, env=None):
    with gram_context(n, buf, nv, k) as nat:
        return compute_pca(nat, k, env)


def compute_pca_bands(ctxs, k):
    from spark_examples_b200 import native
    with solver_env(None):
        before = ctxs[0].stats()
        out = native.computePcaBands(ctxs, k)
        return Solve(out, before, ctxs[0].stats())


def assert_persistent(s):
    assert s.method == 2, s
    assert 16 <= s.iters <= 320 and s.launches < s.iters, s          # one cooperative launch per 16 steps + the checks


def assert_one_band(s):
    # band_norm, band_scale, band_tile, band_reduce, band_combine, 2 x lz_dots, 2 x lz_update: 9 launches per step
    assert s.method == 2, s
    assert 16 <= s.iters <= 320 and s.launches >= 9 * s.iters, s


def assert_direct(s, n, fused):
    # row sums + mean (2), ceil(n / 64) replays of the 64-step graph (1 or 2 launches per step), bisection, inverse
    # iteration, back-transformation (3)
    assert s.method == 1 and s.iters == 0, s
    assert s.launches == 2 + (1 if fused else 2) * 64 * math.ceil(n / 64) + 3, s


# ------------------------------------------------------------------------------------------------------- band helpers
def band_contexts(n, buf, nv, bands, k):
    """owner-computes band contexts (no peers, every variant fed to each) storing rows [row0, row0 + rows) each"""
    from spark_examples_b200 import native
    ctxs = []
    try:
        for band in bands:
            ctxs.append(native.NativePca(n, max_multiplicity=1, num_pc=k, gram_band=band))
        for c in ctxs:
            c.accumulatePanels(buf.data_ptr(), nv, P)
        for c in ctxs:
            c.synchronize()
            c.finalizeGram()
        return ctxs
    except Exception:
        close_all(ctxs)
        raise


def close_all(ctxs):
    for c in ctxs:
        try:
            c.synchronize()
        except Exception:
            pass
    for c in ctxs:
        c.close()


def bands_from_edges(edges):
    return [(a, b - a) for a, b in zip(edges[:-1], edges[1:])]
