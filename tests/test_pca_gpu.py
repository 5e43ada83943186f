"""GPU parity tests of centering + eigensolve (VariantsPca.scala:198-231) against the oracle, through the C ABI.

Tolerance: top-k eigenvectors within 1e-6 relative, sign-normalised:
max_i |u^_i - u_i| / max_i |u_i| <= 1e-6 per component.  Centering is compared bit for bit."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

SEED = 20240901
TOL = 1e-6


def _native(n, **kw):
    from spark_examples_b200 import native
    return native.NativePca(n, **kw)


def _structured_gram(oracle, n, nv, seed=SEED):
    X = oracle.c_synth_dense(seed, n, 0, nv, 0)
    return oracle.np_similarity_dense(X)


@pytest.mark.parametrize("n,nv", [(64, 500), (257, 2000), (1092, 8000)])
def test_centering_bit_exact(oracle, n, nv):
    S = _structured_gram(oracle, n, nv)
    want, row_sums, nz = oracle.c_center(S)
    with _native(n) as nat:
        nat.setGram(S)
        C = nat.getCentered()
    assert np.array_equal(C, want)


@pytest.mark.parametrize("n,nv,method", [(2, 40, "direct"), (3, 60, "direct"), (50, 700, "direct"),
                                         (257, 3000, "direct"), (257, 3000, "lanczos"), (1092, 8000, "direct"),
                                         (1092, 8000, "auto")])
def test_top2_eigenvectors_match_mllib_recipe(oracle, monkeypatch, n, nv, method):
    """Both solvers behind vpca_compute_pca: the direct reduction (Householder + bisection + inverse iteration) and
    Lanczos (auto from 512 samples up; VPCA_EIG=lanczos forces it from 96)."""
    monkeypatch.setenv("VPCA_EIG", method)
    S = _structured_gram(oracle, n, nv)
    want, sv = oracle.compute_pca(S, 2 if n > 2 else 1)
    k = want.shape[1]
    with _native(n) as nat:
        nat.setGram(S)
        vecs, evals, nz = nat.computePca(k)
        st = nat.stats()
        if method == "direct":
            assert st["eig_method"] == 1 and st["eig_iterations"] == 0
            d, e = nat.getTridiagonal()
        else:
            assert st["eig_method"] == 2 and 16 <= st["eig_iterations"] <= 320, st
            with pytest.raises(Exception):
                nat.getTridiagonal()
    C, rs, nz_want = oracle.np_center(S)
    assert nz == nz_want
    w = np.linalg.eigvalsh(C)[::-1]
    # eigenvalues of C (the reference's singular values of Cov are w^2/(n-1))
    assert np.allclose(evals, w[:k], rtol=1e-10, atol=1e-8 * abs(w[0]))
    if method == "direct":
        T = np.diag(d) + np.diag(e, 1) + np.diag(e, -1)
        assert np.allclose(np.linalg.eigvalsh(T)[::-1][: min(n, 8)], w[: min(n, 8)], rtol=1e-9, atol=1e-8 * abs(w[0]))
    # unit norm + sign rule
    assert np.allclose(np.linalg.norm(vecs, axis=0), 1.0, atol=1e-12)
    for c in range(k):
        assert vecs[np.argmax(np.abs(vecs[:, c])), c] > 0
    err = oracle.eigvec_rel_err(vecs, want)
    assert np.all(err <= TOL), err


def _residuals(C, vecs, evals):
    return np.linalg.norm(C @ vecs - vecs * evals[None, :], axis=0) / np.abs(np.linalg.eigvalsh(C)).max()


@pytest.mark.parametrize("k", [1, 2, 6])
def test_lanczos_agrees_with_direct(oracle, monkeypatch, k):
    """Same Gram through both solvers: eigenvalues to 1e-11 relative, eigenvectors far inside the 1e-6 bar."""
    n, nv = 1500, 6000
    S = _structured_gram(oracle, n, nv, seed=SEED + k)
    out = {}
    for method in ("direct", "auto"):
        monkeypatch.setenv("VPCA_EIG", method)
        with _native(n, num_pc=k) as nat:
            nat.setGram(S)
            out[method] = nat.computePca(k) + (nat.stats(),)
    assert out["direct"][3]["eig_method"] == 1
    assert out["auto"][3]["eig_method"] in (2, 3)
    assert np.allclose(out["auto"][1], out["direct"][1], rtol=1e-11)
    C, _, _ = oracle.np_center(S)
    w = np.linalg.eigvalsh(C)[::-1]
    gaps = np.abs(np.diff(w[: k + 1])) / w[0]
    if gaps.min() > 1e-4:
        err = oracle.eigvec_rel_err(out["auto"][0], out["direct"][0])
        assert np.all(err <= 1e-8), err
    assert np.all(_residuals(C, out["auto"][0], out["auto"][1]) <= 1e-11)
    assert np.allclose(out["auto"][0].T @ out["auto"][0], np.eye(k), atol=1e-10)


def test_lanczos_is_deterministic(oracle, monkeypatch):
    monkeypatch.setenv("VPCA_EIG", "auto")
    n = 1092
    S = _structured_gram(oracle, n, 8000)
    runs = []
    for _ in range(2):
        with _native(n) as nat:
            nat.setGram(S)
            runs.append(nat.computePca(2))
    assert np.array_equal(runs[0][0], runs[1][0]) and np.array_equal(runs[0][1], runs[1][1])


def test_flat_spectrum(oracle, monkeypatch):
    """No population structure: the top of the spectrum is the edge of a bulk (relative gaps < 1 %).  Lanczos needs
    more steps, or hands over to the direct reduction; either way the pairs must be eigenpairs of C."""
    monkeypatch.setenv("VPCA_EIG", "auto")
    rng = np.random.default_rng(11)
    n = 640
    B = (rng.random((n, 3000)) < 0.3).astype(np.int64)
    S = (B @ B.T).astype(np.int32)
    C, _, _ = oracle.np_center(S)
    w, V = np.linalg.eigh(C)
    with _native(n) as nat:
        nat.setGram(S)
        vecs, evals, _ = nat.computePca(2)
        st = nat.stats()
    assert st["eig_method"] in (2, 3), st
    assert np.allclose(evals, w[::-1][:2], rtol=1e-10)
    assert np.all(_residuals(C, vecs, evals) <= 1e-11)
    err = oracle.eigvec_rel_err(vecs, V[:, ::-1][:, :2])
    assert np.all(err <= TOL), err


def test_abandoned_lanczos_hands_over_to_the_direct_solver(oracle, monkeypatch):
    """Six components reach into the bulk and need > 32 Lanczos steps; with the step budget cut to one chunk the solve
    must fall back, and then it IS the direct solve, bit for bit."""
    n, nv, k = 1500, 6000, 6
    S = _structured_gram(oracle, n, nv)
    out = {}
    for name, env in (("direct", {"VPCA_EIG": "direct"}), ("cut", {"VPCA_EIG": "auto", "VPCA_EIG_MAXIT": "32"})):
        for key in ("VPCA_EIG", "VPCA_EIG_MAXIT"):
            monkeypatch.delenv(key, raising=False)
        for key, val in env.items():
            monkeypatch.setenv(key, val)
        with _native(n, num_pc=k) as nat:
            nat.setGram(S)
            out[name] = nat.computePca(k) + (nat.stats(),)
    assert out["cut"][3]["eig_method"] == 3 and out["cut"][3]["eig_iterations"] == 32
    assert np.array_equal(out["cut"][0], out["direct"][0]) and np.array_equal(out["cut"][1], out["direct"][1])


def test_multiple_top_eigenvalue_is_not_missed(oracle, monkeypatch):
    """Four identical, disjoint sample blocks: the top eigenvalue of the centred Gram has multiplicity 3.  A single
    Krylov sequence contains one vector of that eigenspace; the deflated re-run must notice (-> direct solver) unless
    rounding already brought the copies in.  Either way both returned eigenvalues are the top one."""
    monkeypatch.setenv("VPCA_EIG", "auto")
    rng = np.random.default_rng(5)
    nb = 160
    B = (rng.random((nb, 900)) < 0.25).astype(np.int64)
    B[:50, :300] = 1
    blk = B @ B.T
    n = 4 * nb
    S = np.zeros((n, n), np.int32)
    for g in range(4):
        S[g * nb:(g + 1) * nb, g * nb:(g + 1) * nb] = blk
    C, _, _ = oracle.np_center(S)
    w = np.linalg.eigvalsh(C)[::-1]
    assert abs(w[0] - w[2]) <= 1e-9 * w[0] and w[3] < 0.999 * w[0]     # the construction really is 3-fold degenerate
    with _native(n) as nat:
        nat.setGram(S)
        vecs, evals, _ = nat.computePca(2)
        st = nat.stats()
    assert st["eig_method"] in (2, 3), st
    assert np.allclose(evals, w[:2], rtol=1e-9), (evals, w[:4], st)
    assert np.all(_residuals(C, vecs, evals) <= 1e-9)
    assert np.allclose(vecs.T @ vecs, np.eye(2), atol=1e-9)


def test_top5_eigenvectors_random_psd(oracle):
    rng = np.random.default_rng(7)
    n = 300
    # integer Gram of a random low-rank-plus-noise design: well separated top-5
    B = rng.integers(0, 2, size=(n, 4000)).astype(np.int64)
    B[:60] |= rng.integers(0, 2, size=(1, 4000))
    B[60:150] |= rng.integers(0, 2, size=(1, 4000))
    B[150:210, ::3] = 1
    S = (B @ B.T).astype(np.int32)
    C, _, _ = oracle.np_center(S)
    w, V = np.linalg.eigh(C)
    with _native(n, num_pc=5) as nat:
        nat.setGram(S)
        vecs, evals, _ = nat.computePca(5)
    assert np.allclose(evals, w[::-1][:5], rtol=1e-10)
    gaps = np.abs(np.diff(w[::-1][:6]))
    assert gaps.min() > 1e-6 * w[-1]
    err = oracle.eigvec_rel_err(vecs, V[:, ::-1][:, :5])
    assert np.all(err <= TOL), err
    assert np.allclose(vecs.T @ vecs, np.eye(5), atol=1e-10)


def test_zero_gram_does_not_crash(oracle):
    n = 32
    with _native(n) as nat:
        nat.setGram(np.zeros((n, n), np.int32))
        vecs, evals, nz = nat.computePca(2)
    assert nz == 0
    assert np.all(np.isfinite(vecs)) and np.allclose(evals, 0.0)


def test_end_to_end_calls_to_pcs(oracle):
    """RDD[Seq[Int]] rows -> encode -> Gram -> PCA, all on device, vs the full oracle chain."""
    n, nv = 1092, 8000
    off, idx = oracle.c_synth_calls(SEED, n, 0, nv)
    S_want = oracle.c_similarity(n, off, idx, 4)
    want, _ = oracle.compute_pca(S_want, 2)
    with _native(n) as nat:
        nat.accumulateCalls(0, off, idx)
        nat.commit(0)
        nat.finalizeGram()
        vecs, evals, nz = nat.computePca(2)
    assert nz == n
    err = oracle.eigvec_rel_err(vecs, want)
    assert np.all(err <= TOL), err
    # README.md:109-119 property: unit-norm eigenvector entries of magnitude ~ 1/sqrt(N)
    assert 0.2 / np.sqrt(n) < np.abs(vecs[:, 0]).mean() < 2.0 / np.sqrt(n)
