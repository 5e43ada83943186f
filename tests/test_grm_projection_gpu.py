"""GRM loadings and projection on the GPU (vpca_grm_loadings_bed, vpca_grm_project_bed; DESIGN.md 14): the loadings
against Z^T U in FP64 at every k from 1 to 16 and at the kernels' tile edges, the tables bit for bit against the Python
floats of tests/grm_ref.py, the bits of w across call splits, chunk caps and strides, the reference cohort projected back
onto its own PCs, a new cohort against the numpy formula, swapped alleles, determinism, the state rules, and the driver
end to end (relatives placed on the GRM axes of an unrelated set)."""
import numpy as np
import pytest

import grm_projection_ref as ref
import grm_ref
from spark_examples_b200 import native, plink, variants_pca

pytestmark = pytest.mark.gpu

FLIP = np.array([3, 1, 2, 0], np.uint8)   # .bed code with A1 and A2 swapped
SWAP = [3, 1, 2, 0]                       # a table re-indexed for it


def _bits(a):
    return np.ascontiguousarray(a, np.float64).view(np.int64)


def _code(seed, n, nv, miss=0.02):
    """(nv, n) codes with a monomorphic, an all-missing and a one-called row at the front."""
    code = grm_ref.balding_nichols(np.random.default_rng(seed), n, nv, miss=miss)
    if nv >= 3:
        code[0] = 0
        code[1] = 1
        code[2] = 1
        code[2, 0] = 2
    return code


def _padded(rows, extra, seed):
    """rows with `extra` bytes of noise after each, and noise in the padding bits of the last real byte."""
    rng = np.random.default_rng(seed)
    nv, nb = rows.shape
    out = rng.integers(0, 256, (nv, nb + extra), dtype=np.uint8)
    out[:, :nb] = rows
    return out


def _solve(nat, rows, k):
    nat.grmBed(rows)
    m = nat.grmFinalize()
    vecs, evals = nat.computePcaGrm(k)
    return m, vecs, evals


def _check_loadings(w, tab, rows, n, U):
    W, tab_ref, bound = ref.loadings(rows, n, U)
    assert np.array_equal(_bits(tab), _bits(tab_ref))
    err = np.abs(w - W)
    assert np.all(err <= bound), f"max err {err.max():.3e} (bound there {bound.flat[err.argmax()]:.3e})"


# ---- loadings against Z^T U --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n,nv", [(2, 40), (3, 41), (4, 255), (5, 256), (127, 257), (128, 300), (129, 300),
                                  (255, 513), (256, 600), (257, 600), (2504, 3000)])
def test_loadings_every_k(n, nv):
    code = _code(n * 7 + nv, n, nv)
    rows = grm_ref.pack(code)
    kmax = min(n, 16)
    with native.NativePca(n, num_pc=16) as nat:
        _, U, _ = _solve(nat, rows, kmax)
        prev = None
        for k in range(1, kmax + 1):
            w, tab = nat.grmLoadingsBed(k, rows)
            _check_loadings(w, tab, rows, n, U[:, :k])
            if prev is not None:   # vpca.h: the first k' columns keep their bits at a larger k
                assert np.array_equal(_bits(w[:, :k - 1]), _bits(prev))
            prev = w
        padded = _padded(rows, 5, n)
        w2, tab2 = nat.grmLoadingsBed(kmax, padded)
        assert np.array_equal(_bits(w2), _bits(prev)) and np.array_equal(_bits(tab2), _bits(tab))


def _free_hbm_gib():
    """Free device memory after handing back the blocks torch's caching allocator keeps from earlier tests (their FP64
    references at 21 845 samples hold tens of GB), so that a context at the sample limit can allocate its ~53 GB."""
    import torch
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    return torch.cuda.mem_get_info()[0] / 2 ** 30


def _context_gib(n):
    """A GRM context at n samples: the int32 Gram, the FP64 matrix, the panel and the Krylov basis, with room to spare."""
    return 1.1 * (12 * n * n + 8 * (1024 + 400) * n) / 2 ** 30 + 1


@pytest.mark.parametrize("n,k,nv", [(21845, 16, 400), (65535, 2, 200)])
def test_loadings_large_cohorts(n, k, nv):
    free = _free_hbm_gib()
    if free < _context_gib(n):   # a device shared with other work: skip as the GRM's own limit test does
        pytest.skip(f"needs {_context_gib(n):.0f} GiB of free HBM, {free:.1f} GiB free")
    rows = grm_ref.pack(_code(n, n, nv, miss=0.01))
    with native.NativePca(n, num_pc=16) as nat:
        _, U, _ = _solve(nat, rows, k)
        w, tab = nat.grmLoadingsBed(k, rows)
    _check_loadings(w, tab, rows, n, U)


def test_loadings_bits_across_splits_chunks_and_strides():
    n = 8
    nv = (1 << 20) + 5                       # two chunks: the 2^20-row cap
    code = np.random.default_rng(3).integers(0, 4, (nv, n)).astype(np.uint8)
    rows = grm_ref.pack(code)
    with native.NativePca(n, num_pc=16) as nat:
        _solve(nat, rows, 4)
        w, tab = nat.grmLoadingsBed(4, rows)
        parts = [nat.grmLoadingsBed(4, rows[lo:hi]) for lo, hi in ((0, 1000), (1000, 1001), (1001, nv))]
        ones = [nat.grmLoadingsBed(4, rows[j:j + 1]) for j in range(0, 2000, 97)]
        wide = nat.grmLoadingsBed(4, _padded(rows[:50000], 13, 1))
        w_again, _ = nat.grmLoadingsBed(4, rows)
    assert np.array_equal(_bits(np.concatenate([p[0] for p in parts])), _bits(w))
    assert np.array_equal(_bits(np.concatenate([p[1] for p in parts])), _bits(tab))
    for j, (wj, tj) in zip(range(0, 2000, 97), ones):
        assert np.array_equal(_bits(wj[0]), _bits(w[j])) and np.array_equal(_bits(tj[0]), _bits(tab[j]))
    assert np.array_equal(_bits(wide[0]), _bits(w[:50000]))
    assert np.array_equal(_bits(w_again), _bits(w))


# ---- projection ---------------------------------------------------------------------------------------------------------
def _reference(n, nv, k, seed=11):
    rows = grm_ref.pack(_code(seed, n, nv, miss=0.01))
    with native.NativePca(n, num_pc=16) as nat:
        m, U, evals = _solve(nat, rows, k)
        w, tab = nat.grmLoadingsBed(k, rows)
    return rows, m, U, evals, w, tab


def _project(n, rows, tab, w, k, m, evals):
    with native.NativePca(n, num_pc=2) as nat:
        nat.projectBegin(k)
        nat.projectGrmBed(rows, tab, w)
        raw = nat.projectGet(np.ones(k))
        nat.projectBegin(k)
        nat.projectGrmBed(rows, tab, w)
        p = nat.projectGet(m * evals)
    return raw, p


@pytest.mark.parametrize("n,k", [(600, 4), (2504, 2), (513, 16)])
def test_reference_projected_onto_itself_gets_u_back(n, k):
    rows, m, U, evals, w, tab = _reference(n, 6000, k)
    _, p = _project(n, rows, tab, w, k, m, evals)
    Z, _ = grm_ref.z_matrix(rows, n)
    bound = ref.round_trip_bound(Z, U, evals, m) + 8 * ref.U_RND * np.abs(U)
    err = np.abs(p - U)
    assert np.all(err <= bound), f"max err {err.max():.3e}, max |u| {np.abs(U).max():.3e}"


@pytest.mark.parametrize("n2", [5, 511, 512, 513, 1500])
@pytest.mark.parametrize("nv", [1023, 1025, 3000])
def test_new_cohort_matches_the_formula(n2, nv):
    k = 4
    rows, m, U, evals, w, tab = _reference(300, nv, k, seed=nv)
    new = grm_ref.pack(_code(n2 + nv, n2, nv, miss=0.1))
    raw, p = _project(n2, new, tab, w, k, m, evals)
    want, bound = ref.projection(new, n2, tab, w)
    assert np.all(np.abs(raw - want) <= bound)
    assert np.array_equal(_bits(p), _bits(raw / (m * evals)[None, :]))
    # the padded stride and swapped alleles give the same bits; a second run too
    raw_pad, _ = _project(n2, _padded(new, 3, 5), tab, w, k, m, evals)
    flipped = grm_ref.pack(FLIP[_code(n2 + nv, n2, nv, miss=0.1)])
    raw_flip, _ = _project(n2, flipped, tab[:, SWAP], w, k, m, evals)
    raw_again, _ = _project(n2, new, tab, w, k, m, evals)
    for other in (raw_pad, raw_flip, raw_again):
        assert np.array_equal(_bits(other), _bits(raw))


# ---- state rules ----------------------------------------------------------------------------------------------------------
def _state(fn):
    with pytest.raises(native.VpcaError) as e:
        fn()
    return e.value.code


def test_state_rules():
    n, nv = 300, 500
    rows = grm_ref.pack(_code(5, n, nv))
    with native.NativePca(n, num_pc=16) as nat:
        assert _state(lambda: nat.grmLoadingsBed(2, rows)) == native.VPCA_ERR_STATE          # never solved
        nat.grmBed(rows)
        nat.grmFinalize()
        assert _state(lambda: nat.grmLoadingsBed(2, rows)) == native.VPCA_ERR_STATE          # finalized, not solved
        vecs, _ = nat.computePcaGrm(3)                                                       # direct: consumes the GRM
        assert _state(lambda: nat.getGrm()) == native.VPCA_ERR_STATE
        w, _ = nat.grmLoadingsBed(3, rows)                                                   # U outlives the GRM
        _check_loadings(w, nat.grmLoadingsBed(3, rows)[1], rows, n, vecs)
        assert _state(lambda: nat.grmLoadingsBed(4, rows)) == native.VPCA_ERR_BAD_ARG        # k > k solved
        assert _state(lambda: nat.grmLoadingsBed(0, rows)) == native.VPCA_ERR_BAD_ARG
        assert _state(lambda: nat.loadingsBed(2, rows)) == native.VPCA_ERR_STATE             # no carrier U
        assert _state(lambda: nat.projectGrmBed(rows, np.zeros((nv, 4)), np.zeros((nv, 2)))) == native.VPCA_ERR_STATE
        nat.reset()
        assert _state(lambda: nat.grmLoadingsBed(2, rows)) == native.VPCA_ERR_STATE          # reset
    with native.NativePca(n, num_pc=16) as nat:                                              # a carrier solve ends it
        nat.accumulateBed(0, rows, 1)
        nat.commit(0)
        nat.finalizeGram()
        nat.grmBed(rows)
        nat.grmFinalize()
        nat.computePcaGrm(2)
        nat.grmLoadingsBed(2, rows)
        nat.computePca(2)
        assert _state(lambda: nat.grmLoadingsBed(2, rows)) == native.VPCA_ERR_STATE


# ---- the driver: relatives on the GRM axes of an unrelated set -------------------------------------------------------------
def test_driver_relatives_on_grm_axes(tmp_path, capsys):
    n_in, n_rel, nv = 600, 60, 4000
    rng = np.random.default_rng(21)
    code = grm_ref.balding_nichols(rng, n_in, nv, miss=0.01)
    parents = rng.integers(0, n_in, (n_rel, 2))
    # a relative takes each call from one of two kept samples, with a few calls missing
    pick = rng.random((nv, n_rel)) < 0.5
    rel = np.where(pick, code[:, parents[:, 0]], code[:, parents[:, 1]])
    rel[rng.random((nv, n_rel)) < 0.02] = 1
    allc = np.concatenate([code, rel], axis=1)
    d = np.where(allc == 0, 2, np.where(allc == 2, 1, np.where(allc == 3, 0, -1))).T
    prefix = str(tmp_path / "c")
    fam = [(f"F{i}", f"I{i}") for i in range(n_in + n_rel)]
    plink.write_fileset(prefix, d, fam=fam)
    (tmp_path / "in.id").write_text("".join(f"F{i}\tI{i}\n" for i in range(n_in)))
    (tmp_path / "out.id").write_text("".join(f"F{i}\tI{i}\n" for i in range(n_in, n_in + n_rel)))
    R, Q, Qin, npz = (str(tmp_path / x) for x in ("R", "Q", "Qin", "r.npz"))
    variants_pca.main(["--bed-path", prefix, "--keep", str(tmp_path / "in.id"), "--grm", "--num-pc", "4",
                       "--save-grm-loadings", npz, "--output-path", R])
    variants_pca.main(["--bed-path", prefix, "--keep", str(tmp_path / "out.id"), "--project-loadings", npz,
                       "--output-path", Q])
    variants_pca.main(["--bed-path", prefix, "--keep", str(tmp_path / "in.id"), "--project-loadings", npz,
                       "--output-path", Qin])
    out = capsys.readouterr().out
    assert out.count(f"GRM projection: {nv} of {nv} loadings variants found in this cohort (0 with A1/A2 swapped).") == 2

    def read(p):
        lines = open(p + ".eigenvec").read().splitlines()[1:]
        return np.array([[float(x) for x in ln.split("\t")[2:]] for ln in lines])
    U, P_rel, P_in = read(R), read(Q), read(Qin)
    with np.load(npz) as f:
        m, evals, w, tab = int(f["n_used"]), f["eigenvalues"], f["loadings"], f["z_table"]
        assert str(f["matrix"]) == "grm" and w.shape == (nv, 4) and int(f["n_samples"]) == n_in
    rows_in = grm_ref.pack(code)
    Z, _ = grm_ref.z_matrix(rows_in, n_in)
    bound = ref.round_trip_bound(Z, U, evals, m) + 8 * ref.U_RND * np.abs(U)
    assert np.all(np.abs(P_in - U) <= bound)
    raw, rb = ref.projection(grm_ref.pack(rel), n_rel, tab, w)
    want = raw / (m * evals)[None, :]
    assert np.all(np.abs(P_rel - want) <= rb / (m * evals)[None, :] + 4 * ref.U_RND * np.abs(want))
