"""Principal coordinates straight from a Gram held as row bands (vpca_compute_pca_bands): Lanczos driven from rank 0 with
the mat-vec sharded over the band contexts, no replica of S and no N x N FP64 matrix.

Band contexts take no setGram, so every Gram here is built by the Gram kernel from panels (the synthetic generator, or
cells written with torch).  On a 1-GPU box the contexts share device 0, as in test_pool_gpu.py."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

SEED = 20240901
P = 1024


def _devices(world):
    import torch
    nd = max(1, torch.cuda.device_count())
    return [g % nd for g in range(world)]


def _panel_buffer(X, dev):
    """int8 cells X (n, nv) -> the panel layout of vpca_accumulate_panels on device `dev`"""
    import torch
    n, nv = X.shape
    npan = -(-nv // P)
    buf = np.zeros((npan, n, P), np.int8)
    for p in range(npan):
        blk = X[:, p * P:(p + 1) * P]
        buf[p, :, :blk.shape[1]] = blk
    return torch.from_numpy(buf.reshape(-1).view(np.uint8)).to(f"cuda:{dev}")


def _contexts(n, nv, world, form, cells=None, num_pc=2):
    """Finalized contexts holding the Gram of n samples x nv variants.  form "full": one context with the whole Gram;
    "flush": band-only contexts wired in owner-rows mode, each fed a contiguous shard of the variants; "computes":
    band-only contexts without peers, each fed every variant.  cells: int8 (n, nv), else the synthetic cohort."""
    import torch
    from spark_examples_b200 import native
    devs = _devices(world)
    bands = [(0, n)] if form == "full" else native.ownerRowBands(n, world)
    assert len(bands) == world
    ctxs, bufs = [], []
    try:
        for r in range(world):
            band = None if form == "full" else bands[r]
            ctxs.append(native.NativePca(n, device=devs[r], max_multiplicity=1, num_pc=num_pc, gram_band=band))
        if form == "flush":
            native.setPeersLocal(ctxs, "owner_rows")
        shards = [(r * nv // world, (r + 1) * nv // world) for r in range(world)] if form == "flush" else [(0, nv)] * world
        for r, c in enumerate(ctxs):
            v0, v1 = shards[r]
            with torch.cuda.device(devs[r]):
                if cells is None:
                    buf = torch.zeros(c.panelBytes(v1 - v0, P), dtype=torch.uint8, device=f"cuda:{devs[r]}")
                    torch.cuda.synchronize(devs[r])   # zeroed before the context's own stream writes the cells
                    c.synthPanelsDevice(SEED, v0, v1 - v0, 0, buf.data_ptr(), P)
                else:
                    buf = _panel_buffer(np.ascontiguousarray(cells[:, v0:v1]), devs[r])
            bufs.append(buf)
        for c in ctxs:
            c.reset()
        for c in ctxs:
            c.synchronize()                       # every band is zero before any rank adds into it
        for r, c in enumerate(ctxs):
            c.accumulatePanels(bufs[r].data_ptr(), shards[r][1] - shards[r][0], P)
        if form == "flush":
            for c in ctxs:
                c.gatherGram()
        for c in ctxs:
            c.synchronize()
        for c in ctxs:
            c.finalizeGram()
        return ctxs
    except Exception:
        _close(ctxs)
        raise


def _close(ctxs):
    for c in ctxs:
        try:
            c.synchronize()
        except Exception:
            pass
    for c in ctxs:
        c.close()


_REF = {}


def _reference(oracle, n, nv, k):
    """S, eigvalsh of the centred S (descending), nonZeroRows and the oracle's top-k vectors of the synthetic cohort"""
    key = (n, nv)
    if key not in _REF:
        S = oracle.np_similarity_dense(oracle.c_synth_dense(SEED, n, 0, nv, 0))
        C, _, nz = oracle.np_center(S)
        _REF[key] = {"S": S, "w": np.linalg.eigvalsh(C)[::-1], "nz": nz}
    ref = _REF[key]
    if k not in ref:
        ref[k] = oracle.compute_pca(ref["S"], k)[0]
    return ref["S"], ref["w"], ref["nz"], ref[k]


def _check_vectors(vecs, k, n):
    assert vecs.shape == (n, k)
    assert np.allclose(np.linalg.norm(vecs, axis=0), 1.0, atol=1e-12)
    for c in range(k):
        assert vecs[np.argmax(np.abs(vecs[:, c])), c] > 0          # sign rule: largest-|.| entry positive


@pytest.mark.parametrize("k", [2, 5])
@pytest.mark.parametrize("world,form", [(1, "full"), (2, "flush"), (2, "computes"), (4, "flush"), (4, "computes")])
def test_band_pca_matches_oracle(oracle, world, form, k):
    """N = 2504 x 4096 synthetic variants: the band solve against the oracle's MLlib recipe, against eigvalsh of the
    centred S, and against vpca_compute_pca of a full context on the same cohort."""
    from spark_examples_b200 import native
    n, nv = 2504, 4096
    S, w, nz_want, U = _reference(oracle, n, nv, k)
    ctxs = _contexts(n, nv, world, form)
    try:
        vecs, evals, nz = native.computePcaBands(ctxs, k)
        st = ctxs[0].stats()
    finally:
        _close(ctxs)
    assert st["eig_method"] == 4 and 16 <= st["eig_iterations"] <= 320 and st["last_eig_ms"] > 0, st
    assert nz == nz_want
    _check_vectors(vecs, k, n)
    assert np.all(oracle.eigvec_rel_err(vecs, U) <= 1e-6)
    assert np.allclose(evals, w[:k], rtol=1e-10)
    with native.NativePca(n, num_pc=k) as full:
        full.setGram(S)
        fvecs, fevals, fnz = full.computePca(k)
    assert fnz == nz
    assert np.all(oracle.eigvec_rel_err(vecs, fvecs) <= 1e-6)
    assert np.allclose(evals, fevals, rtol=1e-10)


@pytest.mark.parametrize("form", ["flush", "computes"])
def test_band_pca_is_reproducible_and_leaves_the_bands_alone(form):
    from spark_examples_b200 import native
    n, nv, world = 2504, 4096, 4
    ctxs = _contexts(n, nv, world, form)
    try:
        bands = [(c_.gramBand(*b)) for c_, b in zip(ctxs, native.ownerRowBands(n, world))]
        runs = [native.computePcaBands(ctxs, 3) for _ in range(2)]
        after = [(c_.gramBand(*b)) for c_, b in zip(ctxs, native.ownerRowBands(n, world))]
    finally:
        _close(ctxs)
    assert np.array_equal(runs[0][0], runs[1][0]) and np.array_equal(runs[0][1], runs[1][1])
    assert runs[0][2] == runs[1][2]
    for b0, b1 in zip(bands, after):
        assert np.array_equal(b0, b1)


def test_band_pca_past_the_reference_sample_limit():
    """N = 70 000 (MLlib's RowMatrix stops at 65 535 columns) on 4 band contexts, 2048 variants; reference: the top left
    singular vectors of J X in FP64 (eigh of the 2048 x 2048 (JX)^T (JX), then u = JX v / sigma)."""
    import torch
    from spark_examples_b200 import native
    from oracle import oracle
    n, nv, world, k = 70_000, 2048, 4, 2
    free, _ = torch.cuda.mem_get_info()
    if free < 30 * 2 ** 30:
        pytest.skip("needs 30 GB of free HBM")
    ctxs = _contexts(n, nv, world, "flush")
    try:
        vecs, evals, nz = native.computePcaBands(ctxs, k)
        st = ctxs[0].stats()
    finally:
        _close(ctxs)
    # the same cells, regenerated by the same generator into one buffer
    with native.NativePca(n, max_multiplicity=1, gram_band=(0, 64)) as gen:     # a generator, not a 20 GB Gram
        buf = torch.zeros(gen.panelBytes(nv, nv), dtype=torch.uint8, device="cuda:0")
        torch.cuda.synchronize(0)   # zeroed before the context's own stream writes the cells
        gen.synthPanelsDevice(SEED, 0, nv, 0, buf.data_ptr(), nv)
        gen.synchronize()
    X = buf.view(torch.int8).view(n, nv).to(torch.float64)
    del buf
    assert nz == int((X.sum(dim=1) > 0).sum())
    JX = X - X.mean(dim=0, keepdim=True)
    del X
    lam, Vr = torch.linalg.eigh(JX.t() @ JX)
    lam, Vr = lam.flip(0)[:k], Vr.flip(1)[:, :k]
    U = ((JX @ Vr) / lam.sqrt()).cpu().numpy()
    lam = lam.cpu().numpy()
    del JX
    assert st["eig_method"] == 4, st
    _check_vectors(vecs, k, n)
    assert np.allclose(evals, lam, rtol=1e-9), (evals, lam)
    assert np.all(oracle.eigvec_rel_err(vecs, U) <= 1e-6)


def test_zero_gram_is_reported():
    from spark_examples_b200 import native
    n, world = 1024, 2
    bands = native.ownerRowBands(n, world)
    ctxs = []
    try:
        for r in range(world):
            ctxs.append(native.NativePca(n, device=_devices(world)[r], gram_band=bands[r]))
        for c in ctxs:
            c.finalizeGram()
        with pytest.raises(native.VpcaError) as ei:
            native.computePcaBands(ctxs, 2)
        assert ei.value.code == native.VPCA_ERR_UNSUPPORTED
        assert ctxs[0].stats()["eig_method"] == 4
    finally:
        _close(ctxs)


def test_step_budget_exhausted_is_reported(oracle, monkeypatch):
    """Six components reach into the bulk and need > 32 steps (the cohort of test_pca_gpu.py's abandoned-Lanczos test):
    with VPCA_EIG_MAXIT=32 the band solve stops after 32 steps and says so -- there is no direct solver to hand over to."""
    from spark_examples_b200 import native
    monkeypatch.setenv("VPCA_EIG_MAXIT", "32")
    n, nv, k = 1500, 6000, 6
    X = oracle.c_synth_dense(SEED, n, 0, nv, 0).astype(np.int8)
    ctxs = _contexts(n, nv, 2, "computes", cells=X, num_pc=k)
    try:
        with pytest.raises(native.VpcaError) as ei:
            native.computePcaBands(ctxs, k)
        st = ctxs[0].stats()
    finally:
        _close(ctxs)
    assert ei.value.code == native.VPCA_ERR_UNSUPPORTED
    assert st["eig_method"] == 4 and st["eig_iterations"] == 32, st


def test_multiple_top_eigenvalue_is_reported_or_right(oracle):
    """Four identical, disjoint sample blocks (test_pca_gpu.py's degenerate construction, as cells): the top eigenvalue
    of the centred Gram has multiplicity 3.  Either the verification run catches the missed copies, or the answer is
    right."""
    from spark_examples_b200 import native
    rng = np.random.default_rng(5)
    nb, vb = 160, 900
    B = (rng.random((nb, vb)) < 0.25).astype(np.int8)
    B[:50, :300] = 1
    n = 4 * nb
    X = np.zeros((n, 4 * vb), np.int8)
    for g in range(4):
        X[g * nb:(g + 1) * nb, g * vb:(g + 1) * vb] = B
    S = oracle.np_similarity_dense(X)
    C, _, _ = oracle.np_center(S)
    w = np.linalg.eigvalsh(C)[::-1]
    assert abs(w[0] - w[2]) <= 1e-9 * w[0] and w[3] < 0.999 * w[0]
    ctxs = _contexts(n, X.shape[1], 2, "computes", cells=X)
    try:
        try:
            vecs, evals, _ = native.computePcaBands(ctxs, 2)
        except native.VpcaError as exc:
            assert exc.code == native.VPCA_ERR_UNSUPPORTED
            return
    finally:
        _close(ctxs)
    assert np.allclose(evals, w[:2], rtol=1e-9), (evals, w[:4])
    res = np.linalg.norm(C @ vecs - vecs * evals[None, :], axis=0) / np.abs(w).max()
    assert np.all(res <= 1e-9)


def test_argument_errors():
    from spark_examples_b200 import native
    n = 512
    (r0, m0), (r1, m1) = native.ownerRowBands(n, 2)
    dev = _devices(1)[0]
    made = []

    def ctx(band, nn=n):
        made.append(native.NativePca(nn, device=dev, gram_band=band))
        return made[-1]

    def status(ctxs, k=2):
        try:
            native.computePcaBands(ctxs, k)
        except native.VpcaError as exc:
            return exc.code
        return native.VPCA_OK

    try:
        a, b = ctx((r0, m0)), ctx((r1, m1))
        assert status([a, b]) == native.VPCA_ERR_STATE                     # not finalized
        a.finalizeGram()
        assert status([a, b]) == native.VPCA_ERR_STATE                     # one of them not finalized
        b.finalizeGram()
        assert status([b, a]) == native.VPCA_ERR_BAD_ARG                   # out of order
        gap = ctx((r1 + 32, m1 - 32))
        assert status([a, gap]) == native.VPCA_ERR_BAD_ARG                 # rows [m0, m0 + 32) missing
        over = ctx((r1 - 32, m1 + 32))
        assert status([a, over]) == native.VPCA_ERR_BAD_ARG                # rows [m0 - 32, m0) twice
        assert status([a]) == native.VPCA_ERR_BAD_ARG                      # does not reach N
        assert status([a, a]) == native.VPCA_ERR_BAD_ARG
        other = ctx((r1, 600 - r1), nn=600)
        assert status([a, other]) == native.VPCA_ERR_BAD_ARG               # mixed N
        assert status([a, b], k=0) == native.VPCA_ERR_BAD_ARG
        assert status([a, b], k=17) == native.VPCA_ERR_BAD_ARG
    finally:
        _close(made)
