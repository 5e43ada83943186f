"""Variant loadings after vpca_compute_pca_bands: every context of a band solve holds U on its own device, so each rank
computes the loadings of the variants it holds (calls, .bed rows or panels), band-only contexts included; past 65 535
samples the loadings sum the samples in 4 fixed ranges (project.cu: loadings_split_kernel up to k = 8,
loadings_ranged_kernel above).

The order of the sums is checked bit for bit against a numpy restatement: with 0/1 cells every product d * u is exact,
so an FMA and numpy's multiply-then-add round alike."""
import numpy as np
import pytest

from eig_ref import structured_cells
from projection_ref import dense_to_csr, np_project

pytestmark = pytest.mark.gpu

SEED = 20240901
COHORT_SEED = 20241015
P = 1024


def _devices(world):
    import torch
    nd = max(1, torch.cuda.device_count())
    return [g % nd for g in range(world)]


def _panel_buffer(X, dev, panel=P, dtype=0):
    """cells X (n, nv) -> the panel layout of vpca_accumulate_panels in the cell type `dtype` (0 int8, 1 bf16, 2 packed
    e2m1) on device `dev`, zero cells after nv"""
    import torch
    n, nv = X.shape
    npan = -(-nv // panel)
    pan = np.zeros((npan, n, panel), np.int64)
    for p in range(npan):
        blk = X[:, p * panel:(p + 1) * panel]
        pan[p, :, :blk.shape[1]] = blk
    if dtype == 0:
        host = pan.astype(np.int8).view(np.uint8)
    elif dtype == 1:
        host = (pan.astype(np.float32).view(np.uint32) >> 16).astype(np.uint16).view(np.uint8)   # exact for integers
    else:
        codes = (2 * pan).astype(np.uint8)
        host = codes[..., 0::2] | (codes[..., 1::2] << 4)
    return torch.from_numpy(np.ascontiguousarray(host).reshape(-1)).to(f"cuda:{dev}")


def _bed_rows(X):
    """0/1 cells (n, nv) -> .bed rows (nv, ceil(n / 4)): a carrier is a heterozygote, so it counts as a carrier of A1"""
    n, nv = X.shape
    code = np.where(X.T > 0, 2, 3).astype(np.uint8)
    pad = (-n) % 4
    if pad:
        code = np.concatenate([code, np.zeros((nv, pad), np.uint8)], axis=1)
    c4 = code.reshape(nv, -1, 4)
    return np.ascontiguousarray((c4[..., 0] | (c4[..., 1] << 2) | (c4[..., 2] << 4) | (c4[..., 3] << 6)).astype(np.uint8))


def _shards(nv, world, form):
    return [(r * nv // world, (r + 1) * nv // world) for r in range(world)] if form == "flush" else [(0, nv)] * world


def _contexts(n, nv, world, form, cells=None, num_pc=2, dtype=0, panel=P):
    """Finalized contexts holding the Gram of n samples x nv variants, and each rank's panels (device buffers of its
    shard).  form "full": one context with the whole Gram; "flush": band-only contexts wired in owner-rows mode, each fed
    a contiguous shard of the variants; "computes": band-only contexts without peers, each fed every variant.
    cells: int8 (n, nv), else the synthetic cohort (written by the generator in the context's own cell type)."""
    import torch
    from spark_examples_b200 import native
    devs = _devices(world)
    bands = [(0, n)] if form == "full" else native.ownerRowBands(n, world)
    ctxs, bufs = [], []
    try:
        for r in range(world):
            band = None if form == "full" else bands[r]
            ctxs.append(native.NativePca(n, device=devs[r], max_multiplicity=1, num_pc=num_pc, dtype=dtype,
                                         gram_band=band))
        if form == "flush":
            native.setPeersLocal(ctxs, "owner_rows")
        shards = _shards(nv, world, form)
        for r, c in enumerate(ctxs):
            v0, v1 = shards[r]
            with torch.cuda.device(devs[r]):
                if cells is None:
                    buf = torch.zeros(c.panelBytes(v1 - v0, panel), dtype=torch.uint8, device=f"cuda:{devs[r]}")
                    torch.cuda.synchronize(devs[r])   # zeroed before the context's own stream writes the cells
                    c.synthPanelsDevice(SEED, v0, v1 - v0, 0, buf.data_ptr(), panel)
                else:
                    buf = _panel_buffer(np.ascontiguousarray(cells[:, v0:v1]), devs[r], panel, dtype)
            bufs.append(buf)
        for c in ctxs:
            c.reset()
        for c in ctxs:
            c.synchronize()
        for r, c in enumerate(ctxs):
            c.accumulatePanels(bufs[r].data_ptr(), shards[r][1] - shards[r][0], panel)
        if form == "flush":
            for c in ctxs:
                c.gatherGram()
        for c in ctxs:
            c.synchronize()
        for c in ctxs:
            c.finalizeGram()
        return ctxs, bufs
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


def _panel_loadings(ctx, k, buf, nv, panel=P):
    """loadingsPanels on the context's device -> (w (nv, k), count (nv,)) on the host"""
    import torch
    dev = buf.device
    w = torch.zeros((max(nv, 1), k), dtype=torch.float64, device=dev)
    cnt = torch.zeros(max(nv, 1), dtype=torch.int32, device=dev)
    torch.cuda.synchronize(dev)                     # the zeros are written before the context's stream writes the outputs
    ctx.loadingsPanels(k, buf.data_ptr(), nv, panel, w.data_ptr(), cnt.data_ptr())
    ctx.synchronize()
    return w[:nv].cpu().numpy(), cnt[:nv].cpu().numpy()


def _rel(a, b):
    return np.max(np.abs(a - b), axis=0) / np.max(np.abs(b), axis=0)


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint64)


def _ordered_loadings(X, U, ranges):
    """w = sum over the sample ranges, in order, of each range's samples summed in order (the kernels' order)"""
    X = np.asarray(X)
    total = None
    for lo, hi in ranges:
        acc = np.zeros((X.shape[1], U.shape[1]))
        for s in range(lo, hi):
            acc += X[s].astype(np.float64)[:, None] * U[s][None, :]
        total = acc if total is None else total + acc
    return total


def _split_ranges(n):
    span = -(-(-(-n // 4)) // 32) * 32
    return [(min(n, j * span), min(n, (j + 1) * span)) for j in range(4)]


def _status(fn):
    from spark_examples_b200 import native
    try:
        fn()
    except native.VpcaError as exc:
        return exc.code
    return native.VPCA_OK


# ---- 1. parity at N = 2504 ------------------------------------------------------------------------------------------
_COHORT = {}


def _cohort(n, nv):
    """20 populations (eig_ref.structured_cells): the top 17 eigenvalues are separated, so the band solve reaches k = 16"""
    if (n, nv) not in _COHORT:
        _COHORT[n, nv] = structured_cells(n, nv, 20, COHORT_SEED)
    return _COHORT[n, nv]


@pytest.mark.parametrize("k", [2, 5, 16])
@pytest.mark.parametrize("world,form", [(1, "full"), (2, "flush"), (2, "computes"), (4, "flush"), (4, "computes")])
def test_every_rank_computes_the_loadings_of_its_variants(world, form, k):
    """Each rank's loadings of its shard against numpy FP64 X^T U of the returned U (1e-12), counts exact, and the bits
    of every variant the same on every rank and in the order the kernel promises; calls, .bed and panels on the last
    rank (a band-only context unless world 1) give the same bits."""
    from spark_examples_b200 import native
    n, nv = 2504, 4096
    X = _cohort(n, nv)
    ctxs, bufs = _contexts(n, nv, world, form, cells=X, num_pc=max(k, 2))
    try:
        U, evals, _ = native.computePcaBands(ctxs, k)
        shards = _shards(nv, world, form)
        per_rank = [_panel_loadings(c, k, bufs[r], shards[r][1] - shards[r][0]) for r, c in enumerate(ctxs)]
        last = ctxs[-1]
        calls = last.loadingsCalls(k, *dense_to_csr(X))
        bed = last.loadingsBed(k, _bed_rows(X), 1)
    finally:
        _close(ctxs)
    want = X.astype(np.float64).T @ U
    cnt_want = X.astype(np.int64).sum(axis=0)
    exact = _ordered_loadings(X, U, [(0, n)])
    for r, (w, cnt) in enumerate(per_rank):
        v0, v1 = shards[r]
        assert np.all(_rel(w, want[v0:v1]) <= 1e-12), (r, _rel(w, want[v0:v1]))
        assert np.array_equal(cnt, cnt_want[v0:v1]), r
        assert np.array_equal(_bits(w), _bits(exact[v0:v1])), r
        assert np.array_equal(_bits(w), _bits(calls[0][v0:v1])), r
    if form == "computes":
        for w, _ in per_rank[1:]:
            assert np.array_equal(_bits(w), _bits(per_rank[0][0]))
    assert np.array_equal(_bits(calls[0]), _bits(bed[0])) and np.array_equal(calls[1], bed[1])
    assert np.array_equal(calls[1], cnt_want)


# ---- 2. self-projection and a second cohort -------------------------------------------------------------------------
@pytest.mark.parametrize("k", [2, 5])
def test_band_loadings_project_the_reference_back_onto_u(oracle, k):
    """Loadings from 4 owner-flush ranks, gathered in variant order: the reference samples projected in an ordinary
    2504-sample context give their rows of U back (1e-9 of max |u|), and a second cohort of 700 samples gets numpy's
    projection (1e-10)."""
    from spark_examples_b200 import native
    n, nv, world = 2504, 4096, 4
    X = _cohort(n, nv)
    ctxs, bufs = _contexts(n, nv, world, "flush", cells=X, num_pc=k)
    try:
        U, evals, _ = native.computePcaBands(ctxs, k)
        shards = _shards(nv, world, "flush")
        parts = [_panel_loadings(c, k, bufs[r], shards[r][1] - shards[r][0]) for r, c in enumerate(ctxs)]
    finally:
        _close(ctxs)
    w = np.concatenate([p[0] for p in parts])
    cnt = np.concatenate([p[1] for p in parts])
    off, idx = dense_to_csr(X)
    with native.NativePca(n) as proj:
        proj.projectBegin(k)
        proj.projectCalls(off, idx, w, cnt / n)
        got = proj.projectGet(evals)
    err = np.max(np.abs(got - U), axis=0) / np.max(np.abs(U), axis=0)
    assert np.all(err <= 1e-9), err
    Y = oracle.c_synth_dense(SEED + 1, 700, 0, nv, 0).astype(np.int64)
    with native.NativePca(Y.shape[0]) as proj:
        proj.projectBegin(k)
        proj.projectCalls(*dense_to_csr(Y), w, cnt / n)
        got = proj.projectGet(evals)
    assert np.all(_rel(got, np_project(Y, w, cnt, n, evals)) <= 1e-10)


# ---- the split kernel's order below the threshold (forced), every cell type and component count ------------------------
@pytest.mark.parametrize("dtype", [0, 1, 2], ids=["int8", "bf16", "e2m1"])
def test_split_order_at_every_k_and_cell_type(monkeypatch, dtype):
    """VPCA_LOADINGS_KERNEL=split at N = 2504 (ranges of 640, 640, 640, 584 samples): k = 1 .. 16 (both kernels of the
    range order) give numpy's sums in range order bit for bit, through panels 384 and 1024 wide and CSR calls; the default kernel at this N gives the
    whole-range order."""
    import torch
    from spark_examples_b200 import native
    n, nv = 2504, 3001
    X = _cohort(n, 4096)[:, :nv]
    ctxs, _ = _contexts(n, nv, 1, "full", cells=X, num_pc=16, dtype=dtype)
    ks = (1, 2, 4, 5, 8, 9, 16)
    got = {}
    try:
        U, _, _ = ctxs[0].computePca(16)
        c = ctxs[0]
        got["whole"] = c.loadingsCalls(16, *dense_to_csr(X))
        monkeypatch.setenv("VPCA_LOADINGS_KERNEL", "split")
        csr = dense_to_csr(X)
        for k in ks:
            got["calls", k] = c.loadingsCalls(k, *csr)
        for pw in (384, 1024):
            d_x = _panel_buffer(X, 0, pw, dtype)
            for k in ks:
                got[pw, k] = _panel_loadings(c, k, d_x, nv, pw)
            del d_x
            torch.cuda.synchronize()
    finally:
        _close(ctxs)
    cnt_want = X.astype(np.int64).sum(axis=0)
    assert np.array_equal(_bits(got["whole"][0]), _bits(_ordered_loadings(X, U, [(0, n)])))
    split = _ordered_loadings(X, U, _split_ranges(n))
    assert not np.array_equal(_bits(split), _bits(got["whole"][0]))      # the two orders are told apart here
    for key, (w, cnt) in got.items():
        if key == "whole":
            continue
        k = key[1]
        assert np.array_equal(cnt, cnt_want), key
        assert np.array_equal(_bits(w), _bits(split[:, :k])), key


# ---- 3. past the sample limit ---------------------------------------------------------------------------------------
def _free_gb():
    import torch
    return torch.cuda.mem_get_info()[0] / 2 ** 30


def _generated_cells(n, nv):
    """The synthetic cohort as a (n, nv) int8 torch tensor on cuda:0 (a generator context, not a Gram)"""
    import torch
    from spark_examples_b200 import native
    with native.NativePca(n, max_multiplicity=1, gram_band=(0, 64)) as gen:
        buf = torch.zeros(gen.panelBytes(nv, nv), dtype=torch.uint8, device="cuda:0")
        torch.cuda.synchronize(0)   # zeroed before the context's own stream writes the cells
        gen.synthPanelsDevice(SEED, 0, nv, 0, buf.data_ptr(), nv)
        gen.synchronize()
    return buf.view(torch.int8).view(n, nv)


def test_band_loadings_past_the_reference_sample_limit():
    """N = 70 000 x 2048 variants on 4 owner-flush band contexts (the split kernel): loadings against torch FP64 X^T U
    (1e-12); the same bits through panels 1024 and 2048 wide, .bed rows and a second run; bf16 and e2m1 contexts of the
    same cohort (built one after another) give the same U and the same loadings bits as int8."""
    import torch
    from spark_examples_b200 import native
    n, nv, world, k = 70_000, 2048, 4, 2
    if _free_gb() < 30:
        pytest.skip("needs 30 GB of free HBM")
    shards = _shards(nv, world, "flush")
    results = {}
    for dtype in (0, 1, 2):
        ctxs, bufs = _contexts(n, nv, world, "flush", dtype=dtype)
        try:
            U, evals, _ = native.computePcaBands(ctxs, k)
            runs = [[_panel_loadings(c, k, bufs[r], shards[r][1] - shards[r][0]) for r, c in enumerate(ctxs)]
                    for _ in range(2)]
            if dtype == 0:
                del bufs
                wide = []
                for r, c in enumerate(ctxs):
                    v0, v1 = shards[r]
                    b2 = torch.zeros(c.panelBytes(v1 - v0, 2048), dtype=torch.uint8, device=f"cuda:{_devices(world)[r]}")
                    torch.cuda.synchronize(_devices(world)[r])   # zeroed before the context's own stream writes the cells
                    c.synthPanelsDevice(SEED, v0, v1 - v0, 0, b2.data_ptr(), 2048)
                    wide.append(_panel_loadings(c, k, b2, v1 - v0, 2048))
                    del b2
                X = _generated_cells(n, nv)
                bed = ctxs[1].loadingsBed(k, _bed_rows(X.cpu().numpy()), 1)        # a band-only rank, all variants
                results["wide"], results["bed"] = wide, bed
        finally:
            _close(ctxs)
        results[dtype] = (U, evals, runs)
    U, evals, runs = results[0]
    w = np.concatenate([p[0] for p in runs[0]])
    cnt = np.concatenate([p[1] for p in runs[0]])
    Xd = X.to(torch.float64)
    want = (Xd.t() @ torch.from_numpy(U).cuda()).cpu().numpy()
    cnt_want = Xd.sum(dim=0).cpu().numpy().astype(np.int64)
    del Xd, X
    assert np.all(_rel(w, want) <= 1e-12), _rel(w, want)
    assert np.array_equal(cnt, cnt_want)
    assert all(np.array_equal(_bits(a[0]), _bits(b[0])) for a, b in zip(runs[0], runs[1]))
    assert np.array_equal(_bits(np.concatenate([p[0] for p in results["wide"]])), _bits(w))
    assert np.array_equal(_bits(results["bed"][0]), _bits(w)) and np.array_equal(results["bed"][1], cnt)
    for dtype in (1, 2):
        U2, evals2, runs2 = results[dtype]
        assert np.array_equal(_bits(U2), _bits(U)) and np.array_equal(_bits(evals2), _bits(evals)), dtype
        assert np.array_equal(_bits(np.concatenate([p[0] for p in runs2[0]])), _bits(w)), dtype
        assert np.array_equal(np.concatenate([p[1] for p in runs2[0]]), cnt), dtype


@pytest.mark.parametrize("n", [65_535, 65_536, 65_537])
def test_split_boundaries_at_the_threshold(n):
    """1024 variants on 4 owner-flush band contexts at N = 65 535 (the last N of the whole-range kernel), 65 536 (the
    first of the split: 4 ranges of 16 384) and 65 537 (3 ranges of 16 416 and one of 16 289): numpy's sums in the
    kernel's order, bit for bit."""
    from spark_examples_b200 import native
    nv, world, k = 1024, 4, 2
    if _free_gb() < 30:
        pytest.skip("needs 30 GB of free HBM")
    shards = _shards(nv, world, "flush")
    ctxs, bufs = _contexts(n, nv, world, "flush")
    try:
        U, _, _ = native.computePcaBands(ctxs, k)
        parts = [_panel_loadings(c, k, bufs[r], shards[r][1] - shards[r][0]) for r, c in enumerate(ctxs)]
    finally:
        _close(ctxs)
    X = _generated_cells(n, nv).cpu().numpy()
    w = np.concatenate([p[0] for p in parts])
    ranges = [(0, n)] if n <= 65_535 else _split_ranges(n)
    if n == 65_537:
        assert [hi - lo for lo, hi in ranges] == [16_416, 16_416, 16_416, 16_289]
    assert np.array_equal(_bits(w), _bits(_ordered_loadings(X, U, ranges)))
    assert np.array_equal(np.concatenate([p[1] for p in parts]), X.astype(np.int64).sum(axis=0))


# ---- 4. states ------------------------------------------------------------------------------------------------------
def test_states_of_band_contexts(oracle, monkeypatch):
    from spark_examples_b200 import native
    n, nv = 1500, 6000
    X = oracle.c_synth_dense(SEED, n, 0, nv, 0).astype(np.int8)
    csr = dense_to_csr(X[:, :500])
    ctxs, _ = _contexts(n, nv, 2, "computes", cells=X, num_pc=6)
    try:
        for c in ctxs:                                                 # outside any solve
            assert _status(lambda: c.loadingsCalls(2, *csr)) == native.VPCA_ERR_UNSUPPORTED
        native.computePcaBands(ctxs, 3)
        first = [c.loadingsCalls(3, *csr) for c in ctxs]
        assert np.array_equal(_bits(first[0][0]), _bits(first[1][0]))
        for c in ctxs:
            assert _status(lambda: c.loadingsCalls(4, *csr)) == native.VPCA_ERR_BAD_ARG
        ctxs[1].reset()                                                # that rank only
        assert _status(lambda: ctxs[1].loadingsCalls(2, *csr)) == native.VPCA_ERR_UNSUPPORTED
        assert np.array_equal(_bits(ctxs[0].loadingsCalls(3, *csr)[0]), _bits(first[0][0]))
        ctxs[0].reset()
        for c in ctxs:                                                 # a zero Gram: the solve breaks down
            c.finalizeGram()
        with pytest.raises(native.VpcaError) as ei:
            native.computePcaBands(ctxs, 2)
        assert ei.value.code == native.VPCA_ERR_UNSUPPORTED
        for c in ctxs:
            assert _status(lambda: c.loadingsCalls(2, *csr)) == native.VPCA_ERR_UNSUPPORTED
    finally:
        _close(ctxs)
    # a failed solve clears U that an earlier solve left: the step budget of test_pca_bands_gpu.py's hard cohort
    ctxs, _ = _contexts(n, nv, 2, "computes", cells=X, num_pc=6)
    try:
        native.computePcaBands(ctxs, 2)
        monkeypatch.setenv("VPCA_EIG_MAXIT", "32")
        with pytest.raises(native.VpcaError):
            native.computePcaBands(ctxs, 6)
        for c in ctxs:
            assert _status(lambda: c.loadingsCalls(2, *csr)) == native.VPCA_ERR_UNSUPPORTED
    finally:
        _close(ctxs)


def test_states_of_a_full_context(oracle):
    from spark_examples_b200 import native
    n = 1024
    X = oracle.c_synth_dense(SEED, n, 0, 3000, 0).astype(np.int8)
    csr = dense_to_csr(X)
    with native.NativePca(n) as zero:                                  # a zero Gram: the band solve breaks down
        zero.finalizeGram()
        with pytest.raises(native.VpcaError):
            native.computePcaBands([zero], 2)
        assert _status(lambda: zero.loadingsCalls(2, *csr)) == native.VPCA_ERR_STATE
    ctxs, _ = _contexts(n, X.shape[1], 1, "full", cells=X, num_pc=4)
    try:
        c = ctxs[0]
        U3, _, _ = c.computePca(3)
        w3, _ = c.loadingsCalls(3, *csr)
        U2, _, _ = native.computePcaBands([c], 2)                      # the most recent solve wins
        assert _status(lambda: c.loadingsCalls(3, *csr)) == native.VPCA_ERR_BAD_ARG
        w2, _ = c.loadingsCalls(2, *csr)
        c.computePca(3)
        assert np.array_equal(_bits(c.loadingsCalls(3, *csr)[0]), _bits(w3))
    finally:
        _close(ctxs)
    assert np.array_equal(_bits(w2), _bits(_ordered_loadings(X, U2, [(0, n)])))
    assert np.array_equal(_bits(w3), _bits(_ordered_loadings(X, U3, [(0, n)])))


def test_projection_still_refuses_band_contexts(oracle):
    from spark_examples_b200 import native
    n, nv = 1024, 2048
    X = oracle.c_synth_dense(SEED, n, 0, nv, 0).astype(np.int8)
    ctxs, _ = _contexts(n, nv, 2, "flush", cells=X)
    try:
        native.computePcaBands(ctxs, 2)
        for c in ctxs:
            assert _status(lambda: c.projectBegin(2)) == native.VPCA_ERR_UNSUPPORTED
    finally:
        _close(ctxs)
