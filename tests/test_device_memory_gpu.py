"""Device memory of a context: every buffer a call needs is kept and grown, never allocated anew on a repeat of the same
call, and vpca_destroy releases all of it.  Measured with vpca_debug_device_bytes, the bytes every context of the process
holds, as deltas (other contexts of the process may be alive)."""
import threading

import numpy as np
import pytest

from eig_ref import P, compute_pca, solver_env, synth_cells

pytestmark = pytest.mark.gpu

N = 256
NV = 2048


def held():
    from spark_examples_b200 import native
    return int(native.load_library().vpca_debug_device_bytes())


def _csr(rng, n, nv):
    counts = rng.integers(0, 12, nv)
    off = np.zeros(nv + 1, np.int64)
    np.cumsum(counts, out=off[1:])
    idx = np.concatenate([np.sort(rng.choice(n, c, replace=False)) for c in counts]).astype(np.int32)
    return off, idx


def _bed(rng, n, nv):
    return rng.integers(0, 256, (nv, (n + 3) // 4), dtype=np.uint8)


def _repeat_then_destroy(make, run):
    """make() -> a context (or list of them); run(ctx) twice: the second run holds no more than the first, and closing
    every context returns to the count before make()"""
    base = held()
    ctx = make()
    ctxs = ctx if isinstance(ctx, list) else [ctx]
    try:
        run(ctx)
        first = held()
        run(ctx)
        assert held() <= first, (held(), first)
    finally:
        for c in ctxs:
            c.close()
    assert held() == base


def test_create_counts_the_owned_gram_only():
    import torch
    from spark_examples_b200 import native
    base = held()
    with native.NativePca(N):
        assert held() - base == (N * N + 64) * 4
    assert held() == base
    gram = torch.zeros(N * N, dtype=torch.int32, device="cuda:0")
    torch.cuda.synchronize()
    with native.NativePca(N, d_gram=gram.data_ptr()):
        assert held() == base
    assert held() == base


def test_accumulate_on_every_lane():
    """CSR, bed and dense host input from as many threads as there are lanes, each into its own partition"""
    from spark_examples_b200 import native
    rng = np.random.default_rng(1)
    off, idx = _csr(rng, N, NV)
    bed = _bed(rng, N, NV)
    dense = rng.integers(0, 3, (N, NV), dtype=np.int8)
    lanes = 3

    def run(nat):
        def task(t):
            nat.accumulateCalls(3 * t, off, idx)
            nat.accumulateBed(3 * t + 1, bed)
            nat.accumulateCalls16(3 * t + 2, off, idx)
        threads = [threading.Thread(target=task, args=(t,)) for t in range(lanes)]
        for th in threads:
            th.start()
        for th in threads:
            th.join()
        for pid in range(3 * lanes):
            nat.commit(pid)
        nat.accumulateDense(dense)
        nat.synchronize()
        nat.reset()

    _repeat_then_destroy(lambda: native.NativePca(N, staging_lanes=lanes, partitions_in_flight=3 * lanes), run)


@pytest.mark.parametrize("env", [None, {"VPCA_LZ_PERSIST": "0"}, {"VPCA_EIG": "direct"}],
                         ids=["persistent-lanczos", "one-band-lanczos", "direct"])
def test_finalize_and_pca(env):
    """vpca_compute_pca on each side of the persistent Lanczos form's fit (the one-band solver past it), and direct"""
    from spark_examples_b200 import native
    n = 1092
    buf, _ = synth_cells(n, 4 * P)

    def run(nat):
        nat.reset()
        nat.accumulatePanels(buf.data_ptr(), 4 * P, P)
        nat.finalizeGram()
        with solver_env(env):
            compute_pca(nat, 4)

    _repeat_then_destroy(lambda: native.NativePca(n, max_multiplicity=1, num_pc=4), run)


def test_subset_loadings_and_projection():
    import torch
    from spark_examples_b200 import native
    rng = np.random.default_rng(2)
    buf, _ = synth_cells(N, 4 * P)
    off, idx = _csr(rng, N, NV)
    bed = _bed(rng, N, NV)
    keep = rng.random(N) < 0.8
    k = 3
    d_w = torch.zeros(4 * P * k, dtype=torch.float64, device="cuda:0")
    d_count = torch.zeros(4 * P, dtype=torch.int32, device="cuda:0")
    d_mean = torch.zeros(4 * P, dtype=torch.float64, device="cuda:0")
    torch.cuda.synchronize()

    def run(nat):
        nat.reset()
        nat.accumulatePanels(buf.data_ptr(), 4 * P, P)
        nat.finalizeGram()
        nat.computePcaSubset(keep, k)
        w, _ = nat.loadingsCalls(k, off, idx)
        nat.loadingsBed(k, bed)
        nat.loadingsPanels(k, buf.data_ptr(), 4 * P, P, d_w.data_ptr(), d_count.data_ptr())
        nat.projectBegin(k)
        nat.projectCalls(off, idx, w, np.zeros(NV))
        nat.projectBed(bed, w, np.zeros(NV))
        nat.projectPanels(buf.data_ptr(), 4 * P, P, d_w.data_ptr(), d_mean.data_ptr())
        nat.projectGet(np.ones(k))

    _repeat_then_destroy(lambda: native.NativePca(N, max_multiplicity=1, num_pc=k), run)


def test_kinship():
    from spark_examples_b200 import native
    bed = _bed(np.random.default_rng(3), N, NV)

    def run(nat):
        nat.reset()
        nat.kinshipBed(bed)
        nat.kinshipPairs()
        nat.kinshipPairs(0.1, max_pairs=10)

    _repeat_then_destroy(lambda: native.NativePca(N), run)


def test_ld_prune():
    from spark_examples_b200 import native
    rng = np.random.default_rng(4)
    bed = _bed(rng, N, NV)
    lo = np.maximum(0, np.arange(NV) - 100)
    eligible = rng.random(NV) < 0.9

    def run(nat):
        nat.ldPruneBed(bed, lo, 0.2, max_pairs=1000)
        nat.ldPruneBed(bed, lo, 0.2, max_pairs=1000, eligible=eligible)

    _repeat_then_destroy(lambda: native.NativePca(N), run)


def test_variant_qc():
    from spark_examples_b200 import native
    bed = _bed(np.random.default_rng(5), N, NV)

    def run(nat):
        counts, _ = nat.variantQcBed(bed)
        nat.variantQcBed(bed, hwe=False)
        nat.hweExact(counts)

    _repeat_then_destroy(lambda: native.NativePca(N), run)


def test_sample_qc():
    from spark_examples_b200 import native
    m = 3 * N
    bed = _bed(np.random.default_rng(6), m, NV)

    def run(nat):
        nat.sampleMissingBed(bed, m)
        nat.subsetBedSamples(bed, m, np.arange(0, m, 3))

    _repeat_then_destroy(lambda: native.NativePca(N), run)


def test_join_merge_and_hash_keys():
    from spark_examples_b200 import native
    rng = np.random.default_rng(7)
    rows = 3000
    keys = [b"chr1:%d:A:G" % rng.integers(0, 2000) for _ in range(rows)]
    off, idx = _csr(rng, N, rows)

    def run(nat):
        nat.joinRows(native.JOIN, keys, off, idx, n_left=rows // 2)
        nat.accumulateJoined(0)
        nat.commit(0)
        nat.joinRows(native.MERGE, keys, off, idx, variant_set_count=2)
        r, z = nat.joinSize()
        nat.joinFetch(r, z)
        nat.joinRows(native.JOIN, keys[:10], off[:11], idx[:off[10]], n_left=10)   # no right rows: no output calls
        nat.hashKeys(keys)
        nat.reset()

    _repeat_then_destroy(lambda: native.NativePca(N), run)


def test_join_without_calls_on_a_fresh_context():
    """The first join of a context yields rows but no calls: the output index buffer is still allocated (one call at
    least), and the rows encode and accumulate as empty variants"""
    from spark_examples_b200 import native
    keys = [b"chr1:%d" % (q % 50) for q in range(200)]
    off = np.zeros(len(keys) + 1, np.int64)
    idx = np.zeros(0, np.int32)

    def run(nat):
        rows, nnz = nat.joinRows(native.JOIN, keys, off, idx, n_left=100)
        assert rows > 0 and nnz == 0
        got_off, got_idx = nat.joinFetch(rows, nnz)
        assert not got_off.any() and len(got_idx) == 0
        nat.accumulateJoined(0)
        nat.commit(0)
        nat.finalizeGram()
        assert not nat.getGram().any()
        nat.reset()

    _repeat_then_destroy(lambda: native.NativePca(N), run)


def test_hash_keys_keeps_nothing():
    from spark_examples_b200 import native
    with native.NativePca(N) as nat:
        before = held()
        nat.hashKeys([b"chr%d:%d" % (c, p) for c in range(3) for p in range(1000)])
        assert held() == before


def test_two_band_contexts_on_one_device():
    """vpca_compute_pca_bands with rank 1's copy of U and both ranks' shares of the mat-vec on device 0"""
    from spark_examples_b200 import native
    n = 1092
    buf, _ = synth_cells(n, 4 * P)
    bands = native.ownerRowBands(n, 2)

    def make():
        return [native.NativePca(n, max_multiplicity=1, num_pc=4, gram_band=b) for b in bands]

    def run(ctxs):
        for c in ctxs:
            c.reset()
            c.synchronize()
        for c in ctxs:
            c.accumulatePanels(buf.data_ptr(), 4 * P, P)
            c.finalizeGram()
        native.computePcaBands(ctxs, 4)

    _repeat_then_destroy(make, run)
