""".bed rows staged through one double-buffered loop: the packed accumulate, loadings, projection and kinship calls stage in
their lane's buffers, and the driver-side calls (GRM, its loadings and projection, GLM, variant and sample QC) share one
pair of the context.  Rows 1 MB apart put 64 rows in a 64 MB chunk and 256 in a lane buffer, so 300 rows take 5 and 2
chunks and both buffers of each pair are reused.  Checked here: interleaved calls on one context give the bits of the
same calls on fresh contexts, the driver-side calls hold one staging pair between them, every call moves exactly its
rows and extra inputs to the device with the kernel launches of its chunks, and the GRM and GLM calls keep their device
memory across repeats."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

N = 200
NV = 300
STRIDE = 1 << 20
K = 2
QC_STEP = (64 << 20) // STRIDE        # rows per driver-side chunk (64 MB)
QC_CHUNKS = -(-NV // QC_STEP)
LANE_CHUNKS = -(-NV // 256)           # 256 rows of 1 MB fill a lane's 64 Mi-entry index buffer


@pytest.fixture(scope="module")
def rows():
    rng = np.random.default_rng(20261019)
    r = np.zeros((NV, STRIDE), np.uint8)
    r[:, :(N + 3) // 4] = rng.integers(0, 256, (NV, (N + 3) // 4), dtype=np.uint8)
    return r


@pytest.fixture(scope="module")
def pheno():
    rng = np.random.default_rng(7)
    y = rng.standard_normal(N)
    y[::17] = np.nan
    cc = (rng.random(N) < 0.4).astype(np.float64)
    cc[::23] = np.nan
    return y, cc


def held():
    from spark_examples_b200 import native
    return int(native.load_library().vpca_debug_device_bytes())


def _ctx():
    from spark_examples_b200 import native
    return native.NativePca(N)


def _pca_and_loadings(nat, rows):
    nat.accumulateBed(0, rows)
    nat.commit(0)
    nat.finalizeGram()
    vecs, evals, _ = nat.computePca(K)
    return nat.getGram(), vecs, evals, *nat.loadingsBed(K, rows)


def _grm(nat, rows):
    nat.grmBed(rows)
    return nat.grmFinalize(), nat.getGrm()


def _kinship(nat, rows):
    nat.kinshipBed(rows)
    return nat.kinshipPairs()


def _calls(rows, pheno):
    y, cc = pheno
    return {
        "variant_qc": lambda nat: nat.variantQcBed(rows),
        "grm": lambda nat: _grm(nat, rows),
        "glm_linear": lambda nat: (nat.glmBegin(y), nat.glmLinearBed(rows)),
        "glm_logistic": lambda nat: (nat.glmLogisticBegin(cc), nat.glmLogisticBed(rows)),
        "sample_missing": lambda nat: nat.sampleMissingBed(rows, N),
        "kinship": lambda nat: _kinship(nat, rows),
        "pca_loadings": lambda nat: _pca_and_loadings(nat, rows),
    }


def _bits(x):
    """every array of a (nested) result as its bytes, so that NaNs compare by their bits"""
    if isinstance(x, np.ndarray):
        return (x.dtype.str, x.shape, x.tobytes())
    if isinstance(x, (tuple, list)):
        return tuple(_bits(e) for e in x)
    return x


def test_interleaved_calls_match_fresh_contexts(rows, pheno):
    calls = _calls(rows, pheno)
    want = {}
    for name, call in calls.items():
        with _ctx() as nat:
            want[name] = _bits(call(nat))
    order = ["variant_qc", "grm", "glm_linear", "glm_logistic", "sample_missing", "kinship", "pca_loadings",
             "glm_linear", "variant_qc", "glm_logistic", "sample_missing"]
    with _ctx() as nat:
        for name in order:
            assert _bits(calls[name](nat)) == want[name], name


def test_driver_side_calls_share_one_staging_pair(rows):
    with _ctx() as nat:
        nat.grmBed(rows)
        base = held()
        nat.variantQcBed(rows)
        assert held() - base <= NV * (4 * 4 + 8)        # the counts and p-values of one batch, no rows
        base = held()
        nat.sampleMissingBed(rows, N)
        assert held() - base <= 4 * N                   # the per-sample counts, no rows


def _moved(nat, call):
    """(H2D bytes, kernel launches) of one call"""
    a = nat.stats()
    call()
    b = nat.stats()
    return b["h2d_bytes"] - a["h2d_bytes"], b["kernel_launches"] - a["kernel_launches"]


def test_h2d_bytes_and_launches_per_chunk(rows, pheno):
    y, cc = pheno
    raw = NV * STRIDE
    rng = np.random.default_rng(3)
    with _ctx() as nat:
        # lane-staged: encode + Gram, encode + loadings, encode + 2 projection kernels, planes + plane Gram per chunk
        assert _moved(nat, lambda: nat.accumulateBed(0, rows)) == (raw, 2 * LANE_CHUNKS)
        nat.commit(0)
        nat.finalizeGram()
        nat.computePca(K)
        assert _moved(nat, lambda: nat.loadingsBed(K, rows)) == (raw, 2 * LANE_CHUNKS)
        nat.projectBegin(K)
        w, mean = rng.standard_normal((NV, K)), rng.random(NV)
        assert _moved(nat, lambda: nat.projectBed(rows, w, mean)) == (raw + NV * (K + 1) * 8, 3 * LANE_CHUNKS)
        assert _moved(nat, lambda: nat.kinshipBed(rows)) == (raw, 2 * LANE_CHUNKS)
        # driver-side: one count kernel per chunk and one HWE launch per batch (one batch here)
        assert _moved(nat, lambda: nat.variantQcBed(rows)) == (raw, QC_CHUNKS + 1)
        assert _moved(nat, lambda: nat.variantQcBed(rows, hwe=False)) == (raw, QC_CHUNKS)
        assert _moved(nat, lambda: nat.sampleMissingBed(rows, N)) == (raw, QC_CHUNKS)
        keep = np.arange(0, N, 3, dtype=np.int32)
        assert _moved(nat, lambda: nat.subsetBedSamples(rows, N, keep)) == (raw + 4 * len(keep), QC_CHUNKS)
        # counts, tables, used list and one panel expand per chunk (every row varies; 300 columns never fill a panel)
        assert _moved(nat, lambda: nat.grmBed(rows)) == (raw, 4 * QC_CHUNKS)
        nat.grmFinalize()
        nat.computePcaGrm(K)
        out = {}
        assert _moved(nat, lambda: out.update(lt=nat.grmLoadingsBed(K, rows))) == (raw, 3 * QC_CHUNKS)
        gw, tab = out["lt"]
        nat.projectBegin(K)
        assert _moved(nat, lambda: nat.projectGrmBed(rows, tab, gw)) == (raw + NV * (K + 4) * 8, 2 * QC_CHUNKS)
        nat.glmBegin(y)
        assert _moved(nat, lambda: nat.glmLinearBed(rows)) == (raw, 3 * QC_CHUNKS)
        nat.glmLogisticBegin(cc)
        assert _moved(nat, lambda: nat.glmLogisticBed(rows)) == (raw, 5 * QC_CHUNKS)


def test_grm_and_glm_device_memory(rows, pheno):
    y, cc = pheno
    base = held()
    nat = _ctx()

    def run():
        nat.reset()
        nat.grmBed(rows)
        nat.grmFinalize()
        nat.computePcaGrm(K)
        w, tab = nat.grmLoadingsBed(K, rows)
        nat.projectBegin(K)
        nat.projectGrmBed(rows, tab, w)
        nat.glmBegin(y)
        nat.glmLinearBed(rows)
        nat.glmLogisticBegin(cc)
        nat.glmLogisticBed(rows)

    try:
        run()
        first = held()
        run()
        assert held() <= first, (held(), first)
    finally:
        nat.close()
    assert held() == base
