"""GPU tests of the CTA-pair Gram kernel (VPCA_CTA_GROUP=2), whose two CTAs form a 2-CTA cluster: every B box is fetched
once, by one CTA, and multicast into both.  These are the schedules in which the two CTAs of a pair load different
things -- filler tiles of the exact block cover, self-B diagonal tiles, tiles of a single B box -- each bit-exact."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

SEED = 20240901
DTYPES = ["i8", "bf16", "e2m1"]


def _dtype(name):
    from spark_examples_b200 import native
    return {"i8": native.DTYPE_I8, "bf16": native.DTYPE_BF16, "e2m1": native.DTYPE_E2M1}[name]


def _gram_of_calls(n, dtype_name, off, idx):
    from spark_examples_b200 import native
    with native.NativePca(n, dtype=_dtype(dtype_name)) as nat:
        nat.accumulateCalls(-1, off, idx)
        nat.finalizeGram()
        S = nat.getGram()
        st = nat.stats()
    assert st["gram_cta_group"] == 2
    return S


def _pair_env(monkeypatch, kb_window=8):
    monkeypatch.setenv("VPCA_CTA_GROUP", "2")
    monkeypatch.setenv("VPCA_KB_WINDOW", str(kb_window))
    for k in ("VPCA_EXACT_COVER", "VPCA_SELF_B"):
        monkeypatch.delenv(k, raising=False)


@pytest.mark.parametrize("dtype_name", DTYPES)
def test_exact_cover_filler_tiles(oracle, monkeypatch, dtype_name):
    """Exact block cover: on a filler tile CTA 1 multiplies a copy of CTA 0's A block in lockstep and drops it."""
    from spark_examples_b200 import native
    _pair_env(monkeypatch)
    monkeypatch.setenv("VPCA_EXACT_COVER", "1")
    n, nv = 700, 3001
    assert (native.debugTiles(n, 2, True)[:, 5] & 2).any()      # kTileFiller
    X = oracle.c_synth_dense(SEED, n, 0, nv, mode=1)
    off, idx = oracle.dense_to_calls(X)
    assert np.array_equal(_gram_of_calls(n, dtype_name, off, idx), oracle.np_similarity_dense(X))


@pytest.mark.parametrize("dtype_name", DTYPES)
def test_self_b_tiles_match_loaded_b(oracle, monkeypatch, dtype_name):
    """Self-B diagonal tiles (each CTA multicasts its A block as half of the B rows) against loading the B rows."""
    from spark_examples_b200 import native
    _pair_env(monkeypatch)
    n, nv = 768, 3001                                            # three B strips of exactly 256 rows
    assert (native.debugTiles(n, 2, False)[:, 5] & 4).any()     # kTileSelfB
    X = oracle.c_synth_dense(SEED, n, 0, nv, mode=1)
    off, idx = oracle.dense_to_calls(X)
    got = {}
    for self_b in (0, 1):
        monkeypatch.setenv("VPCA_SELF_B", str(self_b))
        got[self_b] = _gram_of_calls(n, dtype_name, off, idx)
    assert np.array_equal(got[0], got[1])
    assert np.array_equal(got[1], oracle.np_similarity_dense(X))


@pytest.mark.parametrize("dtype_name", DTYPES)
def test_single_b_box_cohort(oracle, monkeypatch, dtype_name):
    """N <= 128: one B box per tile, issued by CTA 0 alone; CTA 1 loads only its (out-of-range, zero) A block."""
    _pair_env(monkeypatch)
    n, nv = 100, 5003
    X = oracle.c_synth_dense(SEED, n, 0, nv, mode=1)
    off, idx = oracle.dense_to_calls(X)
    assert np.array_equal(_gram_of_calls(n, dtype_name, off, idx), oracle.np_similarity_dense(X))


def test_panels_pair_matches_single_cta(monkeypatch):
    """2504 x 262 144 int8 panels (the benchmark's layout): CTA pairs and single CTAs give the same Gram."""
    import torch
    from spark_examples_b200 import native
    for k in ("VPCA_KB_WINDOW", "VPCA_EXACT_COVER", "VPCA_SELF_B"):
        monkeypatch.delenv(k, raising=False)
    n, nv, P = 2504, 262_144, 8192
    stream = torch.cuda.Stream()
    torch.cuda.set_stream(stream)
    got = {}
    X = None
    for cg in (1, 2):
        monkeypatch.setenv("VPCA_CTA_GROUP", str(cg))
        with native.NativePca(n, stream=stream.cuda_stream, max_multiplicity=1) as nat:
            if X is None:
                X = torch.empty(nat.panelBytes(nv, P), dtype=torch.uint8, device="cuda")
                nat.synthPanelsDevice(SEED, 0, nv, 0, X.data_ptr(), P)
            nat.accumulatePanels(X.data_ptr(), nv, P)
            nat.finalizeGram()
            got[cg] = nat.getGram()
            assert nat.stats()["gram_cta_group"] == cg
    assert np.array_equal(got[1], got[2])
    assert np.array_equal(got[2], got[2].T)
