"""GPU parity tests of the encode + Gram kernels against the CPU oracle (bit-exact), through the C ABI.

Reference behaviour under test: VariantsPca.scala:56-60, :153-168 (encode) and :182-191 (similarity matrix)."""
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

SEED = 20240901


def _native(n, **kw):
    from spark_examples_b200 import native
    return native.NativePca(n, **kw)


def _set_env(monkeypatch, cta_group=None, kb_window=None):
    if cta_group is None:
        monkeypatch.delenv("VPCA_CTA_GROUP", raising=False)
    else:
        monkeypatch.setenv("VPCA_CTA_GROUP", str(cta_group))
    if kb_window is None:
        monkeypatch.delenv("VPCA_KB_WINDOW", raising=False)
    else:
        monkeypatch.setenv("VPCA_KB_WINDOW", str(kb_window))


def _random_rows(rng, n, nv, density=0.3, dup_every=0):
    rows = []
    for v in range(nv):
        k = rng.binomial(n, density)
        r = rng.choice(n, size=k, replace=False).astype(np.int32)
        if dup_every and v % dup_every == 0 and k > 0:
            r = np.concatenate([r, r[:1]])          # one sample listed twice (multi-dataset join case)
        rows.append(r)
    off = np.zeros(nv + 1, np.int64)
    off[1:] = np.cumsum([len(r) for r in rows])
    idx = np.concatenate(rows) if rows else np.zeros(0, np.int32)
    return off, idx.astype(np.int32), rows


def test_encode_tile_bit_exact(oracle):
    rng = np.random.default_rng(1)
    n, nv = 203, 517
    off, idx, rows = _random_rows(rng, n, nv, 0.2, dup_every=7)
    want = np.zeros((n, nv), np.int8)
    for v, r in enumerate(rows):
        np.add.at(want[:, v], r, 1)
    with _native(n) as nat:
        got = nat.encodeCalls(off, idx)
    assert got.dtype == np.int8 and got.shape == (n, nv)
    assert np.array_equal(got, want)


def test_encode_tile_bf16(oracle):
    rng = np.random.default_rng(2)
    n, nv = 130, 260
    off, idx, rows = _random_rows(rng, n, nv, 0.3, dup_every=5)
    want = np.zeros((n, nv), np.int64)
    for v, r in enumerate(rows):
        np.add.at(want[:, v], r, 1)
    from spark_examples_b200 import native
    with _native(n, dtype=native.DTYPE_BF16) as nat:
        got = nat.encodeCalls(off, idx)
    bf16_bits = {0: 0x0000, 1: 0x3F80, 2: 0x4000}
    want_bits = np.vectorize(bf16_bits.get)(want).astype(np.uint16)
    assert np.array_equal(got, want_bits)


@pytest.mark.parametrize("cta_group", [1, 2])
def test_gram_small_dense_host(oracle, monkeypatch, cta_group):
    _set_env(monkeypatch, cta_group)
    rng = np.random.default_rng(3)
    n, nv = 300, 1000
    X = (rng.random((n, nv)) < 0.35).astype(np.int8)
    with _native(n) as nat:
        nat.accumulateDense(X)
        nat.finalizeGram()
        S = nat.getGram()
        st = nat.stats()
    assert st["gram_cta_group"] == cta_group
    assert np.array_equal(S, oracle.np_similarity_dense(X))


@pytest.mark.parametrize("cta_group", [1, 2])
def test_gram_c1_calls_vs_reference_loop(oracle, monkeypatch, cta_group):
    """BASELINE configs[0]: 1092 samples x 8000 variants, through the RDD[Seq[Int]] entry point."""
    _set_env(monkeypatch, cta_group)
    n, nv = 1092, 8000
    off, idx = oracle.c_synth_calls(SEED, n, 0, nv)
    want = oracle.c_similarity(n, off, idx, 4)
    with _native(n) as nat:
        nat.accumulateCalls(-1, off, idx)
        nat.finalizeGram()
        S = nat.getGram()
    assert np.array_equal(S, want)
    assert np.array_equal(S, S.T)
    assert np.array_equal(np.diag(S), np.bincount(idx, minlength=n))


@pytest.mark.parametrize("cta_group", [1, 2])
def test_gram_multi_window_and_ragged_k(oracle, monkeypatch, cta_group):
    """Several L2 windows, K not a multiple of the 128-byte k-block, N not a multiple of the tile."""
    _set_env(monkeypatch, cta_group, kb_window=8)
    rng = np.random.default_rng(4)
    n, nv = 777, 5003
    X = (rng.random((n, nv)) < 0.25).astype(np.int8)
    X[:, 100] = 0                       # an empty variant
    X[5, :] = 0                         # a sample that never varies -> zero row/column must be present
    with _native(n) as nat:
        nat.accumulateDense(X[:, :3000])
        nat.accumulateDense(X[:, 3000:])    # accumulation across calls
        nat.finalizeGram()
        S = nat.getGram()
        st = nat.stats()
    assert st["gram_resident"] == 1
    assert np.array_equal(S, oracle.np_similarity_dense(X))
    assert not S[5].any() and not S[:, 5].any()


@pytest.mark.parametrize("cta_group", [1, 2])
def test_gram_stream_k_many_tiles(oracle, monkeypatch, cta_group):
    """More tiles than workers (N = 5000): the non-resident, double-buffered stream-K path."""
    _set_env(monkeypatch, cta_group)
    rng = np.random.default_rng(5)
    n, nv = 5000, 1500
    X = (rng.random((n, nv)) < 0.2).astype(np.int8)
    with _native(n) as nat:
        nat.accumulateDense(X)
        nat.finalizeGram()
        S = nat.getGram()
        st = nat.stats()
    assert st["gram_resident"] == 0
    Xf = X.astype(np.float32)
    want = (Xf @ Xf.T).astype(np.int32)          # exact: counts < 2^24
    assert np.array_equal(S, want)


@pytest.mark.parametrize("cta_group", [1, 2])
def test_gram_dosage_int8(oracle, monkeypatch, cta_group):
    _set_env(monkeypatch, cta_group)
    n, nv = 500, 2000
    X = oracle.c_synth_dense(SEED, n, 0, nv, mode=1)
    assert X.max() == 2
    with _native(n) as nat:
        nat.accumulateDense(X)
        nat.finalizeGram()
        S = nat.getGram()
    assert np.array_equal(S, oracle.np_similarity_dense(X))


@pytest.mark.parametrize("cta_group", [1, 2])
def test_gram_bf16(oracle, monkeypatch, cta_group):
    _set_env(monkeypatch, cta_group)
    from spark_examples_b200 import native
    n, nv = 640, 3001
    off, idx = oracle.c_synth_calls(SEED, n, 0, nv)
    want = oracle.c_similarity(n, off, idx, 2)
    with _native(n, dtype=native.DTYPE_BF16) as nat:
        nat.accumulateCalls(-1, off, idx)
        nat.finalizeGram()
        S = nat.getGram()
    assert np.array_equal(S, want)


def test_partition_commit_abort_exactly_once(oracle):
    """Task retry semantics (SURVEY 8b): an aborted partition leaves no trace, a committed one counts once."""
    n, nv = 400, 1200
    off, idx = oracle.c_synth_calls(SEED, n, 0, nv)
    nvk = len(off) - 1
    half = nvk // 2
    off_a, idx_a = off[: half + 1], idx[: off[half]]
    off_b, idx_b = off[half:] - off[half], idx[off[half]:]
    with _native(n) as nat:
        nat.accumulateCalls(0, off_a, idx_a)
        nat.accumulateCalls(1, off_b, idx_b)
        nat.abort(1)                                  # task 1 failed ...
        nat.accumulateCalls(1, off_b, idx_b)          # ... and was retried
        nat.commit(0)
        nat.commit(1)
        nat.commit(7)                                 # empty partition: no-op
        nat.finalizeGram()
        S = nat.getGram()
    assert np.array_equal(S, oracle.c_similarity(n, off, idx, 1))


def test_uncommitted_partition_blocks_finalize(oracle):
    from spark_examples_b200 import native
    n = 64
    off, idx = oracle.c_synth_calls(SEED, n, 0, 50)
    with _native(n) as nat:
        nat.accumulateCalls(3, off, idx)
        with pytest.raises(native.VpcaError) as ei:
            nat.finalizeGram()
        assert ei.value.code == native.VPCA_ERR_STATE


def test_index_out_of_range_is_an_error(oracle):
    from spark_examples_b200 import native
    n = 50
    off = np.array([0, 2, 3], np.int64)
    idx = np.array([1, 50, 2], np.int32)               # 50 == n: the reference throws (VariantsPca.scala:188)
    with _native(n) as nat:
        with pytest.raises(IndexError):
            nat.accumulateCalls(-1, off, idx)
        with pytest.raises(native.IndexOutOfRange):
            nat.accumulateCalls(5, off, np.array([1, -1, 2], np.int32))


def test_empty_and_degenerate_inputs(oracle):
    n = 40
    with _native(n) as nat:
        nat.accumulateCalls(-1, np.zeros(1, np.int64), np.zeros(0, np.int32))      # no rows
        nat.accumulateCalls(-1, np.array([0, 0, 0], np.int64), np.zeros(0, np.int32))  # two empty rows
        nat.accumulateCalls(-1, np.array([0, 1], np.int64), np.array([7], np.int32))   # a singleton
        nat.finalizeGram()
        S = nat.getGram()
    want = np.zeros((n, n), np.int32)
    want[7, 7] = 1
    assert np.array_equal(S, want)


def test_synth_device_matches_oracle_generator(oracle):
    import torch
    n, v0, nv = 333, 12345, 1003
    for mode in (0, 1):
        want = oracle.c_synth_dense(SEED, n, v0, nv, mode)
        ld = 1008
        buf = torch.zeros((n, ld), dtype=torch.int8, device="cuda")
        with _native(n) as nat:
            nat.synthDenseDevice(SEED, v0, nv, mode, buf.data_ptr(), ld)
            torch.cuda.synchronize()
        got = buf.cpu().numpy()
        assert np.array_equal(got[:, :nv], want)
        assert not got[:, nv:].any()


def test_resident_device_tile_full_properties(oracle):
    """Device-resident input at a size the O(N^2 V) oracle loop would not finish quickly: check the
    size-independent properties of SURVEY 8d (symmetry, diag = carrier counts, S.1 = X (X^T 1)) and
    bit-exactness on a random 4096-variant slice."""
    import torch
    n, nv = 2504, 200_000
    ld = nv
    X = torch.empty((n, ld), dtype=torch.int8, device="cuda")
    stream = torch.cuda.current_stream().cuda_stream
    with _native(n, stream=stream, max_multiplicity=1) as nat:
        nat.synthDenseDevice(SEED, 0, nv, 0, X.data_ptr(), ld)
        nat.accumulateDenseDevice(X.data_ptr(), nv, ld)
        nat.finalizeGram()
        S = nat.getGram()
    Xi = X.to(torch.int32)
    carriers = Xi.sum(dim=1).cpu().numpy()
    col = Xi.sum(dim=0).to(torch.float64)
    s1 = (X.to(torch.float64) @ col).cpu().numpy()
    assert np.array_equal(S, S.T)
    assert np.array_equal(np.diag(S), carriers)
    assert np.array_equal(S.sum(axis=1).astype(np.float64), s1)
    # slice parity through a fresh context on a 16-byte aligned column offset
    v0 = 77_776
    sl = oracle.c_synth_dense(SEED, n, v0, 4096, 0)
    with _native(n, stream=stream) as nat3:
        nat3.accumulateDenseDevice(X.data_ptr() + v0, 4096, ld)
        nat3.finalizeGram()
        S3 = nat3.getGram()
    assert np.array_equal(S3, oracle.np_similarity_dense(sl))


# ---------------------------------------------------------------------------------------------------------------
# packed 4-bit (e2m1) genotype storage: same Gram, half the HBM/L2 bytes per cell
# ---------------------------------------------------------------------------------------------------------------
def _pack_e2m1(X):
    """(n, nv) multiplicities in {0,1,2} -> packed (n, ld/2) uint8, ld = nv rounded up to 128."""
    n, nv = X.shape
    ld = ((nv + 127) // 128) * 128
    codes = np.zeros((n, ld), np.uint8)
    codes[:, :nv] = 2 * X.astype(np.uint8)
    return (codes[:, 0::2] | (codes[:, 1::2] << 4)).astype(np.uint8)


def test_encode_tile_e2m1(oracle):
    from spark_examples_b200 import native
    rng = np.random.default_rng(8)
    n, nv = 77, 300
    off, idx, rows = _random_rows(rng, n, nv, 0.3, dup_every=6)
    want = np.zeros((n, nv), np.int64)
    for v, r in enumerate(rows):
        np.add.at(want[:, v], r, 1)
    with _native(n, dtype=native.DTYPE_E2M1) as nat:
        got = nat.encodeCalls(off, idx)
    assert np.array_equal(got, _pack_e2m1(want))


@pytest.mark.parametrize("red64", [1, 0])
@pytest.mark.parametrize("cta_group", [1, 2])
def test_gram_e2m1_dense_and_calls(oracle, monkeypatch, cta_group, red64):
    """Packed 4-bit cells, expanded to int8 in shared memory: the exact Gram through both flushes (two cells per 64-bit
    red, or VPCA_RED64=0: one 32-bit red per cell)."""
    _set_env(monkeypatch, cta_group, kb_window=8)
    monkeypatch.setenv("VPCA_RED64", str(red64))
    from spark_examples_b200 import native
    n, nv = 700, 5003
    X = oracle.c_synth_dense(SEED, n, 0, nv, mode=1)           # dosage 0/1/2: all three codes
    want = oracle.np_similarity_dense(X)
    with _native(n, dtype=native.DTYPE_E2M1) as nat:
        nat.accumulateDense(_pack_e2m1(X), nv)
        nat.finalizeGram()
        assert np.array_equal(nat.getGram(), want)
    off, idx = oracle.dense_to_calls(X)
    with _native(n, dtype=native.DTYPE_E2M1) as nat:
        nat.accumulateCalls(-1, off, idx)
        nat.finalizeGram()
        assert np.array_equal(nat.getGram(), want)


def test_synth_device_e2m1_matches_oracle(oracle):
    import torch
    from spark_examples_b200 import native
    n, v0, nv = 333, 4096, 1003
    ld = 1024
    for mode in (0, 1):
        want = _pack_e2m1(oracle.c_synth_dense(SEED, n, v0, nv, mode))
        buf = torch.full((n, ld // 2), 0xEE, dtype=torch.uint8, device="cuda")
        with _native(n, dtype=native.DTYPE_E2M1) as nat:
            nat.synthDenseDevice(SEED, v0, nv, mode, buf.data_ptr(), ld)
            torch.cuda.synchronize()
        assert np.array_equal(buf.cpu().numpy(), want)            # includes the zeroed padding cells


def test_gram_e2m1_resident_matches_int8(oracle):
    import torch
    from spark_examples_b200 import native
    n, nv = 2504, 262_144
    stream = torch.cuda.Stream()
    torch.cuda.set_stream(stream)
    X8 = torch.empty((n, nv), dtype=torch.int8, device="cuda")
    X4 = torch.empty((n, nv // 2), dtype=torch.uint8, device="cuda")
    with _native(n, stream=stream.cuda_stream, max_multiplicity=1) as a, \
            _native(n, dtype=native.DTYPE_E2M1, stream=stream.cuda_stream, max_multiplicity=1) as b:
        a.synthDenseDevice(SEED, 0, nv, 0, X8.data_ptr(), nv)
        b.synthDenseDevice(SEED, 0, nv, 0, X4.data_ptr(), nv)
        a.accumulateDenseDevice(X8.data_ptr(), nv, nv)
        b.accumulateDenseDevice(X4.data_ptr(), nv, nv)
        a.finalizeGram()
        b.finalizeGram()
        assert np.array_equal(a.getGram(), b.getGram())


# ---------------------------------------------------------------------------------------------------------------
# panel layout (the resident-cohort layout of vpca_accumulate_panels)
# ---------------------------------------------------------------------------------------------------------------
def _to_panels(X, P):
    """(n, nv) row-major -> flat panel layout, zero padded to whole panels."""
    n, nv = X.shape
    npan = (nv + P - 1) // P
    out = np.zeros((npan, n, P), X.dtype)
    for p in range(npan):
        w = min(P, nv - p * P)
        out[p, :, :w] = X[:, p * P:p * P + w]
    return out.reshape(-1)


@pytest.mark.parametrize("dtype_name", ["i8", "e2m1", "bf16"])
def test_synth_and_gram_panel_layout(oracle, monkeypatch, dtype_name):
    import torch
    from spark_examples_b200 import native
    _set_env(monkeypatch, 2)
    dt = {"i8": native.DTYPE_I8, "e2m1": native.DTYPE_E2M1, "bf16": native.DTYPE_BF16}[dtype_name]
    n, v0, nv, P = 515, 256, 3000, 1024                       # 3 panels, the last one partial
    Xr = oracle.c_synth_dense(SEED, n, v0, nv, mode=1)
    want = oracle.np_similarity_dense(Xr)
    stream = torch.cuda.Stream()
    torch.cuda.set_stream(stream)
    with _native(n, dtype=dt, stream=stream.cuda_stream) as nat:
        buf = torch.full((nat.panelBytes(nv, P),), 0x5A, dtype=torch.uint8, device="cuda")
        nat.synthPanelsDevice(SEED, v0, nv, 1, buf.data_ptr(), P)
        stream.synchronize()
        got = buf.cpu().numpy()
        if dtype_name == "i8":
            assert np.array_equal(got.view(np.int8), _to_panels(Xr, P))
        elif dtype_name == "e2m1":
            codes = _to_panels((2 * Xr).astype(np.uint8), P)
            assert np.array_equal(got, (codes[0::2] | (codes[1::2] << 4)).astype(np.uint8))
        else:
            bits = np.array([0x0000, 0x3F80, 0x4000], np.uint16)[_to_panels(Xr.astype(np.int64), P)]
            assert np.array_equal(got.view(np.uint16), bits)
        nat.accumulatePanels(buf.data_ptr(), nv, P)
        nat.finalizeGram()
        assert np.array_equal(nat.getGram(), want)


def test_calls_path_spans_several_panels_and_chunks(oracle, monkeypatch):
    """CSR input larger than one staging chunk and one panel (chunk_variants forced small)."""
    monkeypatch.setenv("VPCA_PANEL", "512")
    n, nv = 300, 5000
    off, idx = oracle.c_synth_calls(SEED, n, 0, nv)
    want = oracle.c_similarity(n, off, idx, 2)
    with _native(n, chunk_variants=1536, chunk_nnz=200_000) as nat:
        nat.accumulateCalls(-1, off, idx)
        nat.finalizeGram()
        assert np.array_equal(nat.getGram(), want)
        tile = nat.encodeCalls(off[:1301], idx[:off[1300]])
    X = np.zeros((n, 1300), np.int8)
    for v in range(1300):
        X[idx[off[v]:off[v + 1]], v] = 1
    assert np.array_equal(tile, X)


def test_calls_u16_wire_format(oracle):
    n, nv = 640, 3000
    off, idx = oracle.c_synth_calls(SEED, n, 0, nv)
    want = oracle.c_similarity(n, off, idx, 2)
    with _native(n) as nat:
        nat.accumulateCalls16(0, off, idx.astype(np.uint16))
        nat.commit(0)
        nat.finalizeGram()
        assert np.array_equal(nat.getGram(), want)
        st = nat.stats()
    assert st["h2d_bytes"] == (len(off)) * 8 + len(idx) * 2
    with _native(n) as nat:
        with pytest.raises(IndexError):
            nat.accumulateCalls16(-1, np.array([0, 1], np.int64), np.array([n], np.uint16))


@pytest.mark.parametrize("dtype_name", ["i8", "bf16"])
def test_gram_large_n_stream_k_vs_torch(oracle, dtype_name):
    """N = 9000 (hundreds of tiles, far more than CTA pairs): the double-buffered stream-K path, panel layout.
    Checker: fp32 torch matmul on the same device (exact: every count < 2^24)."""
    import torch
    from spark_examples_b200 import native
    dt = {"i8": native.DTYPE_I8, "bf16": native.DTYPE_BF16}[dtype_name]
    n, nv, P = 9000, 6000, 2048
    stream = torch.cuda.Stream()
    torch.cuda.set_stream(stream)
    with _native(n, dtype=dt, stream=stream.cuda_stream, max_multiplicity=1) as nat:
        buf = torch.empty(nat.panelBytes(nv, P), dtype=torch.uint8, device="cuda")
        nat.synthPanelsDevice(SEED, 0, nv, 0, buf.data_ptr(), P)
        nat.accumulatePanels(buf.data_ptr(), nv, P)
        nat.finalizeGram()
        S = torch.from_numpy(nat.getGram()).cuda()
        st = nat.stats()
    assert st["gram_resident"] == 0
    npan = (nv + P - 1) // P
    view = buf.view(torch.int8 if dtype_name == "i8" else torch.bfloat16).view(npan, n, P)
    Xf = torch.cat([view[p].to(torch.float32) for p in range(npan)], dim=1)[:, :nv]
    want = (Xf @ Xf.t()).to(torch.int32)
    assert torch.equal(S, want)


def test_gram_biobank_scale_n(oracle):
    """N = 70 000 samples (S = 19.6 GB int32 resident in HBM, > 65 535 so beyond what the reference's eigen step takes):
    64-bit indexing of the tiled Gram, spot-checked on random rows against an fp32 matmul; computePca refuses like MLlib."""
    import torch
    from spark_examples_b200 import native
    n, nv, P = 70_000, 4096, 4096
    free, _ = torch.cuda.mem_get_info()
    if free < 30 * 2 ** 30:
        pytest.skip("needs 30 GB of free HBM")
    stream = torch.cuda.Stream()
    torch.cuda.set_stream(stream)
    S = torch.zeros((n, n), dtype=torch.int32, device="cuda")
    with _native(n, stream=stream.cuda_stream, d_gram=S.data_ptr(), max_multiplicity=1) as nat:
        X = torch.empty(nat.panelBytes(nv, P), dtype=torch.uint8, device="cuda")
        nat.synthPanelsDevice(SEED, 0, nv, 0, X.data_ptr(), P)
        nat.accumulatePanels(X.data_ptr(), nv, P)
        nat.finalizeGram()
        stream.synchronize()
        Xf = X.view(torch.int8).view(n, P).to(torch.float16)
        rows = torch.tensor([0, 1, 255, 256, 2503, 32767, 32768, 46340, 46341, 65535, 65536, n - 2, n - 1], device="cuda")
        want = (Xf[rows].to(torch.float32) @ Xf.to(torch.float32).t()).to(torch.int32)
        assert torch.equal(S[rows], want)
        assert torch.equal(S[:, rows].t().contiguous(), want)
        with pytest.raises(native.VpcaError) as ei:
            nat.computePca(2)
        assert ei.value.code == native.VPCA_ERR_UNSUPPORTED


@pytest.mark.parametrize("dtype_name", ["i8", "e2m1", "bf16"])
def test_bitmap_rows_wire_format(oracle, monkeypatch, dtype_name):
    """SURVEY 8f-1: one N-bit row per variant instead of an index list; ragged N (not a multiple of 8 or 32), nv not a
    multiple of 32, garbage bits after sample N-1, several staging chunks."""
    from spark_examples_b200 import native
    monkeypatch.setenv("VPCA_PANEL", "256")
    dt = {"i8": native.DTYPE_I8, "e2m1": native.DTYPE_E2M1, "bf16": native.DTYPE_BF16}[dtype_name]
    n, nv = 333, 1111
    X = oracle.c_synth_dense(SEED, n, 0, nv)                      # (n, nv) binary
    stride = (n + 7) // 8 + 3                                     # padded rows
    bits = np.zeros((nv, stride), np.uint8)
    packed = np.packbits(X.T.astype(np.uint8), axis=1, bitorder="little")
    bits[:, : packed.shape[1]] = packed
    bits[:, (n - 1) // 8] |= np.uint8((0xFF << ((n - 1) % 8 + 1)) & 0xFF)   # garbage after the last sample
    bits[:, (n + 7) // 8:] = 0xFF
    want = oracle.np_similarity_dense(X)
    with _native(n, dtype=dt, chunk_variants=512) as nat:
        nat.accumulateBits(0, bits[:700])
        nat.accumulateBits(0, bits[700:])
        nat.commit(0)
        nat.finalizeGram()
        assert np.array_equal(nat.getGram(), want)
        assert nat.stats()["h2d_bytes"] == nv * stride
