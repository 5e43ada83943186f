"""The Gram and the centring at the edges of their number ranges, against exact integer references.

Every other Gram test feeds cells in {0, 1, 2}, so its counts stay far below the limits the library promises:

  int8  cells up to 127, counts up to 2^31 - 1: check_overflow (vpca.cu) admits variants x max_multiplicity^2 <= 2^31 - 1
  bf16  cells up to 45, accumulated in FP32 by wgmma: launch_gram splits a call so that one launch folds at most
        floor(2^24 / max_multiplicity^2) variants (floored to whole panels), below which FP32 holds every count exactly
  e2m1  packed cells 0..2 through the same sub-launch loop, at half-byte offsets
  the encode kernels' multiplicity flag (VPCA_ERR_OVERFLOW) and the int32 guard, with their bookkeeping of staged
        partitions (inflight_variants)
  matrixMean of the centring, whose total sum S passes 2^53 in whole-genome cohorts

Expected Grams are exact integer arithmetic: numpy int64, the oracle's loop, or FP64 matmuls on the device over column
chunks (every partial sum of non-negative integer products is at most the final count, < 2^31, so FP64 is exact) summed
in int64.  Last, every eigensolver path must be exactly scale invariant: the same cells times 2^5, or the Gram times
2^16, give bit-identical vectors and eigenvalues exactly 4^5 or 2^16 times as large."""
from contextlib import contextmanager

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

SEED = 20261016
INT32_MAX = 2 ** 31 - 1
P = 8192                       # variants per panel (the library's default staging panel)


def _native(n, **kw):
    from spark_examples_b200 import native
    return native.NativePca(n, **kw)


def _need_free_hbm(gib):
    import torch
    free, _ = torch.cuda.mem_get_info()
    if free < gib * 2 ** 30:
        pytest.skip(f"needs {gib} GB of free HBM")


def _release():
    import torch
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


@contextmanager
def _raises(code):
    from spark_examples_b200 import native
    with pytest.raises(native.VpcaError) as ei:
        yield ei
    assert ei.value.code == code, ei.value


def _gram_exact(X, chunk=1 << 16):
    """exact X X^T (int64, numpy) of non-negative integer cells X (n, nv) on the device, by FP64 column chunks"""
    import torch
    n, nv = X.shape
    S = torch.zeros((n, n), dtype=torch.int64, device=X.device)
    for c0 in range(0, nv, chunk):
        Xc = X[:, c0:c0 + chunk].to(torch.float64)
        S += (Xc @ Xc.t()).to(torch.int64)
    return S.cpu().numpy()


def _panels(X, panel=P):
    """(n, nv) device cells -> the panel layout of vpca_accumulate_panels as flat bytes, zero cells after nv"""
    import torch
    n, nv = X.shape
    npan = -(-nv // panel)
    out = torch.zeros((npan, n, panel), dtype=X.dtype, device=X.device)
    for p in range(npan):
        w = min(panel, nv - p * panel)
        out[p, :, :w] = X[:, p * panel:p * panel + w]
    return out.view(-1).view(torch.uint8)


def _finalized_gram(nat):
    nat.finalizeGram()
    return nat.getGram()


# ------------------------------------------------------------------------------------------ 1. int8 at the int32 limit
I8_MAX_VARIANTS = INT32_MAX // 127 ** 2          # 133 144: the most the guard admits at max_multiplicity 127
I8_FULL_ROWS = [0, 1, 130, 319]                  # cells of 127 everywhere, in each of the three (ragged) 128-row blocks


@pytest.fixture(scope="module")
def int8_limit_cohort():
    import torch
    rng = np.random.default_rng(SEED)
    n, nv = 320, I8_MAX_VARIANTS
    X = rng.integers(0, 128, (n, nv), dtype=np.int8)
    X[I8_FULL_ROWS] = 127
    want = _gram_exact(torch.from_numpy(X).cuda())
    _release()
    return X, want


@pytest.mark.parametrize("red64", [1, 0])
@pytest.mark.parametrize("cta_group", [1, 2])
def test_int8_counts_at_the_int32_limit(monkeypatch, int8_limit_cohort, cta_group, red64):
    """max_multiplicity 127, N = 320, 133 144 variants: the all-127 pairs end at 2 147 479 576, 4072 below 2^31.
    Host staging in several chunks, a row-major device tile and the panel layout, both CTA groups, both flushes, all bit
    exact; one variant more is refused and leaves the Gram as it was."""
    import torch
    from spark_examples_b200 import native
    monkeypatch.setenv("VPCA_CTA_GROUP", str(cta_group))
    monkeypatch.setenv("VPCA_RED64", str(red64))
    X, want = int8_limit_cohort
    n, nv = X.shape
    assert want[0, 1] == want[130, 319] == 127 ** 2 * nv == 2_147_479_576
    assert want.max() <= INT32_MAX
    ld = -(-nv // 16) * 16                                       # 16-byte row pitch of a device tile
    tile = torch.zeros((n, ld), dtype=torch.int8, device="cuda")
    tile[:, :nv] = torch.from_numpy(X).cuda()
    panels = _panels(tile[:, :nv])
    torch.cuda.synchronize()
    feeds = {
        "host": (lambda nat: nat.accumulateDense(X), lambda nat: nat.accumulateDense(X[:, :1])),
        "device": (lambda nat: nat.accumulateDenseDevice(tile.data_ptr(), nv, ld),
                   lambda nat: nat.accumulateDenseDevice(tile.data_ptr(), 1, ld)),
        "panels": (lambda nat: nat.accumulatePanels(panels.data_ptr(), nv, P),
                   lambda nat: nat.accumulatePanels(panels.data_ptr(), 1, P)),
    }
    for name, (feed, one_more) in feeds.items():
        with _native(n, max_multiplicity=127, chunk_variants=32768) as nat:
            feed(nat)
            with _raises(native.VPCA_ERR_OVERFLOW):
                one_more(nat)
            assert nat.variantCount() == nv
            S = _finalized_gram(nat)
            st = nat.stats()
        assert st["gram_cta_group"] == cta_group, name
        if name == "host":
            assert st["gram_launches"] == -(-nv // 32768)               # one launch per staging chunk
        assert np.array_equal(S, want), name
    del tile, panels
    _release()


# ----------------------------------------------------------------------------------- 2. bf16 at the FP32 bound of a launch
def _fp32_edge_cells(n, nv, mm, per_launch, seed):
    """(n, nv) int8 cells on the device, random in 0..mm, with rows whose counts over the first launch sit at its edge:
    row 0 is mm everywhere (its diagonal reaches exactly 2^24 there); rows 1, 2 are mm in the first launch except at
    scattered places where their product is 1 (an odd number of them) or 2, so their count is odd and just below 2^24;
    rows 3, 4 are mm there except at one place (mm = 2: product 1, count 2^24 - 3; mm = 1: product 0, count 2^24 - 1,
    the largest odd count each allows).  Returns the cells and the exact Gram of their first rows over the first launch."""
    import torch
    g = torch.Generator(device="cuda")
    g.manual_seed(seed)
    X = torch.randint(0, mm + 1, (n, nv), dtype=torch.int8, device="cuda", generator=g)
    rng = np.random.default_rng(seed)
    X[0] = mm
    X[1:5, :per_launch] = mm
    pos = torch.from_numpy(rng.choice(per_launch, 1777 + 1, replace=False)).cuda()
    ones, mixed, single = pos[:777], pos[777:1777], pos[1777:]
    if mm > 1:
        X[1, ones] = 1
        X[2, ones] = 1
        X[1, mixed] = 1
        X[3, single] = 1
        X[4, single] = 1
    else:
        X[2, ones] = 0
        X[4, single] = 0
    first = _gram_exact(X[:8, :per_launch])
    return X, first


def _bf16_panels(X):
    import torch
    Xb = X.to(torch.bfloat16)
    out = _panels(Xb)
    del Xb
    return out


@pytest.mark.parametrize("mm,n", [(2, 320), (1, 64)])
def test_bf16_at_the_fp32_bound_of_one_launch(mm, n):
    """bf16 cells, panels of 8192: a call of 2^24 / mm^2 variants (+ two panels + 300) is split into a full launch whose
    counts reach exactly 2^24 (odd ones just below) and a ragged one.  At these N the stream-K schedule spreads each
    tile's k-blocks over many workers, so the counts near 2^24 are formed by the int32 flushes, not inside one FP32
    accumulator (test_bf16_whole_launch_in_one_fp32_accumulator covers that): this pins the split, the sub-launch
    offsets and the flush.  Against the exact Gram and against an int8 context on the same cells."""
    import torch
    from spark_examples_b200 import native
    per_launch = 2 ** 24 // mm ** 2
    nv = per_launch + 2 * P + 300
    _need_free_hbm(int(6 * n * nv / 2 ** 30) + 4)    # the cells, their bf16 copy and both panel layouts
    X, first = _fp32_edge_cells(n, nv, mm, per_launch, SEED + mm)
    assert first[0, 0] == 2 ** 24
    assert first[1, 2] % 2 == 1 and 2 ** 24 - 5000 < first[1, 2] < 2 ** 24
    assert first[3, 4] == 2 ** 24 - (3 if mm == 2 else 1)
    want = _gram_exact(X)
    p16 = _bf16_panels(X)
    p8 = _panels(X)
    torch.cuda.synchronize()
    with _native(n, dtype=native.DTYPE_BF16, max_multiplicity=mm) as b, _native(n, max_multiplicity=mm) as a:
        b.accumulatePanels(p16.data_ptr(), nv, P)
        a.accumulatePanels(p8.data_ptr(), nv, P)
        S16, S8 = _finalized_gram(b), _finalized_gram(a)
        launches = b.stats()["gram_launches"]
    assert np.array_equal(S16, want)
    assert np.array_equal(S8, want)
    assert launches == 2
    del X, p16, p8
    _release()


def _whole_tile_n(workers, kbw, rows=6):
    """the smallest N >= 2504 at which the equal split of the Gram kernel's resident schedule (VPCA_CTA_GROUP=1: one
    worker per SM) hands the tiles that hold the cells among samples [0, rows) whole to one worker each, for every
    k-block of the window"""
    from spark_examples_b200 import native
    for n in range(2504, 8193, 8):
        tiles = native.debugTiles(n, 1, exact=False)          # rowA0, rowA1, rowB, n_eff, ...
        try:
            pieces = native.debugPlan(tiles, workers, kbw)    # worker, tile, kb_lo, kb_hi, ...
        except native.VpcaError:
            break                                             # past the resident schedule
        mine = np.flatnonzero((tiles[:, 0] == 0) & (tiles[:, 2] < rows))
        held = pieces[np.isin(pieces[:, 1], mine)]
        if len(mine) and len(held) == len(mine) and ((held[:, 2] == 0) & (held[:, 3] == kbw)).all():
            return n
    pytest.skip(f"the resident schedule of {workers} workers never hands the first tile whole to one worker")


@pytest.mark.parametrize("mm", [2, 45])
def test_bf16_whole_launch_in_one_fp32_accumulator(monkeypatch, mm):
    """The FP32 premise itself.  At N = 320 the resident schedule splits each tile's k-blocks over many workers, so no
    register accumulator holds more than a few percent of a launch's count.  Here N is chosen so that every tile is one
    worker's, whole window after whole window: each cell's count over a launch is summed in one FP32 register and
    flushed once.  mm = 2: launches of 4 194 304 variants, in which a pair counts exactly 2^24 and odd pairs 2^24 - 2331
    and 2^24 - 3; mm = 45: one-panel launches of 8192 variants, counts up to 16 588 800 and odd ones just below.  The
    schedule is pinned to its equal split (VPCA_ADAPTIVE=0) so that it is the one the host-side planner reports."""
    import torch
    from spark_examples_b200 import native
    monkeypatch.setenv("VPCA_CTA_GROUP", "1")
    monkeypatch.setenv("VPCA_ADAPTIVE", "0")
    monkeypatch.delenv("VPCA_KB_WINDOW", raising=False)
    monkeypatch.delenv("VPCA_EXACT_COVER", raising=False)
    kbw = P // 64                                        # one L2 window per panel: 128 k-blocks of 64 bf16 cells
    n = _whole_tile_n(torch.cuda.get_device_properties(0).multi_processor_count, kbw)
    L = 2 ** 24 // mm ** 2 // P * P                      # variants of one launch
    nv = L + (P + 300 if mm == 2 else 2 * P + 300)
    npan, lp = -(-nv // P), L // P
    _need_free_hbm(int(3 * npan * n * P / 2 ** 30) + 4)  # int8 cells and their bf16 copy
    g = torch.Generator(device="cuda")
    g.manual_seed(SEED + mm)
    Xp = torch.randint(0, mm + 1, (npan, n, P), dtype=torch.int8, device="cuda", generator=g)   # panel layout
    Xp[:, 0, :] = mm
    Xp[:lp, 1:6, :] = mm
    pos = np.random.default_rng(SEED + mm).choice(L, 778, replace=False)
    for rows, at in (((2, 3), pos[:777]), ((4, 5), pos[777:])):
        pi, ci = torch.from_numpy(at // P).cuda(), torch.from_numpy(at % P).cuda()
        for r in rows:
            Xp[pi, r, ci] = mm - 1
    Xp[-1, :, nv - (npan - 1) * P:] = 0
    head = Xp[:lp, :6, :].permute(1, 0, 2).reshape(6, L).to(torch.float64)
    first = (head @ head.t()).to(torch.int64).cpu().numpy()
    del head
    full = mm * mm * L
    assert first[0, 1] == full and (mm != 2 or full == 2 ** 24)
    assert first[2, 3] == full - (2 * mm - 1) * 777 and first[2, 3] % 2 == 1
    assert first[4, 5] == full - (2 * mm - 1) and first[4, 5] % 2 == 1
    want = torch.zeros((n, n), dtype=torch.int64, device="cuda")
    for p in range(npan):
        Xc = Xp[p].to(torch.float64)
        want += (Xc @ Xc.t()).to(torch.int64)
    want = want.cpu().numpy()
    p16 = Xp.to(torch.bfloat16)
    del Xp
    torch.cuda.synchronize()
    with _native(n, dtype=native.DTYPE_BF16, max_multiplicity=mm) as nat:
        nat.accumulatePanels(p16.data_ptr(), nv, P)
        S = _finalized_gram(nat)
        st = nat.stats()
    assert np.array_equal(S, want)
    assert st["gram_resident"] == 1 and st["gram_cta_group"] == 1, st
    assert st["gram_launches"] == -(-nv // L)
    del p16
    _release()


# ---------------------------------------------------------------------------------------- 3. bf16 at multiplicity 45
def test_bf16_at_multiplicity_45():
    """bf16 cells random in 0..45, two rows 45 everywhere, 1 060 485 variants (the guard's maximum): the all-45 pair ends
    at 2 147 482 125 and each launch is one panel whose count reaches 16 588 800 (at N = 320 summed over several workers'
    FP32 accumulators and the int32 flush, see above).  The panel layout and the host staging
    path (sub-launches inside each staging chunk) are exact; one variant more is refused, and so are panels of 16 384,
    wider than the exact FP32 window; neither refusal touches the Gram."""
    import torch
    from spark_examples_b200 import native
    n, mm = 320, 45
    nv = INT32_MAX // mm ** 2
    _need_free_hbm(6)
    g = torch.Generator(device="cuda")
    g.manual_seed(SEED)
    X = torch.randint(0, mm + 1, (n, nv), dtype=torch.int8, device="cuda", generator=g)
    X[[0, 200]] = mm
    want = _gram_exact(X)
    assert want[0, 200] == mm ** 2 * nv == 2_147_482_125 and want.max() <= INT32_MAX
    Xb = X.to(torch.bfloat16)
    host = Xb.view(torch.int16).cpu().numpy().view(np.uint16)
    panels = _panels(Xb)
    del X, Xb
    torch.cuda.synchronize()
    with _native(n, dtype=native.DTYPE_BF16, max_multiplicity=mm) as nat:
        nat.accumulatePanels(panels.data_ptr(), nv, P)
        with _raises(native.VPCA_ERR_OVERFLOW):
            nat.accumulatePanels(panels.data_ptr(), 1, P)
        assert nat.variantCount() == nv
        assert np.array_equal(_finalized_gram(nat), want)
        assert nat.stats()["gram_launches"] == -(-nv // P)
    with _native(n, dtype=native.DTYPE_BF16, max_multiplicity=mm) as nat:
        nat.accumulateDense(host)
        with _raises(native.VPCA_ERR_OVERFLOW):
            nat.accumulateDense(host[:, :1])
        assert nat.variantCount() == nv
        assert np.array_equal(_finalized_gram(nat), want)
    with _native(n, dtype=native.DTYPE_BF16, max_multiplicity=mm) as nat:
        with _raises(native.VPCA_ERR_UNSUPPORTED):
            nat.accumulatePanels(panels.data_ptr(), 2 * P, 2 * P)
        assert nat.variantCount() == 0
        assert not _finalized_gram(nat).any()
    del panels
    _release()


# ------------------------------------------------------------------------------------------ 4. e2m1 across sub-launches
def test_e2m1_across_sub_launches():
    """Packed e2m1 dosage cells (0/1/2) of 4 194 304 + 8192 + 128 variants at max_multiplicity 2: two launches, the second
    starting 512 panels in and ending in a partial panel.  Equal to the int8 Gram of the generator's same cells, whose
    diagonal is sum_v x_sv^2, and to the exact Gram."""
    import torch
    from spark_examples_b200 import native
    n = 128
    nv = 2 ** 24 // 4 + P + 128
    _need_free_hbm(4)
    npan = -(-nv // P)
    with _native(n, dtype=native.DTYPE_E2M1) as e, _native(n) as a:
        b4 = torch.empty(e.panelBytes(nv, P), dtype=torch.uint8, device="cuda")
        b8 = torch.empty(a.panelBytes(nv, P), dtype=torch.uint8, device="cuda")
        torch.cuda.synchronize()
        e.synthPanelsDevice(SEED, 0, nv, 1, b4.data_ptr(), P)
        a.synthPanelsDevice(SEED, 0, nv, 1, b8.data_ptr(), P)
        e.accumulatePanels(b4.data_ptr(), nv, P)
        a.accumulatePanels(b8.data_ptr(), nv, P)
        S4, S8 = _finalized_gram(e), _finalized_gram(a)
        assert e.stats()["gram_launches"] == 2
    X = b8.view(torch.int8).view(npan, n, P).permute(1, 0, 2).reshape(n, npan * P)[:, :nv]
    assert int(X.max()) == 2
    diag = sum((X[:, c:c + (1 << 20)].to(torch.int32) ** 2).sum(dim=1, dtype=torch.int64) for c in range(0, nv, 1 << 20))
    assert np.array_equal(S4, S8)
    assert np.array_equal(np.diag(S4), diag.cpu().numpy())
    assert np.array_equal(S4, _gram_exact(X))
    del X, b4, b8
    _release()


# ------------------------------------------------------------------ 5. multiplicity up to each type's limit, every wire
def _csr(rows):
    off = np.zeros(len(rows) + 1, np.int64)
    off[1:] = np.cumsum([len(r) for r in rows])
    idx = np.asarray([s for r in rows for s in r], np.int32)
    return off, idx


def _multiplicity_rows(n, nv, m, seed, over=False):
    """nv rows split into a left and a right half (the two datasets of a join): row v lists sample v % n exactly m
    times in all (m // 2 on the left), plus a few other samples once; over=True: row 3 lists it once more (on the left,
    so with m = 1 it is present once in each dataset)"""
    rng = np.random.default_rng(seed)
    left, right = [], []
    for v in range(nv):
        hot = v % n
        others = [int(s) for s in rng.choice(n, 6, replace=False) if s != hot]
        a = m // 2 + (1 if over and v == 3 else 0)
        left.append([hot] * a + others[:3])
        right.append([hot] * (m - m // 2) + others[3:])
    return left, right


def _dense_gram(n, rows):
    X = np.zeros((n, len(rows)), np.int64)
    for v, r in enumerate(rows):
        np.add.at(X[:, v], r, 1)
    return X @ X.T


def _feed(nat, wire, pid, left, right):
    from spark_examples_b200 import native
    if wire == "join":
        off, idx = _csr(left + right)
        keys = [b"variant-%d" % v for v in range(len(left))] * 2
        nat.joinRows(native.JOIN, keys, off, idx, n_left=len(left))
        nat.accumulateJoined(pid)
        return
    off, idx = _csr([a + b for a, b in zip(left, right)])
    if wire == "calls":
        nat.accumulateCalls(pid, off, idx)
    else:
        nat.accumulateCalls16(pid, off, idx.astype(np.uint16))


# (dtype, max_multiplicity, m = the largest multiplicity the encoder takes at that setting)
MULTIPLICITY_CASES = [("i8", 1, 1), ("i8", 2, 2), ("i8", 127, 127), ("i8", 200, 127), ("bf16", 45, 45),
                      ("e2m1", 1, 1), ("e2m1", 2, 2)]


@pytest.mark.parametrize("wire", ["calls", "calls16", "join"])
@pytest.mark.parametrize("dtype_name,max_mult,m", MULTIPLICITY_CASES,
                         ids=[f"{d}-max{mx}-m{m}" for d, mx, m in MULTIPLICITY_CASES])
def test_multiplicity_up_to_each_cell_type_limit(dtype_name, max_mult, m, wire):
    """A sample listed m times in a row (through a join: present in both datasets, counted twice) is exact up to the
    cell type's limit (int8 127, also when max_multiplicity asks for more; bf16 45; e2m1 2).  Listed m + 1 times the call
    fails with VPCA_ERR_OVERFLOW: a staged partition is poisoned while another still commits exactly, and a direct call
    reports that the Gram needs a reset, after which the context accumulates exactly again."""
    from spark_examples_b200 import native
    dt = {"i8": native.DTYPE_I8, "bf16": native.DTYPE_BF16, "e2m1": native.DTYPE_E2M1}[dtype_name]
    n, nv = 100, 256
    left, right = _multiplicity_rows(n, nv, m, SEED + m)
    rows = [a + b for a, b in zip(left, right)]
    assert max(max(np.bincount(r)) for r in rows) == m
    bad = _multiplicity_rows(n, nv, m, SEED + m, over=True)
    want = _dense_gram(n, rows)
    assert np.diag(want).min() >= 2 * m * m           # every sample is the repeated one in at least two rows
    with _native(n, dtype=dt, max_multiplicity=max_mult) as nat:
        _feed(nat, wire, 0, left, right)
        with _raises(native.VPCA_ERR_OVERFLOW):
            _feed(nat, wire, 1, *bad)
        nat.commit(1)                     # the poisoned partition left nothing to commit
        nat.commit(0)
        assert nat.variantCount() == nv
        assert np.array_equal(_finalized_gram(nat), want)
    with _native(n, dtype=dt, max_multiplicity=max_mult) as nat:
        with _raises(native.VPCA_ERR_OVERFLOW) as ei:
            _feed(nat, wire, -1, *bad)
        assert "vpca_reset" in str(ei.value)
        nat.reset()
        _feed(nat, wire, -1, left, right)
        assert np.array_equal(_finalized_gram(nat), want)


# -------------------------------------------------------------------- 6. overflow accounting across staged partitions
def test_overflow_accounting_across_staged_partitions(oracle):
    """max_multiplicity 127: three staged partitions of 133 144 light rows in all fill the int32 bound, so a fourth
    partition, a direct call and one row more on a staged partition are all refused (without poisoning it); an abort
    gives its partition's room back exactly, the retry fits, and after the commits the Gram is exact."""
    from spark_examples_b200 import native
    n, nv = 64, I8_MAX_VARIANTS
    rng = np.random.default_rng(SEED)
    counts = rng.integers(1, 4, nv)
    off = np.zeros(nv + 1, np.int64)
    off[1:] = np.cumsum(counts)
    idx = rng.integers(0, n, int(off[-1])).astype(np.int32)
    want = oracle.c_similarity(n, off, idx, 1)

    def rows(a, b):
        return off[a:b + 1] - off[a], idx[off[a]:off[b]]

    parts = [(0, 60_000), (60_000, 110_000), (110_000, nv)]
    with _native(n, max_multiplicity=127, partitions_in_flight=4) as nat:
        for pid, (a, b) in enumerate(parts):
            nat.accumulateCalls(pid, *rows(a, b))
        for pid in (3, -1, 0):
            with _raises(native.VPCA_ERR_OVERFLOW):
                nat.accumulateCalls(pid, *rows(0, 1))
        nat.abort(1)
        with _raises(native.VPCA_ERR_OVERFLOW):
            nat.accumulateCalls(1, *rows(60_000, 110_001))
        nat.accumulateCalls(1, *rows(60_000, 110_000))
        with _raises(native.VPCA_ERR_OVERFLOW):
            nat.accumulateCalls(3, *rows(0, 1))
        for pid in range(3):
            nat.commit(pid)
        with _raises(native.VPCA_ERR_OVERFLOW):
            nat.accumulateCalls(-1, *rows(0, 1))
        assert nat.variantCount() == nv
        assert np.array_equal(_finalized_gram(nat), want)


# ----------------------------------------------------------------------------------------------- 7. centring past 2^53
def _centred(S, total):
    """C of VariantsPca.scala:199-223 with rowSums exact and matrixMean = RN(RN(float(total) / N) / N), float(total) the
    correctly rounded sum of S; element-wise the left-to-right formula of center_kernel"""
    n = S.shape[0]
    rm = S.astype(np.int64).sum(axis=1).astype(np.float64) / n
    mm = float(total) / n / n
    return ((S.astype(np.float64) - rm[:, None]) - rm[None, :]) + mm


def _block_tree_sum(values, threads=1024):
    """double sum in the order of a one-block reduction: strided sums per thread, then xor butterflies over the 32
    lanes of each warp and over the 32 warps"""
    acc = np.zeros(threads)
    for i in range(0, len(values), threads):
        acc = acc + values[i:i + threads]
    lanes = np.arange(32)
    for _ in range(2):
        acc = acc.reshape(-1, 32)
        for o in (16, 8, 4, 2, 1):
            acc = acc + acc[:, lanes ^ o]
        acc = acc[:, 0]
    return float(acc[0])


def test_centring_past_2_53(oracle):
    """N = 4096 with similarity counts in [2^30, 2^31): sum S is about 3 x 2^53, where a double sum of the row sums
    depends on its order -- for this S both the reference's sequential sum and a block-reduction tree miss the correctly
    rounded total.  The centred matrix uses the exact total rounded once.  Below 2^53 it stays the oracle's, bit for
    bit."""
    n = 4096
    rng = np.random.default_rng(SEED + 1)
    A = np.triu(rng.integers(2 ** 30, INT32_MAX, (n, n), dtype=np.int64))
    S = (A + np.triu(A, 1).T).astype(np.int32)
    assert np.array_equal(S, S.T)
    rowsums = S.astype(np.int64).sum(axis=1)
    total = int(rowsums.sum())
    assert total >= 2 ** 53
    sequential = 0.0
    for r in rowsums.tolist():           # the reference's rowSums.reduce(_ + _)
        sequential += float(r)
    assert sequential != float(total)
    assert _block_tree_sum(rowsums.astype(np.float64)) != float(total)
    small = (np.triu(rng.integers(0, 2 ** 20, (n, n), dtype=np.int64)))
    small = (small + np.triu(small, 1).T).astype(np.int32)
    assert int(small.astype(np.int64).sum()) < 2 ** 53
    with _native(n) as nat:
        nat.setGram(S)
        C = nat.getCentered()
        nat.setGram(small)
        C_small = nat.getCentered()
    assert np.array_equal(C, _centred(S, total))
    want_small, _, _ = oracle.c_center(small)
    assert np.array_equal(C_small, want_small)
    assert np.array_equal(C_small, _centred(small, int(small.astype(np.int64).sum())))


# --------------------------------------------------------------------------- 8. scale invariance of every eigensolver
SCALE = 32                   # cells 0 / 2^5: the Gram is exactly 4^5 S
GRAM_SHIFT = 16              # setGram(S << 16): entries stay below 2^31 at 4096 variants


def _cells_context(n, buf, nv, mm, k, band=None):
    from eig_ref import P as EP
    nat = _native(n, max_multiplicity=mm, num_pc=k, gram_band=band)
    try:
        nat.accumulatePanels(buf.data_ptr(), nv, EP)
        nat.synchronize()
        nat.finalizeGram()
    except Exception:
        nat.close()
        raise
    return nat


def _set_context(n, S, k):
    nat = _native(n, num_pc=k)
    nat.setGram(S)
    return nat


def _assert_scaled(base, scaled, factor, what):
    assert np.array_equal(scaled.vecs, base.vecs), what
    assert np.array_equal(scaled.evals, base.evals * factor), what
    assert scaled.nz == base.nz, what


@pytest.mark.parametrize("path,env", [("direct-fused", {"VPCA_EIG": "direct"}),
                                      ("direct-two-kernels", {"VPCA_EIG": "direct", "VPCA_EIG_TWO_KERNELS": "1"}),
                                      ("persistent-lanczos", {}),
                                      ("one-band-lanczos", {"VPCA_LZ_PERSIST": "0"}),
                                      ("bands", None)])
def test_eigensolver_scale_invariance(path, env):
    """The same cohort's cells times 2^5 (int8 cells 0/32, max_multiplicity 32) and its Gram times 2^16 (setGram) give
    bit-identical vectors and eigenvalues exactly 4^5 and 2^16 times as large on every solver path, and each solve
    passes the FP64 reference."""
    import torch
    from eig_ref import (Reference, assert_direct, assert_one_band, assert_persistent, check_pairs, close_all,
                         compute_pca, compute_pca_bands, synth_cells)
    n, nv, k = 1092, 4096, 4
    buf, X = synth_cells(n, nv)
    buf_scaled = buf * SCALE
    ref = Reference(X, k)
    ref_scaled = Reference(X.to(torch.int32) * SCALE, k)
    with _cells_context(n, buf, nv, 1, k) as nat:
        S = nat.getGram()
    assert S.max() < 2 ** (31 - GRAM_SHIFT)
    S_shift = (S.astype(np.int64) << GRAM_SHIFT).astype(np.int32)
    solves = {}
    if path == "bands":
        # the cells through two owner-computes band contexts, the set Grams through one full context (world 1): each
        # scaled solve is compared with the unscaled one of the same band layout, which fixes the order of its sums
        bands = [(0, 500), (500, n - 500)]
        for name, data, mm in (("base", buf, 1), ("cells", buf_scaled, SCALE)):
            ctxs = [_cells_context(n, data, nv, mm, k, band) for band in bands]
            try:
                solves[name] = compute_pca_bands(ctxs, k)
            finally:
                close_all(ctxs)
        for name, G in (("gram_base", S), ("gram", S_shift)):
            with _set_context(n, G, k) as nat:
                solves[name] = compute_pca_bands([nat], k)
        assert all(s.method == 4 for s in solves.values()), solves
    else:
        with _cells_context(n, buf, nv, 1, k) as nat:
            solves["base"] = solves["gram_base"] = compute_pca(nat, k, env)
        with _cells_context(n, buf_scaled, nv, SCALE, k) as nat:
            assert np.array_equal(nat.getGram(), S * SCALE ** 2)
            solves["cells"] = compute_pca(nat, k, env)
        with _set_context(n, S_shift, k) as nat:
            solves["gram"] = compute_pca(nat, k, env)
        ran_as_named = {"direct-fused": lambda s: assert_direct(s, n, fused=True),
                        "direct-two-kernels": lambda s: assert_direct(s, n, fused=False),
                        "persistent-lanczos": assert_persistent, "one-band-lanczos": assert_one_band}[path]
        for s in solves.values():
            ran_as_named(s)
    for name, r in (("base", ref), ("cells", ref_scaled), ("gram_base", ref)):
        check_pairs(r, solves[name].vecs, solves[name].evals, solves[name].nz, k)
    _assert_scaled(solves["base"], solves["cells"], float(SCALE ** 2), f"{path}: cells x {SCALE}")
    _assert_scaled(solves["gram_base"], solves["gram"], float(2 ** GRAM_SHIFT), f"{path}: Gram << {GRAM_SHIFT}")
    del buf, buf_scaled, X
    _release()
