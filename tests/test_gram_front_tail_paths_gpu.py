"""The Gram kernel's front/tail schedule on every path and launch length that reaches it, bit for bit against exact Grams.

When the tiles T of a Gram number more than half the workers W and fewer than all of them (W / 2 < T < W), front worker
t multiplies tile t over the k-blocks [0, s) and the W - T tail workers split T tiles x [s, K), flushing every piece
(Sched in csrc/gram_sm90.cu).  tests/test_gram_tail_schedule_gpu.py covers long panel launches at 2504 samples; this
file drives the schedule through the other ways a run reaches it:

  1. launch length: K = 1 (s = 0: every front worker idle, the tail does the whole launch), 2, 3, one k-block either
     side of a window and several windows, each with a ragged last k-block, so that the window is clamped to K below
     its length; device panels, device row-major tiles (automatic window) and host row-major tiles (staged into panels),
     in every cell type and both CTA groups, at the first and the last N of the range, with s fixed and adapting;
  2. kernel options under front/tail, with s inside a window of a multi-window launch: window pacing
     (VPCA_SYNC_LEAD = 1, 2), one 32-bit red per cell (VPCA_RED64=0, odd and even N), B rows loaded on self-B tiles
     (VPCA_SELF_B=0) and the exact 128-block cover;
  3. staged partitions of 1 .. 700 variants (CSR with int32 and uint16 indices, bitmaps, .bed rows counting A1 and A2
     with missing calls), committed one by one, an abort and a retry, and two host threads feeding one context;
  4. the kinship plane Gram (3N rows) at both edges of its range and at N = 700, with chunk tails of 1 and 128 rows;
  5. the LD plane Gram (3c rows, c the variants rounded up to 32) at both edges of its range, at 100 samples (K = 1),
     2504 and 40 000 (several sample pieces added into one Gram), with the pair list truncated too;
  6. s adapting over long launches interleaved with K = 1 and K = 3 launches, a kinship context, and a fresh context
     that starts from the s the first one left behind.

The ranges come from the device: W is its SM count (single CTAs) or min(SMs / 2, 2-CTA clusters it holds) (CTA pairs),
and T is the tile list of the host replay (debugTiles).  Before its launches every case asserts through the host replay
of the whole launch (debugSchedule) that each launch takes the front/tail schedule, and prints the N (Gram rows), CTA
group, K, window and split point s it tests; with the split point adapting, s is its initial value.  The references
are exact: FP64 X X^T on the device (every count stays far below 2^53), the oracle's similarity for CSR rows,
tests/kinship_ref.py and tests/ld_ref.py.
"""
import functools
import threading

import numpy as np
import pytest

import ld_ref
from kinship_ref import MISSING, dosage_codes, king_pairs, pack_codes

pytestmark = pytest.mark.gpu

SEED = 20261017
DTYPES = ("i8", "bf16", "e2m1")
CELLS_PER_KB = {"i8": 128, "bf16": 64, "e2m1": 128}   # cells per k-block: one 128-byte swizzle atom
PANEL = 8192           # cells per panel row: the device panels here and the library's staging panels (VPCA_PANEL unset)
RAGGED = 5             # cells the last k-block of a launch is short of full
SWITCHES = ("VPCA_KB_WINDOW", "VPCA_PANEL", "VPCA_EXACT_COVER", "VPCA_ADAPTIVE", "VPCA_REBALANCE_GAIN", "VPCA_GRAM_PROF",
            "VPCA_SELF_B", "VPCA_RED64", "VPCA_SYNC_LEAD")


def _native():
    import __graft_entry__ as entry
    from spark_examples_b200 import native
    if not native.library_path().exists():
        entry.build()
    native.load_library()
    return native


def _dtype(dt):
    native = _native()
    return {"i8": native.DTYPE_I8, "bf16": native.DTYPE_BF16, "e2m1": native.DTYPE_E2M1}[dt]


def _env(monkeypatch, cg, **extra):
    """The CTA group and the given switches; every other switch of the Gram kernel at its default."""
    monkeypatch.setenv("VPCA_CTA_GROUP", str(cg))
    for k in SWITCHES:
        monkeypatch.delenv(k, raising=False)
    for k, v in extra.items():
        monkeypatch.setenv(k, str(v))


@pytest.fixture
def say(capsys):
    """Prints a line past pytest's capture, so that the schedule each case tests shows in every run."""
    def _say(line):
        with capsys.disabled():
            print(f"\n    [front/tail] {line}", end="", flush=True)
    return _say


# ---------------------------------------------------------------------------------------------------------------------
# the schedule, from the device's worker count and the host replay
# ---------------------------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def _workers(cg):
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    return sms if cg == 1 else min(sms // 2, _native().maxClusters(0, 2))


def _tiles(rows, cg, exact=False):
    return len(_native().debugTiles(rows, cg, exact))


@functools.lru_cache(maxsize=None)
def _row_range(cg, exact=False):
    """(first, last) Gram row count whose tiles number more than half the workers and fewer than all of them."""
    W = _workers(cg)
    inside = []
    n = 2
    while True:
        T = _tiles(n, cg, exact)
        if T >= W:
            break
        if 2 * T > W:
            inside.append(n)
        n += 1
    assert inside, f"no Gram size puts between {W // 2 + 1} and {W - 1} tiles on {W} workers"
    assert inside == list(range(inside[0], inside[-1] + 1)), "the front/tail range has a hole"
    return inside[0], inside[-1]


def _in_range(rows, cg, exact=False):
    lo, hi = _row_range(cg, exact)
    return lo <= rows <= hi


def _ragged_n(cg, exact=False):
    """2504 (the flagship cohort, N % 16 != 0) where it is in the range, else the first N of the range that is not a
    multiple of 16."""
    lo, hi = _row_range(cg, exact)
    return 2504 if lo <= 2504 <= hi else next(n for n in range(lo, hi + 1) if n % 16)


def _odd_n(cg, exact=False):
    lo, hi = _row_range(cg, exact)
    return 2503 if lo <= 2503 <= hi else next(n for n in range(lo, hi + 1) if n % 2)


def _schedule(say, what, rows, cg, kbw, K, exact=False):
    """Asserts that a launch of K k-blocks over `rows` Gram rows with a window of kbw k-blocks (clamped to K, as the
    launch clamps it) takes the front/tail schedule, prints it and returns its split point s."""
    W, T = _workers(cg), _tiles(rows, cg, exact)
    _, kind, s = _native().debugSchedule(rows, cg, exact, W, min(kbw, K), K)
    assert kind == 2, f"{what}: N={rows} cg={cg}: {T} tiles on {W} workers, K={K}: schedule {kind}, not front/tail"
    say(f"{what}: N={rows} cg={cg} T={T} W={W} K={K} kbw={min(kbw, K)} s={s}")
    return s


# ---------------------------------------------------------------------------------------------------------------------
# cells on the device, their layouts, and the exact reference
# ---------------------------------------------------------------------------------------------------------------------
def _dosage(seed, n, nv):
    """(n, nv) int8 dosages 0 / 1 / 2 on the device; the last sample and the last variant are never 0, so that a cell lost
    or added at a ragged edge (the last row of a tile, the last k-block) changes the Gram."""
    import torch
    g = torch.Generator(device="cuda").manual_seed(seed)
    u = torch.rand((n, nv), generator=g, device="cuda")
    X = (u < 0.4).to(torch.int8) + (u < 0.12).to(torch.int8)
    X[-1, :] = 1 + (u[-1, :] < 0.3).to(torch.int8)
    X[:, -1] = 1 + (u[:, -1] < 0.3).to(torch.int8)
    return X


def _pack_e2m1(codes):
    """uint8 e2m1 codes (even count along the last axis) -> bytes, cell j in nibble j & 1."""
    return codes[..., 0::2] | (codes[..., 1::2] << 4)


def _stored(X, dt):
    """int8 cells -> the stored bytes (uint8): int8, bf16 bits, or packed e2m1 codes 2 m."""
    import torch
    if dt == "i8":
        return X.view(torch.uint8)
    if dt == "bf16":
        return X.to(torch.bfloat16).view(torch.uint8)
    return _pack_e2m1((2 * X).to(torch.uint8))


def _panels(X, dt):
    """Panel layout of vpca_accumulate_panels as a flat uint8 device buffer: ceil(nv / PANEL) panels of n x PANEL cells,
    zero after nv."""
    import torch
    n, nv = X.shape
    npan = -(-nv // PANEL)
    Xp = torch.zeros((npan, n, PANEL), dtype=torch.int8, device="cuda")
    for p in range(npan):
        w = min(PANEL, nv - p * PANEL)
        Xp[p, :, :w] = X[:, p * PANEL:p * PANEL + w]
    return _stored(Xp, dt).reshape(-1)


def _row_major(X, dt):
    """Row-major device tile with junk in every column past nv that the contract leaves to the caller (int8 127, bf16 NaN
    bits; e2m1: zero cells up to the next multiple of 128 cells, junk bytes after) -> (uint8 (n, row bytes), ld).  ld
    runs past nv and keeps every row 16-byte aligned (e2m1: a multiple of 128 cells)."""
    import torch
    n, nv = X.shape
    if dt == "e2m1":
        ld = -(-nv // 128) * 128 + 128
        codes = torch.zeros((n, ld), dtype=torch.uint8, device="cuda")
        codes[:, :nv] = (2 * X).to(torch.uint8)
        out = _pack_e2m1(codes).contiguous()
        out[:, -(-nv // 128) * 64:] = 0xFF
        return out, ld
    step = 16 if dt == "i8" else 8
    ld = -(-nv // step) * step + step
    if dt == "i8":
        T = torch.full((n, ld), 127, dtype=torch.int8, device="cuda")
        T[:, :nv] = X
    else:
        T = torch.full((n, ld), float("nan"), dtype=torch.bfloat16, device="cuda")
        T[:, :nv] = X.to(torch.bfloat16)
    return T.view(torch.uint8), ld


def _exact(X):
    import torch
    Xf = X.to(torch.float64)
    return (Xf @ Xf.t()).to(torch.int32)


def _assert_equal(got, want, what):
    import torch
    if not torch.equal(got, want):
        bad = torch.nonzero(got != want)
        r, c = (int(v) for v in bad[0])
        raise AssertionError(f"{what}: {len(bad)} cells differ, rows {int(bad[:, 0].min())}..{int(bad[:, 0].max())}, "
                             f"cols {int(bad[:, 1].min())}..{int(bad[:, 1].max())}; first ({r}, {c}): got "
                             f"{int(got[r, c])}, want {int(want[r, c])}")


def _assert_partial(nat, ref, what):
    """The lower triangle of the accumulated (not finalized) Gram equals that of the FP64 running sum."""
    import torch
    part = torch.from_numpy(nat.partialGram()).cuda()
    _assert_equal(torch.tril(part), torch.tril(ref.to(torch.int32)), what)


# ---------------------------------------------------------------------------------------------------------------------
# 1. launch length: K = 1, 2, 3, either side of a window and several windows, in every layout, cell type and CTA group
# ---------------------------------------------------------------------------------------------------------------------
def _window(layout, dt, n):
    """Window length the launch uses with VPCA_KB_WINDOW unset: one panel for panels (the device's or the staging's), and
    for a row-major device tile a 16 MiB slice of X, at least 8 k-blocks."""
    if layout == "devrows":
        return max(8, min(4096, (16 << 20) // (n * 128)))
    return PANEL // CELLS_PER_KB[dt]


@pytest.mark.parametrize("adapt", ("fixed", "adaptive"))
@pytest.mark.parametrize("layout", ("panels", "devrows", "hostrows"))
@pytest.mark.parametrize("edge", ("first", "last"))
@pytest.mark.parametrize("cg", (1, 2))
@pytest.mark.parametrize("dt", DTYPES)
def test_launch_lengths_at_the_range_edges(monkeypatch, say, dt, cg, edge, layout, adapt):
    """K in {1, 2, 3, kbw - 1, kbw, kbw + 1, 3 kbw + 5}, every last k-block RAGGED cells short.  K = 1 gives s = 0: the
    front workers have no piece and the tail multiplies every tile.  K < kbw clamps the window to K."""
    import torch
    native = _native()
    _env(monkeypatch, cg, **({"VPCA_ADAPTIVE": 0} if adapt == "fixed" else {}))
    n = _row_range(cg)[0 if edge == "first" else 1]
    kbw = _window(layout, dt, n)
    with native.NativePca(n, dtype=_dtype(dt)) as nat:
        for K in (1, 2, 3, kbw - 1, kbw, kbw + 1, 3 * kbw + 5):
            s = _schedule(say, f"{dt} {layout} {adapt}", n, cg, kbw, K)
            if K == 1:
                assert s == 0
            nv = K * CELLS_PER_KB[dt] - RAGGED
            X = _dosage(SEED + 7919 * K + 101 * n + 10 * cg + DTYPES.index(dt), n, nv)
            if layout == "panels":
                buf = _panels(X, dt)
                torch.cuda.synchronize()                       # the context's stream reads what torch's wrote
                nat.accumulatePanels(buf.data_ptr(), nv, PANEL)
            elif layout == "devrows":
                buf, ld = _row_major(X, dt)
                torch.cuda.synchronize()
                nat.accumulateDenseDevice(buf.data_ptr(), nv, ld)
            else:
                host = _row_major(X, dt)[0].cpu().numpy()
                nat.accumulateDense(host.view({"i8": np.int8, "bf16": np.uint16, "e2m1": np.uint8}[dt]), nv)
            nat.finalizeGram()
            st = nat.stats()
            S = torch.from_numpy(nat.getGram()).cuda()
            assert st["gram_resident"] == 1 and st["gram_cta_group"] == cg
            _assert_equal(S, _exact(X), f"{dt} {layout} {adapt} N={n} cg={cg} K={K} s={s}")
            nat.reset()


# ---------------------------------------------------------------------------------------------------------------------
# 2. kernel options under front/tail, s inside a window of a multi-window launch
# ---------------------------------------------------------------------------------------------------------------------
OPTION_KBW = PANEL // 128          # int8 panels: one window per panel

OPTIONS = [
    pytest.param(cg, size, exact, env, id=f"{name}-cg{cg}")
    for name, size, exact, env, cgs in (
        ("sync_lead1", "ragged", False, {"VPCA_SYNC_LEAD": 1}, (1, 2)),
        ("sync_lead2", "ragged", False, {"VPCA_SYNC_LEAD": 2}, (1, 2)),
        ("red32_odd_n", "odd", False, {"VPCA_RED64": 0}, (1, 2)),        # odd N flushes per cell whatever VPCA_RED64 is
        ("red32_even_n", "ragged", False, {"VPCA_RED64": 0}, (1, 2)),    # even N: the switch takes the 32-bit path
        ("no_self_b", "ragged", False, {"VPCA_SELF_B": 0}, (2,)),        # self-B tiles exist with CTA pairs only
        ("exact_cover", "ragged", True, {"VPCA_EXACT_COVER": 1}, (1, 2)),
    )
    for cg in cgs
]


def _multi_window_k(n, cg, exact, kbw):
    """Smallest K >= 4 kbw whose initial split point lies inside the third window or later (the front walks at least
    three windows, so a pacing lead of 2 waits)."""
    W = _workers(cg)
    for K in range(4 * kbw, 40 * kbw):
        _, kind, s = _native().debugSchedule(n, cg, exact, W, kbw, K)
        if kind == 2 and s > 2 * kbw and s % kbw:
            return K
    raise AssertionError(f"no K puts the split point inside a window (N={n}, cg={cg})")


@pytest.mark.parametrize("cg,size,exact,env", OPTIONS)
def test_kernel_options_under_front_tail(monkeypatch, say, cg, size, exact, env):
    """A multi-window launch with s inside a window, then a K = 1 launch, on one context with each option."""
    import torch
    native = _native()
    _env(monkeypatch, cg, VPCA_ADAPTIVE=0, **env)
    n = _odd_n(cg, exact) if size == "odd" else _ragged_n(cg, exact)
    opt = " ".join(f"{k}={v}" for k, v in env.items())
    with native.NativePca(n) as nat:
        ref = torch.zeros((n, n), dtype=torch.float64, device="cuda")
        for K in (_multi_window_k(n, cg, exact, OPTION_KBW), 1):
            s = _schedule(say, opt, n, cg, OPTION_KBW, K, exact)
            nv = K * 128 - RAGGED
            X = _dosage(SEED + 31 * K + n + cg, n, nv)
            buf = _panels(X, "i8")
            torch.cuda.synchronize()
            nat.accumulatePanels(buf.data_ptr(), nv, PANEL)
            Xf = X.to(torch.float64)
            ref += Xf @ Xf.t()
            _assert_partial(nat, ref, f"{opt} N={n} cg={cg} K={K} s={s}")
        nat.finalizeGram()
        assert nat.stats()["gram_cta_group"] == cg
        _assert_equal(torch.from_numpy(nat.getGram()).cuda(), ref.to(torch.int32), f"{opt} N={n} cg={cg}")


# ---------------------------------------------------------------------------------------------------------------------
# 3. staged partitions of every host form, committed one by one; an abort and a retry; two threads on one context
# ---------------------------------------------------------------------------------------------------------------------
STAGED_SIZES = (1, 127, 128, 129, 700)
STAGED_FORMS = ("csr32", "csr16", "bits", "bedA1", "bedA2")


def _np_dosage(rng, n, nv):
    u = rng.random((n, nv))
    X = ((u < 0.4).astype(np.int8) + (u < 0.12).astype(np.int8)).astype(np.int8)
    X[-1, :] = 1 + (u[-1, :] < 0.3)
    X[:, -1] = 1 + (u[:, -1] < 0.3)
    return X


def _csr(X):
    """CSR rows of dosage cells: a sample with cell 2 is listed twice."""
    XT = np.ascontiguousarray(X.T)
    v, s = np.nonzero(XT)
    idx = np.repeat(s.astype(np.int32), XT[v, s].astype(np.int64))
    off = np.zeros(X.shape[1] + 1, np.int64)
    off[1:] = np.cumsum(XT.sum(axis=1, dtype=np.int64))
    return off, idx


def _bitmap_rows(rng, Xb):
    """Bitmap rows of binary cells: every padding bit after sample n - 1 set, three junk bytes after ceil(n / 8)."""
    n, nv = Xb.shape
    nb = -(-n // 8)
    rows = np.zeros((nv, nb + 3), np.uint8)
    rows[:, :nb] = np.packbits(Xb.T.astype(np.uint8), axis=1, bitorder="little")
    if n % 8:
        rows[:, nb - 1] |= np.uint8((0xFF << (n % 8)) & 0xFF)
    rows[:, nb:] = rng.integers(0, 256, (nv, 3), dtype=np.uint8)
    return rows


def _bed_rows(rng, n, nv):
    """.bed rows of random codes (00 hom A1, 01 missing, 10 het, 11 hom A2; a quarter of the calls missing), random
    padding codes after sample n - 1 and five junk bytes after ceil(n / 4) -> (rows, carriers of A1, carriers of A2)."""
    nb = -(-n // 4)
    codes = rng.integers(0, 4, (nv, 4 * nb), dtype=np.uint8)
    rows = np.zeros((nv, nb + 5), np.uint8)
    rows[:, :nb] = codes[:, 0::4] | (codes[:, 1::4] << 2) | (codes[:, 2::4] << 4) | (codes[:, 3::4] << 6)
    rows[:, nb:] = rng.integers(0, 256, (nv, 5), dtype=np.uint8)
    c = codes[:, :n].T
    return rows, ((c == 0) | (c == 2)).astype(np.int8), ((c == 2) | (c == 3)).astype(np.int8)


def _stage(nat, rng, form, pid, nv):
    """Stages nv variants of `form` into partition pid -> (the (n, nv) int8 cells they add to the Gram, CSR rows or None)."""
    n = nat.n
    if form in ("csr32", "csr16"):
        X = _np_dosage(rng, n, nv)
        off, idx = _csr(X)
        if form == "csr32":
            nat.accumulateCalls(pid, off, idx)
        else:
            nat.accumulateCalls16(pid, off, idx.astype(np.uint16))
        return X, (off, idx)
    if form == "bits":
        X = (rng.random((n, nv)) < 0.3).astype(np.int8)
        X[-1, :] = X[:, -1] = 1
        nat.accumulateBits(pid, _bitmap_rows(rng, X))
        return X, None
    rows, a1, a2 = _bed_rows(rng, n, nv)
    nat.accumulateBed(pid, rows, counted_allele=1 if form == "bedA1" else 2)
    return (a1 if form == "bedA1" else a2), None


def _add(ref, X):
    import torch
    Xf = torch.from_numpy(X).cuda().to(torch.float64)
    ref += Xf @ Xf.t()


@pytest.mark.parametrize("where", ("ragged", "last"))
@pytest.mark.parametrize("cg", (1, 2))
def test_staged_partitions(monkeypatch, say, oracle, cg, where):
    """Every form in partitions of 1, 127, 128, 129 and 700 variants (K = 1, 1, 1, 2, 6), each committed and the partial
    Gram checked after it; the CSR int32 partitions also against the oracle; then a partition staged in two calls,
    aborted and staged again; the committed Gram at the end.  At the last N of the range a single tail worker takes the
    pieces of every tile."""
    import torch
    native = _native()
    _env(monkeypatch, cg)
    n = _ragged_n(cg) if where == "ragged" else _row_range(cg)[1]
    for nv in STAGED_SIZES:
        _schedule(say, f"staged partition of {nv} variants", n, cg, PANEL // 128, -(-nv // 128))
    rng = np.random.default_rng([SEED, n, cg])
    ref = torch.zeros((n, n), dtype=torch.float64, device="cuda")
    with native.NativePca(n) as nat:
        pid = 0
        for form in STAGED_FORMS:
            csr = []
            for nv in STAGED_SIZES:
                X, rows = _stage(nat, rng, form, pid, nv)
                nat.commit(pid)
                _add(ref, X)
                _assert_partial(nat, ref, f"{form} partition {pid} of {nv} variants, N={n} cg={cg}")
                if rows is not None:
                    csr.append(rows)
                pid += 1
            if form == "csr32":                                # every partition so far: the oracle's similarity
                offs, base = [np.zeros(1, np.int64)], 0
                for o, i in csr:
                    offs.append(o[1:] + base)
                    base += len(i)
                want = oracle.c_similarity(n, np.concatenate(offs), np.concatenate([i for _, i in csr]))
                part = nat.partialGram()
                assert np.array_equal(np.tril(part), np.tril(want)), f"csr32 partitions against the oracle, N={n} cg={cg}"
        # staged in two calls (two launches into one staging Gram), aborted: the Gram keeps none of it; staged again
        X = _np_dosage(rng, n, 300)
        for attempt in ("aborted", "retried"):
            for a, b in ((0, 129), (129, 300)):
                nat.accumulateCalls(pid, *_csr(X[:, a:b]))
            if attempt == "aborted":
                nat.abort(pid)
            else:
                nat.commit(pid)
                _add(ref, X)
            _assert_partial(nat, ref, f"{attempt} partition, N={n} cg={cg}")
        nat.finalizeGram()
        assert nat.stats()["gram_cta_group"] == cg
        _assert_equal(torch.from_numpy(nat.getGram()).cuda(), ref.to(torch.int32), f"committed Gram, N={n} cg={cg}")


def test_two_threads_feed_one_context(monkeypatch, say):
    """Two host threads stage and commit partitions into one context at the same time, so that both staging lanes run
    their own Gram plan (and adapt their own split point) concurrently."""
    import torch
    native = _native()
    _env(monkeypatch, 2)
    n = _ragged_n(2)
    for nv in STAGED_SIZES:
        _schedule(say, f"two threads, partitions of {nv} variants", n, 2, PANEL // 128, -(-nv // 128))
    added = [[], []]
    errors = []
    with native.NativePca(n) as nat:
        start = threading.Barrier(2)

        def feed(t):
            try:
                rng = np.random.default_rng([SEED, t])
                start.wait()
                for r in range(3):
                    for i, nv in enumerate(STAGED_SIZES):
                        pid = 1000 * (t + 1) + 10 * r + i
                        X, _ = _stage(nat, rng, STAGED_FORMS[(i + r + t) % len(STAGED_FORMS)], pid, nv)
                        nat.commit(pid)
                        added[t].append(X)
            except Exception as e:                             # re-raised by the main thread
                errors.append(e)

        threads = [threading.Thread(target=feed, args=(t,)) for t in range(2)]
        for th in threads:
            th.start()
        for th in threads:
            th.join()
        if errors:
            raise errors[0]
        nat.finalizeGram()
        S = torch.from_numpy(nat.getGram()).cuda()
    ref = torch.zeros((n, n), dtype=torch.float64, device="cuda")
    for X in added[0] + added[1]:
        _add(ref, X)
    assert len(added[0]) == len(added[1]) == 3 * len(STAGED_SIZES)
    _assert_equal(S, ref.to(torch.int32), f"two threads, N={n}")


# ---------------------------------------------------------------------------------------------------------------------
# 4. the kinship plane Gram (3N x 3N) in the front/tail range
# ---------------------------------------------------------------------------------------------------------------------
KIN_STEP = 8832        # rows per staged kinship chunk: 69 k-blocks of an 8192-variant panel, windows of 64 and 5


def _kin_geometry(n, stride):
    """(rows per chunk, k-blocks per window) of vpca_kinship_bed for a context made with chunk_nnz = _kin_chunk_nnz."""
    R = 3 * n
    panel = min(PANEL, max(128, ((256 << 20) // R // 128) * 128))
    chunk = max(panel, ((256 << 20) // R // panel) * panel)
    cap_rows = _kin_chunk_nnz(stride) * 4 // stride
    return min(chunk, cap_rows // 32 * 32), panel // 128


def _kin_chunk_nnz(stride):
    return -(-KIN_STEP * stride // 4)                  # the staging buffer holds KIN_STEP raw rows


def _kin_codes(rng, n, nv, missing=0.01):
    p = rng.uniform(0.05, 0.95, size=nv)[:, None]
    d = (rng.random((nv, n)) < p).astype(np.int64) + (rng.random((nv, n)) < p)
    c = dosage_codes(d.T)
    c[rng.random((nv, n)) < missing] = MISSING
    return c


def _assert_kinship(got, want, what):
    ids, counts, kin = got
    wids, wcounts, wkin = want
    assert np.array_equal(ids, wids), f"{what}: pair ids differ"
    assert np.array_equal(counts, wcounts), f"{what}: {int((counts != wcounts).any(axis=1).sum())} pairs' counts differ"
    assert np.array_equal(kin.view(np.int64), wkin.view(np.int64)), f"{what}: KINSHIP bits differ"


@pytest.mark.parametrize("which", ("first", "last", "700"))
@pytest.mark.parametrize("cg", (1, 2))
def test_kinship_plane_gram(monkeypatch, say, cg, which):
    """N at both edges of the range where 3N rows take the front/tail schedule, and N = 700.  Two calls of KIN_STEP + 1
    and KIN_STEP + 128 rows: chunks of KIN_STEP rows (two windows, s inside the first or second), then tails of 1 and
    128 rows (K = 1, s = 0)."""
    native = _native()
    _env(monkeypatch, cg)
    lo, hi = _row_range(cg)
    n = {"first": -(-lo // 3), "last": hi // 3, "700": 700}[which]
    stride = -(-n // 4)
    step, kbw = _kin_geometry(n, stride)
    assert step == KIN_STEP
    for K in (KIN_STEP // 128, 1):
        _schedule(say, f"kinship of {n} samples", 3 * n, cg, kbw, K)
    codes = _kin_codes(np.random.default_rng([SEED, n, cg]), n, 2 * KIN_STEP + 129)
    rows = pack_codes(codes)
    with native.NativePca(n, chunk_nnz=_kin_chunk_nnz(stride)) as nat:
        nat.kinshipBed(rows[:KIN_STEP + 1])
        nat.kinshipBed(rows[KIN_STEP + 1:])
        got = nat.kinshipPairs()
    _assert_kinship(got, king_pairs(codes), f"kinship N={n} cg={cg}")


# ---------------------------------------------------------------------------------------------------------------------
# 5. the LD plane Gram (3c x 3c) in the front/tail range
# ---------------------------------------------------------------------------------------------------------------------
LD_R2 = 0.2


def _ld_launches(n, c):
    """(k-blocks, window) of every plane-Gram launch of vpca_ld_prune_bed for one chunk of c variants of n samples: one
    per piece of the sample axis, as the library cuts it."""
    R = 3 * c
    n128 = -(-n // 128) * 128
    P = min(n128, max(128, min(PANEL, (16 << 20) // R // 128 * 128)))
    piece = max(P, min(32768, (256 << 20) // R) // P * P)
    piece = min(piece, -(-n // P) * P)
    return [(-(-min(piece, n - s0) // 128), P // 128) for s0 in range(0, n, piece)]


def _ld_dosage(rng, n, v, block=6, copy=0.85, missing=0.02):
    """(n, v) A1 counts in LD blocks: each variant copies its block's founder on a `copy` share of the samples."""
    nb = -(-v // block)
    founder = rng.binomial(2, rng.uniform(0.05, 0.5, nb)[:, None], size=(nb, n))
    own = rng.binomial(2, rng.uniform(0.05, 0.5, v)[:, None], size=(v, n))
    d = np.where(rng.random((v, n)) < copy, founder[np.arange(v) // block], own)
    d[rng.random((v, n)) < missing] = -1
    return d.T


@functools.lru_cache(maxsize=None)
def _ld_case(n, nv):
    """.bed rows of nv variants on two contigs, 1 kb apart (windows of 30 kb: 30 variants back), their window starts and
    the reference result; shared by both CTA groups where nv is the same."""
    rows = pack_codes(dosage_codes(_ld_dosage(np.random.default_rng([SEED, n, nv]), n, nv)))
    contigs = ["1"] * (nv // 2) + ["2"] * (nv - nv // 2)
    positions = np.concatenate([np.arange(nv // 2), np.arange(nv - nv // 2)]) * 1000 + 1
    window_lo = ld_ref.window_starts(contigs, positions, 30)
    return rows, window_lo, ld_ref.prune(rows, n, window_lo, LD_R2)


@pytest.mark.parametrize("n", (100, 2504, 40000))
@pytest.mark.parametrize("edge", ("first", "last"))
@pytest.mark.parametrize("cg", (1, 2))
def test_ld_plane_gram(monkeypatch, say, cg, edge, n):
    """nv variants (one chunk of c = nv rounded up to 32) with 3c rows at the first or last c of the range (the first
    with nv 31 short of c); keep, pairs and r2 bits against ld_ref, and the pair list truncated to half."""
    native = _native()
    _env(monkeypatch, cg)
    lo, hi = _row_range(cg)
    c = -(-lo // 96) * 32 if edge == "first" else hi // 96 * 32
    nv = c - 31 if edge == "first" else c
    assert c <= 1024 and _in_range(3 * c, cg)
    for i, (K, kbw) in enumerate(_ld_launches(n, c)):
        _schedule(say, f"LD of {nv} variants x {n} samples, piece {i}", 3 * c, cg, kbw, K)
    rows, window_lo, (want_keep, want_pairs, want_r2) = _ld_case(n, nv)
    assert len(want_pairs) > 10
    with native.NativePca(n) as nat:
        keep, pairs, r2 = nat.ldPruneBed(rows, window_lo, LD_R2, max_pairs=len(want_pairs) + 1)
        what = f"LD nv={nv} n={n} cg={cg}"
        assert np.array_equal(pairs, want_pairs), f"{what}: pairs differ"
        assert np.array_equal(r2.view(np.int64), want_r2.view(np.int64)), f"{what}: r2 bits differ"
        assert np.array_equal(keep, want_keep), f"{what}: keep differs"
        m = len(want_pairs) // 2
        keep, pairs, r2 = nat.ldPruneBed(rows, window_lo, LD_R2, max_pairs=m)
        assert np.array_equal(pairs, want_pairs[:m]) and np.array_equal(r2.view(np.int64), want_r2[:m].view(np.int64))
        assert np.array_equal(keep, want_keep), f"{what}: keep differs when the pairs are truncated"


# ---------------------------------------------------------------------------------------------------------------------
# 6. the split point adapting across shapes in one process
# ---------------------------------------------------------------------------------------------------------------------
ADAPT_N = 2504
ADAPT_LONG = 16 * PANEL             # 1024 k-blocks: ~0.65 ms on an H100 SXM, past the 0.3 ms a launch needs to be timed


def test_split_point_adapts_across_shapes(monkeypatch, say):
    """16 long launches with VPCA_REBALANCE_GAIN=1, each followed by a K = 1 or K = 3 launch (a window clamped to 1 or 3,
    another entry of the remembered split points); a kinship context at N = 700 after the eighth; then a fresh context
    at N = 2504 that starts from the split point the first one left.  The lower triangle is checked after every launch."""
    import torch
    native = _native()
    _env(monkeypatch, 2, VPCA_REBALANCE_GAIN=1)
    n, kbw = ADAPT_N, PANEL // 128
    shorts = (1 * 128 - RAGGED, 3 * 128 - RAGGED)
    for nv in (ADAPT_LONG,) + shorts:
        _schedule(say, "adapting launches (initial s)", n, 2, kbw, -(-nv // 128))
    stream = torch.cuda.Stream()
    buf = torch.empty(ADAPT_LONG * n, dtype=torch.uint8, device="cuda")
    v0 = [0]

    def launch(nat, ref, nv, what):
        stream.wait_stream(torch.cuda.current_stream())       # ref was made on torch's stream
        with torch.cuda.stream(stream):
            nat.synthPanelsDevice(SEED, v0[0], nv, 1, buf.data_ptr(), PANEL)
            nat.accumulatePanels(buf.data_ptr(), nv, PANEL)
            X = buf[:-(-nv // PANEL) * n * PANEL].view(torch.int8).view(-1, n, PANEL)
            for p in range(X.shape[0]):
                Xf = X[p].to(torch.float64)
                ref += Xf @ Xf.t()
            stream.synchronize()
        v0[0] += nv
        assert nat.stats()["gram_resident"] == 1
        _assert_partial(nat, ref, what)

    with native.NativePca(n, stream=stream.cuda_stream) as nat:
        ref = torch.zeros((n, n), dtype=torch.float64, device="cuda")
        for i in range(16):
            launch(nat, ref, ADAPT_LONG, f"long launch {i}")
            launch(nat, ref, shorts[i % 2], f"short launch after long launch {i}")
            if i == 7:
                kn = 700
                _schedule(say, "kinship between the adapting launches", 3 * kn, 2, PANEL // 128, 8)
                codes = _kin_codes(np.random.default_rng([SEED, kn]), kn, 8 * 128 - RAGGED)
                with native.NativePca(kn) as kin:
                    kin.kinshipBed(pack_codes(codes))
                    _assert_kinship(kin.kinshipPairs(), king_pairs(codes), "kinship between the adapting launches")
                _assert_partial(nat, ref, "after the kinship context")
        nat.finalizeGram()
        _assert_equal(torch.from_numpy(nat.getGram()).cuda(), ref.to(torch.int32), "first context")
    with native.NativePca(n, stream=stream.cuda_stream) as nat:
        ref = torch.zeros((n, n), dtype=torch.float64, device="cuda")
        for i in range(4):
            launch(nat, ref, ADAPT_LONG, f"fresh context, long launch {i}")
        launch(nat, ref, shorts[0], "fresh context, K = 1")
        nat.finalizeGram()
        _assert_equal(torch.from_numpy(nat.getGram()).cuda(), ref.to(torch.int32), "fresh context")
