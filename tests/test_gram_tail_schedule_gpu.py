"""The Gram kernel's front/tail schedule on the device: bit-exact Grams against FP64 X X^T of the same cells (exact: every
count stays far below 2^53).

At 2504 samples the tiles (55 CTA-pair tiles, 110 single-CTA tiles) number more than half the workers and fewer than
all of them, so the front workers multiply their tile over k-blocks [0, s) and the tail workers split the rest of
every tile over [s, K), flushing each piece.  The cases put s on a window edge and inside a panel, in every cell type
and both CTA groups, route the tail's flushes to peers on one device (replicate and owner-rows, 2 and 3 ranks), and
run 16 launches while s adapts, then a second context that starts from the remembered s.
"""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

N = 2504
P = 8192                    # panel width in cells
KBW = 64                    # pinned window: VPCA_KB_WINDOW
CELLS_PER_KB = {"i8": 128, "bf16": 64, "e2m1": 128}


def _native():
    import __graft_entry__ as entry
    from spark_examples_b200 import native
    if not native.library_path().exists():
        entry.build()
    native.load_library()
    return native


def _workers(cg):
    import torch
    native = _native()
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    return sms if cg == 1 else min(sms // 2, native.maxClusters(0, 2))


def _env(monkeypatch, cg, **extra):
    monkeypatch.setenv("VPCA_CTA_GROUP", str(cg))
    monkeypatch.setenv("VPCA_KB_WINDOW", str(KBW))
    for k in ("VPCA_EXACT_COVER", "VPCA_ADAPTIVE", "VPCA_REBALANCE_GAIN", "VPCA_GRAM_PROF", "VPCA_SELF_B", "VPCA_RED64",
              "VPCA_SYNC_LEAD"):
        monkeypatch.delenv(k, raising=False)
    for k, v in extra.items():
        monkeypatch.setenv(k, str(v))


def _dosage(seed, nv):
    """(N, nv) int8 dosages 0 / 1 / 2 on the device; the last sample and the last variant never 0."""
    import torch
    g = torch.Generator(device="cuda").manual_seed(seed)
    u = torch.rand((N, nv), generator=g, device="cuda")
    X = (u < 0.4).to(torch.int8) + (u < 0.12).to(torch.int8)
    X[-1, :] = 1 + (u[-1, :] < 0.3).to(torch.int8)
    X[:, -1] = 1 + (u[:, -1] < 0.3).to(torch.int8)
    return X


def _panels(X, dt):
    """Panel layout of vpca_accumulate_panels as a uint8 device buffer: ceil(nv / P) panels of N x P cells, zero after nv."""
    import torch
    nv = X.shape[1]
    npan = -(-nv // P)
    Xp = torch.zeros((npan, N, P), dtype=torch.int8, device="cuda")
    for p in range(npan):
        w = min(P, nv - p * P)
        Xp[p, :, :w] = X[:, p * P:p * P + w]
    if dt == "i8":
        return Xp.view(torch.uint8).reshape(-1)
    if dt == "bf16":
        return Xp.to(torch.bfloat16).view(torch.uint8).reshape(-1)
    codes = (2 * Xp).to(torch.uint8)                          # e2m1 code of 0, 1, 2: 0, 2, 4
    return (codes[..., 0::2] | (codes[..., 1::2] << 4)).reshape(-1)


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


def _dtype(native, dt):
    return {"i8": native.DTYPE_I8, "bf16": native.DTYPE_BF16, "e2m1": native.DTYPE_E2M1}[dt]


def _kb_total_with_split(cg, where):
    """K (>= 380) whose initial split point s = floor(K T / W) is a window edge (s % 64 == 0) or mid-window (32)."""
    native = _native()
    W = _workers(cg)
    T = len(native.debugTiles(N, cg, False))
    if not W < 2 * T < 2 * W:
        pytest.skip(f"{T} tiles on {W} workers: no front/tail schedule on this device")
    want = 0 if where == "edge" else KBW // 2
    for K in range(380, 4000):
        _, kind, s = native.debugSchedule(N, cg, False, W, KBW, K)
        assert kind == 2
        if 0 < s < K and s % KBW == want:
            return K, s
    raise AssertionError("no K found")


@pytest.mark.parametrize("where", ("edge", "inside"))
@pytest.mark.parametrize("cg", (1, 2))
@pytest.mark.parametrize("dt", ("i8", "bf16", "e2m1"))
def test_split_point_at_window_edge_and_inside_a_panel(monkeypatch, dt, cg, where):
    import torch
    native = _native()
    _env(monkeypatch, cg, VPCA_ADAPTIVE=0)                 # s stays at its initial value
    K, s = _kb_total_with_split(cg, where)
    nv = K * CELLS_PER_KB[dt] - 5                            # ragged last k-block, same K
    X = _dosage(1000 + K, nv)
    buf = _panels(X, dt)
    torch.cuda.synchronize()
    with native.NativePca(N, dtype=_dtype(native, dt)) as nat:
        nat.accumulatePanels(buf.data_ptr(), nv, P)
        nat.finalizeGram()
        st = nat.stats()
        S = torch.from_numpy(nat.getGram()).cuda()
    assert st["gram_resident"] == 1 and st["gram_cta_group"] == cg
    _assert_equal(S, _exact(X), f"s = {s} of K = {K}")


@pytest.mark.parametrize("world", (2, 3))
@pytest.mark.parametrize("mode", ("replicate", "owner_rows"))
def test_tail_flushes_into_peers(monkeypatch, world, mode):
    """Ranks on one device, each with a shard of the variants: every flush, the tail's included, goes to all ranks'
    Grams (replicate) or to the row's owner (owner-rows, then gathered)."""
    import torch
    native = _native()
    _env(monkeypatch, 2, VPCA_ADAPTIVE=0)
    K, _ = _kb_total_with_split(2, "inside")
    nv = K * 128 * world
    X = _dosage(77 + world, nv)
    shards = [(r * nv // world // 128 * 128, (r + 1) * nv // world // 128 * 128) for r in range(world)]
    ctxs = []
    try:
        for _ in range(world):
            ctxs.append(native.NativePca(N, device=0))
        native.setPeersLocal(ctxs, mode)
        for c in ctxs:
            c.reset()
        for c in ctxs:
            c.synchronize()
        bufs = [_panels(X[:, a:b], "i8") for a, b in shards]
        torch.cuda.synchronize()                             # the contexts' streams read what torch's wrote
        for (a, b), c, buf in zip(shards, ctxs, bufs):
            c.accumulatePanels(buf.data_ptr(), b - a, P)
        for c in ctxs:
            c.peerBarrier()                                  # every rank's flushes have landed
        for c in ctxs:
            c.synchronize()
        want = _exact(X)
        L = torch.tril(want)
        bands = native.ownerRowBands(N, world) if mode == "owner_rows" else [(0, N)] * world
        for q, c in enumerate(ctxs):
            assert c.stats()["gram_resident"] == 1
            r0, rows = bands[q]
            routed = torch.zeros_like(L)
            routed[r0:r0 + rows] = L[r0:r0 + rows]
            _assert_equal(torch.from_numpy(c.partialGram()).cuda(), routed, f"rank {q} before the gather")
        for c in ctxs:
            c.gatherGram()
        for c in ctxs:
            c.finalizeGram()
        for q, c in enumerate(ctxs):
            _assert_equal(torch.from_numpy(c.getGram()).cuda(), want, f"rank {q}")
    finally:
        for c in ctxs:
            c.synchronize()
        for c in ctxs:
            c.close()


def _launches(nat, first, count, nv):
    """`count` launches of fresh dosages on one context, the lower triangle of the partial Gram exact after each."""
    import torch
    ref = torch.zeros((N, N), dtype=torch.float64, device="cuda")
    for i in range(count):
        X = _dosage(5000 + first + i, nv)
        buf = _panels(X, "i8")
        torch.cuda.synchronize()                             # the context's stream reads what torch's wrote
        nat.accumulatePanels(buf.data_ptr(), nv, P)
        Xf = X.to(torch.float64)
        ref += Xf @ Xf.t()
        part = torch.from_numpy(nat.partialGram()).cuda()
        _assert_equal(torch.tril(part), torch.tril(ref.to(torch.int32)), f"launch {first + i}")
        assert nat.stats()["gram_resident"] == 1
    return ref.to(torch.int32)


def test_adaptive_split_point_over_many_launches(monkeypatch):
    """16 launches of 16 panels (~0.65 ms each on an H100 SXM, long enough to be timed) with the split point moved after
    each, then a second context that starts from the split point the first one ended with."""
    import torch
    native = _native()
    _env(monkeypatch, 2, VPCA_REBALANCE_GAIN=1)
    _kb_total_with_split(2, "edge")                          # skips where the schedule does not apply
    nv = 16 * P
    with native.NativePca(N) as nat:
        want = _launches(nat, 0, 16, nv)
        nat.finalizeGram()
        assert torch.equal(torch.from_numpy(nat.getGram()).cuda(), want)
    with native.NativePca(N) as nat:
        want = _launches(nat, 16, 4, nv)
        nat.finalizeGram()
        assert torch.equal(torch.from_numpy(nat.getGram()).cuda(), want)
