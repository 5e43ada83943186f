"""The fused multi-context Gram reductions against exact integer Grams, bit for bit on every rank: the replicate epilogue,
the owner-rows reduce-scatter with its push / pull / copy gather, commits of staged partitions into peers and owners,
band-only owner-flush contexts and owner-computes bands.

On a one-GPU machine all contexts share device 0 (DESIGN.md 5), so every reduction runs there too.  Each case names the
edge it hits (N % 4, odd N, 32-row bands at N = 64 x world, band ends inside a 128-row A block or a 256-row B strip) and
asserts the band geometry it relies on.  Every barrier (peerBarrier / gatherGram) is enqueued on all ranks before the
host blocks on any of them, and the cases are small, so no barrier spins for long."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

SEED = 20261016
P = 512                          # panel width of the device-resident shards
COHORTS = (0, 1 << 20)           # first variant of the cohort of pass 0 / pass 1: stale rows of pass 0 cannot match
CHUNK = dict(chunk_variants=8192, chunk_nnz=1 << 22)   # host-input staging sized for the test, not ~1 GB per context


def _devices(world):
    import torch
    nd = max(1, torch.cuda.device_count())
    return [g % nd for g in range(world)]


_CELLS = {}
_GRAM = {}


def _cells(oracle, n, v0, nv, mode=1):
    """the synthetic generator's cells (mode 1: dosages 0/1/2, mode 0: carriers) of variants [v0, v0 + nv)"""
    key = (n, v0, nv, mode)
    if key not in _CELLS:
        _CELLS[key] = oracle.c_synth_dense(SEED, n, v0, nv, mode)
    return _CELLS[key]


def _gram(oracle, n, v0, nv, mode=1):
    """exact S = X X^T of those cells (float64 BLAS: every count is far below 2^53)"""
    key = (n, v0, nv, mode)
    if key not in _GRAM:
        X = _cells(oracle, n, v0, nv, mode).astype(np.float64)
        S = X @ X.T
        assert S.max() < 2 ** 31
        _GRAM[key] = S.astype(np.int32)
    return _GRAM[key]


def _edges(n, world):
    """the named edges (n, world) hits"""
    out = {"n%4==0" if n % 4 == 0 else ("n%4==2" if n % 4 == 2 else "odd")}
    if n >= 64 * world and world > 1:
        from spark_examples_b200 import native
        bands = native.ownerRowBands(n, world)
        ends = [r0 + rows for r0, rows in bands][:-1]
        if n == 64 * world and min(rows for _, rows in bands) == 32:
            out.add("32-row bands")
        if any(e % 128 for e in ends):
            out.add("end inside a 128-row block")
        if any(e % 256 for e in ends):
            out.add("end inside a 256-row strip")
    return out


def _env(monkeypatch, cta_group=None, **env):
    for name in ("VPCA_CTA_GROUP", "VPCA_EXACT_COVER", "VPCA_RED64", "VPCA_GATHER"):
        monkeypatch.delenv(name, raising=False)
    if cta_group is not None:
        monkeypatch.setenv("VPCA_CTA_GROUP", str(cta_group))
    for name, value in env.items():
        monkeypatch.setenv(name, str(value))


def _close(ctxs):
    for c in ctxs:
        try:
            c.synchronize()
        except Exception:
            pass
    for c in ctxs:
        c.close()


def _shards(nv, world):
    return [(r * nv // world, (r + 1) * nv // world) for r in range(world)]


def _panels(ctx, dev, v0, nv):
    """a zeroed device buffer holding the generator's cells of variants [v0, v0 + nv) in panel layout"""
    import torch
    with torch.cuda.device(dev):
        buf = torch.zeros(ctx.panelBytes(nv, P), dtype=torch.uint8, device=f"cuda:{dev}")
        torch.cuda.synchronize(dev)   # zeroed before the context's own stream writes the cells
    ctx.synthPanelsDevice(SEED, v0, nv, 1, buf.data_ptr(), P)
    return buf


def _begin(ctxs):
    for c in ctxs:
        c.reset()
    for c in ctxs:
        c.synchronize()                  # every Gram is zero before any peer adds into it


def _check_routing(ctxs, S, mode):
    """before the gather: owner-rows -> rank q holds tril(S) in exactly the rows it owns, zeros elsewhere; replicate ->
    every rank holds all of tril(S).  Catches a misrouted flush that the push would later overwrite, and a doubled one."""
    from spark_examples_b200 import native
    for c in ctxs:
        c.peerBarrier()                  # enqueued on every rank before the host blocks on any
    for c in ctxs:
        c.synchronize()
    L = np.tril(S)
    world, n = len(ctxs), S.shape[0]
    bands = native.ownerRowBands(n, world) if mode == "owner_rows" else [(0, n)] * world
    for q, c in enumerate(ctxs):
        r0, rows = bands[q]
        want = np.zeros_like(L)
        want[r0:r0 + rows] = L[r0:r0 + rows]
        got = c.partialGram()
        assert np.array_equal(got, want), (q, np.argwhere(got != want)[:5])


def _finish_full(ctxs, S):
    for c in ctxs:
        c.gatherGram()
    for c in ctxs:
        c.finalizeGram()
    for q, c in enumerate(ctxs):
        got = c.getGram()
        assert np.array_equal(got, S), (q, np.argwhere(got != S)[:5])


def _check_bands(ctxs, bands, S):
    """every band holds its rows of tril(S) and nothing above the diagonal (a band of all N rows is a whole Gram, which
    finalizeGram mirrors: it holds S)"""
    L = np.tril(S)
    for q, (c, (r0, rows)) in enumerate(zip(ctxs, bands)):
        got = c.gramBand(r0, rows)
        if rows == S.shape[0]:
            assert np.array_equal(got, S), q
            continue
        low = np.tril(got, k=r0)
        assert np.array_equal(low, L[r0:r0 + rows]), (q, np.argwhere(low != L[r0:r0 + rows])[:5])
        assert not np.triu(got, k=r0 + 1).any(), q


# ---- A / B / F: full contexts fed device panels, both modes, two passes -------------------------------------------
def _case(world, n, edge, mode, cta_group=None, dtype="i8", nv=2048, tag="", **env):
    cg = f"-cg{cta_group}" if cta_group else ""
    extra = "".join(f"-{k}={v}" for k, v in env.items())
    return pytest.param(world, n, edge, mode, cta_group, dtype, nv, env,
                        id=f"{mode}-w{world}-n{n}-{edge.replace(' ', '_')}{cg}-{dtype}{extra}{tag}")


_GRID = [(1, 777, "odd"), (2, 128, "32-row bands"), (2, 1094, "n%4==2"), (3, 320, "n%4==0"), (3, 1093, "odd"),
         (5, 320, "32-row bands"), (5, 1029, "end inside a 128-row block"), (8, 512, "32-row bands"),
         (8, 1500, "end inside a 256-row strip"), (16, 1024, "32-row bands"), (16, 1094, "n%4==2")]
FULL_CASES = [_case(w, n, e, m, cg) for m in ("replicate", "owner_rows") for cg in (1, 2) for w, n, e in _GRID]
FULL_CASES += [_case(3, 1093, "odd", m, 2, VPCA_EXACT_COVER=1) for m in ("replicate", "owner_rows")]
FULL_CASES += [_case(2, 1094, "n%4==2", m, 1, VPCA_EXACT_COVER=1) for m in ("replicate", "owner_rows")]
FULL_CASES += [_case(3, 320, "n%4==0", m, VPCA_RED64=0) for m in ("replicate", "owner_rows")]
FULL_CASES += [_case(3, 1093, "odd", m, dtype=d) for m in ("replicate", "owner_rows") for d in ("bf16", "e2m1")]
FULL_CASES += [_case(4, 5000, "stream-K", m, nv=1024) for m in ("replicate", "owner_rows")]
FULL_CASES += [_case(4, 5000, "stream-K", "owner_rows", dtype="bf16", nv=1024)]
FULL_CASES += [_case(w, n, e, "owner_rows", VPCA_GATHER=g) for g in ("push", "pull", "copy")
               for w, n, e in ((2, 1024, "n%4==0"), (2, 1093, "odd"), (5, 1500, "n%4==0"), (5, 1029, "odd"))]


@pytest.mark.parametrize("world,n,edge,mode,cta_group,dtype,nv,env", FULL_CASES)
def test_full_contexts_reduce_exactly(oracle, monkeypatch, world, n, edge, mode, cta_group, dtype, nv, env):
    """Every rank's Gram kernel flushes its variant shard into the peers (replicate) or the row owners (owner_rows); two
    passes with reset, each on another cohort.  Before the gather the routing is exact; after it every rank holds S."""
    from spark_examples_b200 import native
    _env(monkeypatch, cta_group, **env)
    if edge == "stream-K":
        assert len(native.debugTiles(n, cta_group or 2)) > 200
    else:
        assert edge in _edges(n, world), (edge, _edges(n, world))
    dt = {"i8": native.DTYPE_I8, "bf16": native.DTYPE_BF16, "e2m1": native.DTYPE_E2M1}[dtype]
    devs = _devices(world)
    ctxs = []
    try:
        for r in range(world):
            ctxs.append(native.NativePca(n, device=devs[r], dtype=dt))
        native.setPeersLocal(ctxs, mode)
        for v0 in COHORTS:
            S = _gram(oracle, n, v0, nv)
            shards = _shards(nv, world)
            bufs = [_panels(c, devs[r], v0 + shards[r][0], shards[r][1] - shards[r][0]) for r, c in enumerate(ctxs)]
            _begin(ctxs)
            for r, c in enumerate(ctxs):
                c.accumulatePanels(bufs[r].data_ptr(), shards[r][1] - shards[r][0], P)
            _check_routing(ctxs, S, mode)
            _finish_full(ctxs, S)
            for r, c in enumerate(ctxs):
                st = c.stats()
                assert st["variants_accumulated"] == shards[r][1] - shards[r][0]
                if cta_group is not None:
                    assert st["gram_cta_group"] == cta_group
                if edge == "stream-K":
                    assert st["gram_resident"] == 0, st
            del bufs
    finally:
        _close(ctxs)


# ---- C: staged partitions into full contexts --------------------------------------------------------------------
def _calls(X):
    from oracle import oracle
    return oracle.dense_to_calls(X)


def _bits(X):
    """carrier cells (n, nv) -> (nv, ceil(n / 8)) bitmap rows, bit s (LSB first) of row v = sample s"""
    return np.packbits(X.T.astype(bool), axis=1, bitorder="little")


def _stage(ctx, pid, X, wire, n):
    """one partition of carrier cells X through `wire`; pid % 4 == 1: written, aborted and retried; pid % 4 == 2: a
    corrupt batch poisons the partition first.  Returns the number of variants committed (those with carriers; a
    bitmap row without carriers counts too, so these cells have none)."""
    assert X.any(axis=0).all()
    off, idx = _calls(X)
    if pid % 4 == 1:
        ctx.accumulateCalls(pid, off, idx)
        ctx.abort(pid)
    if pid % 4 == 2:
        bad = idx.copy()
        bad[len(bad) // 2] = n + 5
        with pytest.raises(IndexError):
            ctx.accumulateCalls(pid, off, bad)
    if wire == "calls":
        ctx.accumulateCalls(pid, off, idx)
    elif wire == "calls16":
        ctx.accumulateCalls16(pid, off, idx)
    else:
        assert wire == "bits"
        ctx.accumulateBits(pid, _bits(X))
    ctx.commit(pid)
    return len(off) - 1


@pytest.mark.parametrize("mode", ["replicate", "owner_rows"])
@pytest.mark.parametrize("world,n", [(2, 1092), (3, 777)], ids=["w2-n1092-n%4==0", "w3-n777-odd"])
def test_staged_partitions_commit_into_peers_and_owners(oracle, monkeypatch, world, n, mode):
    """Every rank stages three partitions (calls, 16-bit calls, bitmap rows; one aborted and retried, one poisoned) and
    also accumulates a device shard directly, in the same pass.  The commit goes through add_i32_peers_kernel (replicate)
    or add_i32_owner_kernel (owner_rows).  Two passes with reset."""
    from spark_examples_b200 import native
    _env(monkeypatch)
    nvc, nvp, parts = 1536, 1024, 3
    devs = _devices(world)
    ctxs = []
    try:
        for r in range(world):
            ctxs.append(native.NativePca(n, device=devs[r], max_multiplicity=2, **CHUNK))
        native.setPeersLocal(ctxs, mode)
        for v0 in COHORTS:
            Xc = _cells(oracle, n, v0, nvc, 0)
            S = _gram(oracle, n, v0, nvc, 0) + _gram(oracle, n, v0 + nvc, nvp)
            cuts = _shards(nvc, world * parts)
            shards = _shards(nvp, world)
            bufs = [_panels(c, devs[r], v0 + nvc + shards[r][0], shards[r][1] - shards[r][0]) for r, c in enumerate(ctxs)]
            _begin(ctxs)
            staged = [0] * world
            for r, c in enumerate(ctxs):
                for j, wire in enumerate(("calls", "calls16", "bits")):
                    p = r * parts + j
                    staged[r] += _stage(c, p, Xc[:, cuts[p][0]:cuts[p][1]], wire, n)
                c.accumulatePanels(bufs[r].data_ptr(), shards[r][1] - shards[r][0], P)
            _check_routing(ctxs, S, mode)
            _finish_full(ctxs, S)
            for r, c in enumerate(ctxs):
                assert c.stats()["variants_accumulated"] == staged[r] + shards[r][1] - shards[r][0]
            del bufs
    finally:
        _close(ctxs)


@pytest.mark.parametrize("gpus,n", [(2, 100), (8, 500), (3, 777)],
                         ids=["G2-n100-replicate", "G8-n500-replicate", "G3-n777-owner_rows-odd"])
def test_pool_below_and_above_the_owner_rows_threshold(oracle, gpus, n):
    """The pool reduces in replicate mode when n < 64 x G and in owner-rows mode otherwise; partitions go to GPU p % G.
    Calls, 16-bit calls and bitmap rows, with abort + retry and a poisoned partition; two passes with reset."""
    from spark_examples_b200 import native
    nv, parts = 2048, 2 * gpus + 1
    with native.NativePcaPool(n, gpus, devices=_devices(gpus), max_multiplicity=2, **CHUNK) as pool:
        for v0 in COHORTS:
            X = _cells(oracle, n, v0, nv, 0)
            S = _gram(oracle, n, v0, nv, 0)
            pool.reset()
            sent = 0
            for p, (a, b) in enumerate(_shards(nv, parts)):
                off, idx = _calls(X[:, a:b])
                if p % 3 == 2:
                    off, idx = _calls(X[:, a:b][:, X[:, a:b].any(axis=0)])   # bitmap rows: the same variants
                sent += len(off) - 1
                if p % 4 == 1:
                    pool.accumulateCalls(p, off, idx)
                    pool.abort(p)
                if p % 4 == 2:
                    bad = idx.copy()
                    bad[len(bad) // 2] = n + 5
                    with pytest.raises(IndexError):
                        pool.accumulateCalls(p, off, bad)
                if p % 3 == 0:
                    pool.accumulateCalls16(p, off, idx)
                elif p % 3 == 1:
                    pool.accumulateCalls(p, off, idx)
                else:
                    pool.accumulateBits(p, _bits(X[:, a:b][:, X[:, a:b].any(axis=0)]))
                pool.commit(p)
            pool.reduceAndFinalize()
            got = pool.getGram()
            assert np.array_equal(got, S), np.argwhere(got != S)[:5]
            assert pool.stats()["variants_accumulated"] == sent


# ---- D / F: band-only owner-flush contexts ----------------------------------------------------------------------
def _band_case(world, n, edge, feed, dtype="i8", nv=2048, **env):
    extra = "".join(f"-{k}={v}" for k, v in env.items())
    return pytest.param(world, n, edge, feed, dtype, nv, env,
                        id=f"w{world}-n{n}-{edge.replace(' ', '_')}-{feed}-{dtype}{extra}")


BAND_CASES = [_band_case(w, n, e, f) for f in ("panels", "staged")
              for w, n, e in ((2, 128, "32-row bands"), (4, 256, "32-row bands"), (8, 512, "32-row bands"),
                              (16, 1024, "32-row bands"), (4, 1029, "odd"))]
BAND_CASES += [_band_case(4, 5000, "stream-K", "panels", nv=1024)]
BAND_CASES += [_band_case(w, n, e, "panels", VPCA_EXACT_COVER=1)
               for w, n, e in ((4, 1029, "odd"), (8, 512, "32-row bands"))]
BAND_CASES += [_band_case(w, n, e, f, dtype=d) for d in ("bf16", "e2m1") for f in ("panels", "staged")
               for w, n, e in ((4, 1029, "odd"),)]
BAND_CASES += [_band_case(8, 512, "32-row bands", "panels", dtype=d) for d in ("bf16", "e2m1")]


@pytest.mark.parametrize("world,n,edge,feed,dtype,nv,env", BAND_CASES)
def test_band_only_owner_flush(oracle, monkeypatch, world, n, edge, feed, dtype, nv, env):
    """Contexts that store only the band they own, wired in owner-rows mode.  Fed device panels (the Gram kernel flushes
    each row to its owner's band through the band's virtual origin) or staged partitions (add_i32_owner_kernel commits
    into the same virtual origins).  The bands are the result: no gather.  Two passes with reset."""
    from spark_examples_b200 import native
    _env(monkeypatch, **env)
    if edge == "stream-K":
        assert len(native.debugTiles(n, 2)) > 200
    else:
        assert edge in _edges(n, world), (edge, _edges(n, world))
    dt = {"i8": native.DTYPE_I8, "bf16": native.DTYPE_BF16, "e2m1": native.DTYPE_E2M1}[dtype]
    devs = _devices(world)
    bands = native.ownerRowBands(n, world)
    ctxs = []
    try:
        for r in range(world):
            ctxs.append(native.NativePca(n, device=devs[r], dtype=dt, gram_band=bands[r], **CHUNK))
        native.setPeersLocal(ctxs, "owner_rows")
        for v0 in COHORTS:
            S = _gram(oracle, n, v0, nv)
            shards = _shards(nv, world)
            bufs = []
            if feed == "panels":
                bufs = [_panels(c, devs[r], v0 + shards[r][0], shards[r][1] - shards[r][0]) for r, c in enumerate(ctxs)]
            X = _cells(oracle, n, v0, nv)
            _begin(ctxs)
            sent = [shards[r][1] - shards[r][0] for r in range(world)]
            for r, c in enumerate(ctxs):
                a, b = shards[r]
                if feed == "panels":
                    c.accumulatePanels(bufs[r].data_ptr(), b - a, P)
                else:
                    mid = (a + b) // 2
                    sent[r] = 0
                    for pid, (lo, hi) in ((2 * r, (a, mid)), (2 * r + 1, (mid, b))):
                        off, idx = _calls(X[:, lo:hi])
                        sent[r] += len(off) - 1
                        if pid % 2:                                     # written, aborted and retried
                            c.accumulateCalls16(pid, off, idx)
                            c.abort(pid)
                        c.accumulateCalls(pid, off, idx)
                        c.commit(pid)
            for c in ctxs:
                c.gatherGram()                   # closing barrier only: the bands stay where they are
            for c in ctxs:
                c.finalizeGram()
            _check_bands(ctxs, bands, S)
            for r, c in enumerate(ctxs):
                st = c.stats()
                assert st["variants_accumulated"] == sent[r]
                if edge == "stream-K":
                    assert st["gram_resident"] == 0, st
            del bufs
    finally:
        _close(ctxs)


# ---- E: owner-computes bands (no peers) -------------------------------------------------------------------------
@pytest.mark.parametrize("world,n,dtype,cta_group", [
    (1, 257, "i8", 2), (2, 300, "bf16", 1), (3, 449, "e2m1", 2), (4, 1029, "i8", 1),
    (5, 334, "bf16", 2), (6, 900, "e2m1", 1), (7, 455, "i8", 2), (8, 1500, "bf16", 1)],
    ids=["w1-n257-i8-cg2", "w2-n300-bf16-cg1", "w3-n449-e2m1-cg2", "w4-n1029-i8-cg1", "w5-n334-bf16-cg2",
         "w6-n900-e2m1-cg1", "w7-n455-i8-cg2", "w8-n1500-bf16-cg1"])
def test_owner_computes_bands_from_panels_and_staged_partitions(oracle, monkeypatch, world, n, dtype, cta_group):
    """Band-only contexts without peers: every context is fed ALL variants and computes only the tiles of its own rows.
    Pass 0 feeds device panels; pass 1 (after reset, another cohort) feeds staged partitions, one written, aborted and
    retried, and commits them into the band.  A direct host call (partition_id -1) is refused and changes nothing."""
    from spark_examples_b200 import native
    _env(monkeypatch, cta_group)
    dt = {"i8": native.DTYPE_I8, "bf16": native.DTYPE_BF16, "e2m1": native.DTYPE_E2M1}[dtype]
    nv = 2048
    devs = _devices(world)
    bands = native.ownerRowBands(n, world)
    ctxs = []
    try:
        for r in range(world):
            ctxs.append(native.NativePca(n, device=devs[r], dtype=dt, gram_band=bands[r], **CHUNK))
        for feed, v0 in zip(("panels", "staged"), COHORTS):
            S = _gram(oracle, n, v0, nv)
            X = _cells(oracle, n, v0, nv)
            _begin(ctxs)
            for r, c in enumerate(ctxs):
                if feed == "panels":
                    buf = _panels(c, devs[r], v0, nv)
                    c.accumulatePanels(buf.data_ptr(), nv, P)
                    c.synchronize()
                    del buf
                else:
                    sent = 0
                    for pid, (lo, hi) in enumerate(_shards(nv, 2)):
                        off, idx = _calls(X[:, lo:hi])
                        sent += len(off) - 1
                        if pid == 1:
                            c.accumulateCalls(pid, off, idx)
                            c.abort(pid)
                        c.accumulateCalls(pid, off, idx)
                        c.commit(pid)
                    if c.n != bands[r][1]:                               # world 1: the band is the whole matrix
                        off, idx = _calls(X[:, :64])
                        with pytest.raises(native.VpcaError) as ei:
                            c.accumulateCalls(-1, off, idx)
                        assert ei.value.code == native.VPCA_ERR_STATE
                assert c.stats()["variants_accumulated"] == (nv if feed == "panels" else sent)
            for c in ctxs:
                c.finalizeGram()
            _check_bands(ctxs, bands, S)
            for c in ctxs:
                assert c.stats()["gram_cta_group"] == cta_group
    finally:
        _close(ctxs)


# ---- G: arguments -----------------------------------------------------------------------------------------------
def test_owner_rows_needs_64_rows_per_rank_and_replicate_still_works(oracle):
    """n < 64 x world: owner-rows mode is refused with VPCA_ERR_UNSUPPORTED, and the wired contexts still reduce
    exactly in replicate mode."""
    from spark_examples_b200 import native
    world, n, nv = 3, 191, 1024
    devs = _devices(world)
    L = native.load_library()
    ctxs = []
    try:
        for r in range(world):
            ctxs.append(native.NativePca(n, device=devs[r]))
        with pytest.raises(native.VpcaError) as ei:
            native.setPeersLocal(ctxs, "owner_rows")
        assert ei.value.code == native.VPCA_ERR_UNSUPPORTED
        for c in ctxs:
            assert L.vpca_gram_set_peer_mode(c._h, 1) == native.VPCA_ERR_UNSUPPORTED
            assert L.vpca_gram_set_peer_mode(c._h, 0) == native.VPCA_OK
        S = _gram(oracle, n, 0, nv)
        shards = _shards(nv, world)
        bufs = [_panels(c, devs[r], shards[r][0], shards[r][1] - shards[r][0]) for r, c in enumerate(ctxs)]
        _begin(ctxs)
        for r, c in enumerate(ctxs):
            c.accumulatePanels(bufs[r].data_ptr(), shards[r][1] - shards[r][0], P)
        _check_routing(ctxs, S, "replicate")
        _finish_full(ctxs, S)
    finally:
        _close(ctxs)
