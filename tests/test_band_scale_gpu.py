"""Row-band Grams at 100 000 samples, the size they exist for: a 40 GB int32 Gram held as bands (DESIGN §5).

At N = 100 000 the cell offsets of a band pass 2^31 at its row 21 475 and 2^32 at its row 42 950; band 0 of 4 owner row
bands holds 50 016 rows (5.0e9 cells), band 0 of 2 holds 70 720 rows (7.1e9 cells), and the virtual origin
d_S - own_lo * N through which the Gram kernel addresses band 3 of 4 lies 8.7e9 cells below its allocation.  The cohort is
2048 structured variants (eig_ref.structured_cells, 8 populations) with cells in {0, 1, 2}, fed as device panels.

Cells (test_band_cells_are_exact_at_100k): every cell of every band, read back with vpca_get_gram_band in blocks of 1024
rows, equals X X^T of the same cells in FP64 on the GPU.  That reference is exact: every product and every partial sum is
an integer below 2048 * 2^2 < 2^53.  In band contexts the cells above the diagonal are never written and must stay zero;
the full context (world 1) is checked after finalizeGram in both triangles, which symmetrize_kernel mirrors.  owner-flush
(a variant shard per rank, flushed into the owner's band) and owner-computes (every variant per rank, only its own tiles)
must both give these exact bits.

Centring past 2^63 (test_band_centring_with_counts_near_2_31): the same cohort plus V_fill = 131 072 filler variants whose
every cell is 127 adds exactly 16129 * V_fill = 2 114 060 288 (0.984 * 2^31) to every cell; the guard's bound
(2048 + V_fill) * 127^2 = 2 147 092 480 stays below 2^31 - 1, and the sum of all cells passes 2^64, so matrix_mean_kernel's
128-bit total needs more than one shift in i128_to_double_rn.  J S J is unchanged by a constant, so the band solve must
give the principal coordinates of the structured cells alone: against the FP64 eigh of (JX)^T (JX) the eigenvalues agree to
1e-9 relative and the vectors to 1e-6, as at 70 000 samples in test_pca_bands_gpu.py, and both agree with the solve of the
same contexts without the filler.

What the filler costs in FP64: the band mat-vec evaluates S v with S = S_x + c 1 1^T, whose norm is c N = 2.1e14, and the
centring cancels the constant afterwards.  A rounding error of eps * ||S|| = 2.3e-2 is 1.2e-8 of lambda_1 = 2.0e6, which
is what the solves show: residuals ||C u - lambda u|| / lambda_1 of 1.5e-8 - 1.9e-8 with the filler (6e-15 without),
eigenvalues within 2.1e-10 and vectors within 5.5e-8 of the reference.  So the bars hold with a margin of 5 and 18.

Where the mean enters: the band operator is (C v)_i = (S v)_i - rbar_i sum(v) - rbar . v + mean sum(v), so a wrong mean
m' adds (m' - m) 1 1^T, which moves only the eigenvalue of the constant vector (0 for C) to (m' - m) N.  A mean too large
by a factor 2 (a wrong scale in i128_to_double_rn) puts that eigenvalue at 2.1e14, on top of the spectrum, and these tests
fail; a total summed in 64 bits wraps by -2^64, lowers it to -1.8e14 and leaves every top eigenpair as it was: no output
of the band solve shows it.

Host (staged) input is out of scope at this size: its N x N staging Gram would be another 40 GB.  Every context lives on
cuda:0, so one 80 GB H100 runs the whole file; the layouts are built and closed one after another."""
import numpy as np
import pytest

from eig_ref import P, Reference, close_all, compute_pca_bands, panel_buffer, structured_cells

pytestmark = pytest.mark.gpu

N = 100_000
NV = 2048
POPS = 8
COHORT_SEED = 20261017
BLOCK = 1024                         # rows per read-back: 400 MB of int32
FILL = 127
FILL_PANELS = 32                     # one filler buffer of 32 panels (3.3 GB) ...
FILL_FEEDS = 4                       # ... fed four times
V_FILL = FILL_PANELS * P * FILL_FEEDS
GIB = 2 ** 30
NEED = 52 * GIB                      # 40 GB of bands, 3.3 GB of filler, the FP64 cells and JX, read-back blocks, solver

LAYOUTS = {"computes-4": ("computes", 4), "computes-2": ("computes", 2), "flush-4": ("flush", 4), "full-1": ("full", 1)}


@pytest.fixture(scope="module")
def cohort():
    import torch
    torch.cuda.empty_cache()
    free, _ = torch.cuda.mem_get_info(0)
    if free < NEED:
        pytest.skip(f"needs {NEED / GIB:.0f} GiB of free HBM on cuda:0 for a 100 000-sample Gram, has {free / GIB:.1f} GiB: "
                    f"{(NEED - free) / GIB:.1f} GiB short")
    X = structured_cells(N, NV, POPS, COHORT_SEED)
    rng = np.random.default_rng(COHORT_SEED + 1)
    X += X & (rng.random((N, NV), dtype=np.float32) < 0.35).astype(np.int8)          # a third of the carriers: dosage 2
    Xd = torch.from_numpy(X).to("cuda:0").to(torch.float64)
    colsum = X.sum(axis=0, dtype=np.int64)
    out = {"X": X, "buf": panel_buffer(X), "Xd": Xd, "sq": (Xd * Xd).sum(dim=1),
           "sum_S": int(colsum @ colsum)}                                              # sum of all cells of X X^T
    torch.cuda.synchronize()
    yield out
    out.clear()
    torch.cuda.empty_cache()


@pytest.fixture(scope="module")
def ref(cohort):
    return Reference(cohort["Xd"], 5)


def _bands(form, world):
    from spark_examples_b200 import native
    return [(0, N)] if form == "full" else native.ownerRowBands(N, world)


def _contexts(form, world, max_mult):
    from spark_examples_b200 import native
    ctxs = []
    try:
        for band in _bands(form, world):
            ctxs.append(native.NativePca(N, device=0, max_multiplicity=max_mult, num_pc=5,
                                         gram_band=None if form == "full" else band))
        if form == "flush":
            native.setPeersLocal(ctxs, "owner_rows")
        return ctxs
    except Exception:
        close_all(ctxs)
        raise


def _accumulate(ctxs, form, feeds):
    """Reset the contexts, feed rank r the (panel buffer, variants) pairs feeds[r], close the owner-flush reduction and
    finalize"""
    import torch
    torch.cuda.synchronize()                      # the panels are written before any context stream reads them
    for c in ctxs:
        c.reset()
    for c in ctxs:
        c.synchronize()                           # every band is zero before any rank adds into it
    for c, feed in zip(ctxs, feeds):
        for buf, nv in feed:
            c.accumulatePanels(buf.data_ptr(), nv, P)
    if form == "flush":
        for c in ctxs:
            c.gatherGram()
    for c in ctxs:
        c.synchronize()
    for c in ctxs:
        c.finalizeGram()


def _row_blocks(bands, every, seed):
    """[r0, r1) blocks of at most BLOCK rows per band: all its rows, or (every=False) its first and last 512 rows (both
    sides of every band boundary), rows 21 000 - 43 500 of band 0 (cell offsets 2^31 and 2^32) and 8 seeded 64-row runs"""
    rng = np.random.default_rng(seed)
    for q, (row0, rows) in enumerate(bands):
        end = row0 + rows
        if every:
            sel = [(row0, end)]
        else:
            sel = [(row0, min(end, row0 + 512)), (max(row0, end - 512), end)]
            if q == 0:
                sel.append((min(end, 21_000), min(end, 43_500)))
            sel += [(int(r), min(end, int(r) + 64)) for r in rng.integers(row0, end, 8)]
        sel.sort()
        merged = []
        for a, b in sel:
            if merged and a <= merged[-1][1]:
                merged[-1][1] = max(merged[-1][1], b)
            elif b > a:
                merged.append([a, b])
        for a, b in merged:
            for r0 in range(a, b, BLOCK):
                yield q, r0, min(b, r0 + BLOCK)


def _check_cells(ctxs, form, cohort, every, extra=0, seed=0):
    """The band cells against X X^T (+ extra) in FP64, on cuda:0; returns the number of rows checked"""
    import torch
    Xd, sq = cohort["Xd"], cohort["sq"]
    bands = _bands(form, len(ctxs))
    pinned = torch.empty((BLOCK, N), dtype=torch.int32, pin_memory=True)
    cols = torch.arange(N, device="cuda:0")
    checked = 0
    for q, r0, r1 in _row_blocks(bands, every, seed):
        m = r1 - r0
        c = ctxs[q]
        c._check(c._lib.vpca_get_gram_band(c._h, r0, m, pinned.data_ptr()))
        got = pinned[:m].to("cuda:0").to(torch.float64)
        want = Xd[r0:r1] @ Xd.t()
        want += extra
        rows = torch.arange(r0, r1, device="cuda:0")
        if form != "full":
            want.masked_fill_(cols[None, :] > rows[:, None], 0.0)      # above the diagonal: never written
        diag = got[torch.arange(m, device="cuda:0"), rows]
        assert torch.equal(diag, sq[r0:r1] + extra), f"band {q}: diagonal of rows [{r0}, {r1}) is not sum c^2"
        if not torch.equal(got, want):
            bad = (got != want).nonzero()
            i, j = int(bad[0, 0]), int(bad[0, 1])
            raise AssertionError(f"{form}: band {q} rows [{r0}, {r1}): {bad.shape[0]} cells differ, first S[{r0 + i}][{j}] "
                                 f"= {int(got[i, j])}, want {int(want[i, j])}")
        checked += m
    return checked


@pytest.mark.parametrize("layout", list(LAYOUTS))
def test_band_cells_are_exact_at_100k(cohort, layout):
    """Every cell of the 100 000-sample Gram in each band layout, bit for bit; owner-computes at world 4 is the geometry in
    which band 0 passes 2^32 cells and band 3's virtual origin lies 8.7e9 cells below its allocation."""
    form, world = LAYOUTS[layout]
    bands = _bands(form, world)
    if layout == "computes-4":
        assert bands[0][1] * N > 2 ** 32 and bands[3][0] * N > 2 ** 33, bands
    if layout == "computes-2":
        assert bands[0][1] * N > 7 * 10 ** 9, bands
    if form == "flush":              # a contiguous shard of 512 variants per rank, in panels of its own
        shards = [np.ascontiguousarray(cohort["X"][:, r * NV // world:(r + 1) * NV // world]) for r in range(world)]
        feeds = [[(panel_buffer(s), s.shape[1])] for s in shards]
    else:
        feeds = [[(cohort["buf"], NV)]] * world
    ctxs = _contexts(form, world, 2)
    try:
        _accumulate(ctxs, form, feeds)
        assert _check_cells(ctxs, form, cohort, every=True) == N
    finally:
        close_all(ctxs)


def _check_solve(s, ref, k):
    from oracle import oracle
    assert s.method == 4, s
    assert s.nz == N == ref.nz
    assert s.vecs.shape == (N, k) and s.evals.shape == (k,)
    assert np.allclose(s.evals, ref.lam[:k], rtol=1e-9, atol=0), (s.evals, ref.lam[:k])
    err = oracle.eigvec_rel_err(s.vecs, ref.U[:, :k])
    assert np.all(err <= 1e-6), err
    assert np.allclose(np.linalg.norm(s.vecs, axis=0), 1.0, atol=1e-12)
    for c in range(k):
        assert s.vecs[np.argmax(np.abs(s.vecs[:, c])), c] > 0          # sign rule: largest-|.| entry positive
    # reported, not asserted: with the filler it is set by eps * ||S|| / lambda_1 ~ 1e-8 (see the module docstring), a
    # property of FP64 on a Gram whose constant part is 1e8 times lambda_1, not of the solver
    res = ref.residuals(s.vecs, s.evals)
    return float(np.max(np.abs(s.evals / ref.lam[:k] - 1))), float(err.max()), float(res.max())


@pytest.mark.parametrize("layout", ["computes-4", "full-1"])
def test_band_centring_with_counts_near_2_31(cohort, ref, layout):
    """Structured cells plus a constant 127-cell filler: cells near 2^31, a cell total past 2^64; the band solve must
    return the structured cohort's principal coordinates, as it does without the filler."""
    import torch
    from oracle import oracle
    form, world = LAYOUTS[layout]
    const = FILL * FILL * V_FILL
    assert float(cohort["sq"].max()) + const > 0.98 * 2 ** 31
    assert (NV + V_FILL) * FILL * FILL <= 2 ** 31 - 1                  # check_overflow's bound with max_multiplicity 127
    assert cohort["sum_S"] + N * N * const > 2 ** 64
    ctxs = _contexts(form, world, FILL)
    try:
        _accumulate(ctxs, form, [[(cohort["buf"], NV)]] * world)
        plain = {k: compute_pca_bands(ctxs, k) for k in (2, 5)}
        for k, s in plain.items():
            margins = _check_solve(s, ref, k)
            print(f"{layout} k={k} without the filler: max |lambda / lambda_ref - 1| {margins[0]:.2e}, vectors "
                  f"{margins[1]:.2e}, residual / lambda_1 {margins[2]:.2e}")
        fill = torch.full((FILL_PANELS * N * P,), FILL, dtype=torch.uint8, device="cuda:0")
        _accumulate(ctxs, form, [[(cohort["buf"], NV)] + [(fill, FILL_PANELS * P)] * FILL_FEEDS] * world)
        del fill
        assert _check_cells(ctxs, form, cohort, every=False, extra=const, seed=COHORT_SEED) > 22_500
        for k in (2, 5):
            s = compute_pca_bands(ctxs, k)
            margins = _check_solve(s, ref, k)
            print(f"{layout} k={k}: max |lambda / lambda_ref - 1| {margins[0]:.2e}, vectors {margins[1]:.2e}, "
                  f"residual / lambda_1 {margins[2]:.2e}")
            assert np.allclose(s.evals, plain[k].evals, rtol=1e-9, atol=0), (s.evals, plain[k].evals)
            assert np.all(oracle.eigvec_rel_err(s.vecs, plain[k].vecs) <= 1e-6)
    finally:
        close_all(ctxs)
        torch.cuda.empty_cache()
