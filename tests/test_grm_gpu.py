"""The variance-standardized relationship matrix on the GPU (vpca_grm_*, vpca_compute_pca_grm; DESIGN.md 13): the GRM
against an FP64 reference (numpy up to 2504 samples, torch float64 above) within the bound of DESIGN.md 13, M exact, its
bits independent of the split of the rows, skipped variants, the counted allele and padding, the staging chunks at their
row caps, its PCs on every solver path and FP64 band-tile layout against the small eigh of Z^T Z, the state rules and
refusals, and the driver end to end."""
import numpy as np
import pytest

import grm_ref
from spark_examples_b200 import native, plink, variants_pca

pytestmark = pytest.mark.gpu

KC = 1024   # kGrmPanelK: used variants per panel


def _bits(a):
    return np.ascontiguousarray(a, np.float64).view(np.int64)


def _run(n, rows, splits=None, num_pc=2):
    with native.NativePca(n, num_pc=num_pc) as nat:
        if splits is None:
            nat.grmBed(rows)
        else:
            for lo, hi in zip([0] + splits, splits + [rows.shape[0]]):
                nat.grmBed(rows[lo:hi])
        m = nat.grmFinalize()
        return nat.getGrm(), m


def _cohort(seed, n, nv, miss=0.01, pops=3):
    rng = np.random.default_rng(seed)
    return grm_ref.pack(grm_ref.balding_nichols(rng, n, nv, pops=pops, miss=miss))


def _check(G, rows, n):
    want, M, Z = grm_ref.grm(rows, n)
    tol = grm_ref.tolerance(Z)
    err = np.abs(G - want)
    assert np.all(err <= tol), f"max err {err.max():.3e}, max |G| {np.abs(want).max():.3e}"
    assert np.array_equal(_bits(G), _bits(G.T))
    return M


# ---- 1. the GRM against the FP64 reference ------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [2, 3, 63, 64, 65, 127, 128, 129, 1000])
@pytest.mark.parametrize("nv", [1, 15, 16, 17, KC - 1, KC + 1])
def test_grm_matches_reference(n, nv):
    rows = _cohort(1000 * n + nv, n, nv, miss=0.01)
    G, m = _run(n, rows)
    assert m == _check(G, rows, n)


@pytest.mark.parametrize("miss", [0.0, 0.5])
@pytest.mark.parametrize("n", [65, 1000])
def test_grm_missing_rates_and_an_uncalled_sample(n, miss):
    rng = np.random.default_rng(n)
    code = grm_ref.balding_nichols(rng, n, 3 * KC + 7, miss=miss)
    code[:, n // 2] = 1   # a sample with no call
    rows = grm_ref.pack(code)
    G, m = _run(n, rows)
    assert m == _check(G, rows, n)
    assert not G[n // 2].any() and not G[:, n // 2].any()


def test_grm_2504_over_several_chunks():
    """2504 samples: 110 000 rows of 626 bytes pass one 64 MB staging chunk."""
    n = 2504
    rows = _cohort(7, n, 110_000)
    G, m = _run(n, rows)
    assert m == _check(G, rows, n)


def test_grm_many_chunks_through_a_wide_stride():
    """Rows 1 MB apart: 64 rows per staged chunk, so 300 rows take five chunks; the junk bytes are ignored."""
    n, nv, stride = 200, 300, 1 << 20
    rows = _cohort(9, n, nv)
    wide = np.random.default_rng(3).integers(0, 256, (nv, stride), dtype=np.uint8)
    wide[:, :rows.shape[1]] = rows
    G, m = _run(n, wide)
    G0, m0 = _run(n, rows)
    assert m == m0 and np.array_equal(_bits(G), _bits(G0))
    _check(G, rows, n)


def _bed_launches(used, stride, fill=0):
    """kernel_launches of one grmBed call (vpca_grm_bed), restated: rows are staged in chunks of min(64 MB / stride, 2^20)
    rows, at least one; each chunk takes 3 (counts, tables, compaction), then one per expand of its used columns into the
    panel (an expand stops where the panel fills) and one per full panel (the SYRK).  -> (launches, chunks)"""
    nv = len(used)
    step = max(1, min(nv, (64 << 20) // stride, 1 << 20))
    launches = 0
    for lo in range(0, nv, step):
        u, j = int(used[lo:lo + step].sum()), 0
        launches += 3
        while j < u:
            cnt = min(KC - fill, u - j)
            launches += 1
            fill, j = fill + cnt, j + cnt
            if fill == KC:
                launches, fill = launches + 1, 0
    return launches, -(-nv // step)


def _run_counted(n, rows):
    """_run with the kernel_launches of the grmBed call"""
    with native.NativePca(n) as nat:
        before = nat.stats()["kernel_launches"]
        nat.grmBed(rows)
        launches = nat.stats()["kernel_launches"] - before
        m = nat.grmFinalize()
        return nat.getGrm(), m, launches


@pytest.mark.parametrize("n,extra", [(64, 1500), (253, 700)], ids=["row-cap-64", "both-caps-253"])
def test_grm_chunks_at_the_row_cap(n, extra):
    """2^20 + extra rows in one call: a staged chunk holds at most kGrmMaxChunk = 2^20 rows, which grm_compact_kernel scans
    1024 per thread.  At N = 64 (16-byte rows) that cap binds alone; at N = 253 (64-byte rows) 64 MB is 2^20 rows, so the
    staging cap binds at the same count.  The first chunk is 2^20 rows and about 1000 panels are multiplied in turn."""
    rows = _cohort(40 + n, n, (1 << 20) + extra)
    G, m, launches = _run_counted(n, rows)
    _, used = grm_ref.z_tables(grm_ref.counts(rows, n))
    want, chunks = _bed_launches(used, rows.shape[1])
    assert chunks == 2 and launches == want, (launches, want)
    assert m == int(used.sum()) > 1000 * KC
    assert m == _check(G, rows, n)


def test_grm_one_row_chunks():
    """Rows 64 MiB + 32 bytes apart: not one whole row fits the 64 MB staging chunk, so every chunk is a single row
    (step = 1); one of the five rows is monomorphic and uses no column.  The bits are those of the packed rows."""
    n, nv, stride = 100, 5, (64 << 20) + 32
    rows = _cohort(43, n, nv)
    rows[3] = 0xFF                                          # every call HOM_A2: monomorphic
    wide = np.full((nv, stride), 0x5A, np.uint8)            # junk past the row's 25 bytes
    wide[:, :rows.shape[1]] = rows
    G, m, launches = _run_counted(n, wide)
    _, used = grm_ref.z_tables(grm_ref.counts(rows, n))
    assert int(used.sum()) == nv - 1 and not used[3]
    assert (launches, nv) == _bed_launches(used, stride) == (3 * nv + nv - 1, nv)
    G0, m0 = _run(n, rows)
    assert m == m0 == nv - 1 and np.array_equal(_bits(G), _bits(G0))
    _check(G, rows, n)


def test_grm_21845_against_torch():
    torch = pytest.importorskip("torch")
    n, nv = 21845, 1500
    rows = _cohort(11, n, nv)
    G, m = _run(n, rows)
    tab, used = grm_ref.z_tables(grm_ref.counts(rows, n))
    assert m == int(used.sum())
    dev = torch.device("cuda")
    code = torch.from_numpy(grm_ref.codes(rows, n).astype(np.int64)).to(dev)
    Zt = torch.gather(torch.from_numpy(tab).to(dev), 1, code)[torch.from_numpy(used).to(dev)]   # (M, n)
    want = (Zt.T @ Zt) / m
    A = Zt.abs()
    depth = KC + -(-m // KC) + 2 * (256 + -(-m // 256)) + 4
    tol = depth * 2.0 ** -53 * (A.T @ A) / m
    Gd = torch.from_numpy(G).to(dev)
    assert bool(((Gd - want).abs() <= tol).all())
    assert bool((Gd == Gd.T).all())


def test_grm_counts_used_variants_exactly():
    n = 40
    rng = np.random.default_rng(5)
    code = grm_ref.balding_nichols(rng, n, 60)
    code[3] = 0                 # monomorphic HOM_A1
    code[4] = 3                 # monomorphic HOM_A2
    code[5] = 1                 # nothing called
    code[6] = 2                 # all het: a = n, used
    code[7, :] = 1
    code[7, 0] = 0              # one called sample, homozygous: skipped
    rows = grm_ref.pack(code)
    G, m = _run(n, rows)
    _, used = grm_ref.z_matrix(rows, n)
    assert not used[[3, 4, 5, 7]].any() and used[6]
    assert m == int(used.sum()) == _check(G, rows, n)


# ---- 2. bit identity ---------------------------------------------------------------------------------------------------
def test_grm_bits_do_not_depend_on_splits_skips_allele_or_padding():
    n = 130
    rng = np.random.default_rng(17)
    code = grm_ref.balding_nichols(rng, n, 2 * KC + 300, miss=0.01)
    rows = grm_ref.pack(code)
    G, m = _run(n, rows)
    G2, _ = _run(n, rows)
    assert np.array_equal(_bits(G), _bits(G2))                                       # two runs
    splits = sorted(rng.choice(np.arange(1, rows.shape[0]), 9, replace=False).tolist())
    assert np.array_equal(_bits(_run(n, rows, splits)[0]), _bits(G))                # arbitrary splits
    skip = np.zeros((40, n), np.uint8)                                               # monomorphic / uncalled rows
    skip[::3] = 1
    skip[1::3] = 3
    pos = np.sort(rng.choice(np.arange(rows.shape[0] + 1), 40))
    mixed = grm_ref.pack(np.insert(code, pos, skip, axis=0))
    Gm, mm = _run(n, mixed, [5, 700, 1500])
    assert mm == m and np.array_equal(_bits(Gm), _bits(G))
    flip = {0: 3, 3: 0, 1: 1, 2: 2}                                                  # A2 counted instead of A1
    lut = np.array([flip[c] for c in range(4)], np.uint8)
    assert np.array_equal(_bits(_run(n, grm_ref.pack(lut[code]))[0]), _bits(G))
    some = code.copy()
    sel = rng.random(code.shape[0]) < 0.5
    some[sel] = lut[code[sel]]
    assert np.array_equal(_bits(_run(n, grm_ref.pack(some))[0]), _bits(G))
    padded = np.concatenate([rows, rng.integers(0, 256, (rows.shape[0], 5), dtype=np.uint8)], axis=1)
    padded[:, rows.shape[1] - 1] |= np.uint8(0xF0)                                   # garbage in the padding bits (n % 4 = 2)
    Gp, mp = _run(n, padded)
    assert mp == m and np.array_equal(_bits(Gp), _bits(G))


def test_grm_table_bits_match_the_host_restatement():
    """One used variant at a tie (HOM_A1, HET, HOM_A2 = 1, 3, 1: a = n = 5) and a missing call: G = z z^T with every z
    bit that of the Python-float table."""
    n = 6
    code = np.array([[0, 2, 3, 1, 2, 2]], np.uint8)
    rows = grm_ref.pack(code)
    G, m = _run(n, rows)
    t = grm_ref.z_table(1, 3, 1)
    z = np.array([t[c] for c in code[0]])
    assert m == 1 and np.array_equal(_bits(G), _bits(np.outer(z, z) / 1 + 0.0))   # the sum starts at +0


# ---- 3. PCs against numpy.linalg.eigh ----------------------------------------------------------------------------------
def _pcs_check(vecs, evals, G, k):
    w, V = np.linalg.eigh(G)
    w, V = w[::-1][:k], V[:, ::-1][:, :k]
    assert np.all(np.abs(evals - w) <= 1e-10 * w[0])
    for c in range(k):
        v = V[:, c] * np.sign(V[:, c] @ vecs[:, c])
        assert np.abs(vecs[:, c] - v).max() <= 1e-6, c


DIRECT, LANCZOS, MAXIT16 = {"VPCA_EIG": "direct"}, {"VPCA_EIG": "lanczos"}, {"VPCA_EIG_MAXIT": "16"}
# The FP64 band tiles (kBandTR = 64 rows x kBandTC = 1024 columns): N mod 4 picks the vector or the scalar loads, N past
# 1024 and 2048 a second and third column tile, N mod 64 a partial row tile.
BAND_N = [512, 513, 1023, 1024, 1025, 1026, 1027, 2047, 2048, 2049, 2503, 2504, 3001]
FORCED_N = [96, 97, 98, 99, 127, 128, 129, 255]   # VPCA_EIG=lanczos reaches down to kLzForcedMinN = 96


# pops: populations of the cohort; with k + 1 of them the top k eigenvalues stand apart.  The fallback cases ask for PCs
# 3 and 4 of three populations, which lie in the bulk, so Lanczos gives up within 16 steps.
@pytest.mark.parametrize("n,k,pops,nv,env", [
    (300, 1, 3, 4000, {}), (300, 10, 11, 4000, {}), (600, 2, 3, 4000, {}), (600, 16, 17, 4000, {}),
    (600, 20, 21, 4000, {}), (2504, 10, 11, 4000, DIRECT), (700, 4, 3, 4000, MAXIT16),
    *[(n, 4, 5, 3000, {}) for n in BAND_N], (511, 4, 5, 3000, {}), *[(n, 4, 5, 3000, LANCZOS) for n in FORCED_N],
    (3073, 4, 5, 3000, DIRECT), (3073, 4, 3, 3000, MAXIT16),
], ids=["direct-300-k1", "direct-300-k10", "lanczos-600-k2", "lanczos-600-k16", "lanczos-600-k20", "direct-2504",
        "fallback-700", *[f"lanczos-{n}" for n in BAND_N], "direct-511", *[f"forced-lanczos-{n}" for n in FORCED_N],
        "direct-two-kernels-3073", "fallback-3073"])
def test_grm_pcs(monkeypatch, n, k, pops, nv, env):
    """Every solver path a GRM reaches, against the small eigh of Z^T Z (never the device's own G).  Lanczos on a GRM is
    always the band solver on FP64 cells; its tile kernel reads four cells as two double2 when N mod 4 = 0 (d_C is a
    256-byte-aligned allocation, so every row then starts 32-byte aligned) and one double at a time otherwise."""
    for key, val in env.items():
        monkeypatch.setenv(key, val)
    rows = _cohort(n + k, n, nv, pops=pops)
    with native.NativePca(n, num_pc=max(k, 2)) as nat:
        nat.grmBed(rows)
        nat.grmFinalize()
        s = grm_ref.Solve(nat, k)
    method = 1 if env is DIRECT or (n < 512 and env is not LANCZOS) else 3 if env is MAXIT16 else 2
    grm_ref.assert_path(s, method, n)
    Z, _ = grm_ref.z_matrix(rows, n)
    grm_ref.check_grm_pairs(grm_ref.Pcs(Z, k), s.vecs, s.evals, k, note=repr(s))


# ---- 4. state rules and refusals ---------------------------------------------------------------------------------------
def test_grm_state_rules():
    n = 600
    rows = _cohort(21, n, 2000)
    with native.NativePca(n, num_pc=2) as nat:
        nat.accumulateBed(0, rows, 1)
        nat.commit(0)
        nat.finalizeGram()
        S = nat.getGram()
        nat.kinshipBed(rows[:300])
        kin = nat.kinshipPairs()
        with pytest.raises(native.VpcaError) as e:      # nothing finalized yet
            nat.getGrm()
        assert e.value.code == native.VPCA_ERR_STATE
        nat.grmBed(rows[:1000])
        nat.grmBed(rows[1000:])
        m = nat.grmFinalize()
        assert nat.grmFinalize() == m
        with pytest.raises(native.VpcaError) as e:
            nat.grmBed(rows[:1])
        assert e.value.code == native.VPCA_ERR_STATE
        assert np.array_equal(nat.getGram(), S)
        k2 = nat.kinshipPairs()
        assert all(np.array_equal(a, b) for a, b in zip(kin[:2], k2[:2])) and np.array_equal(_bits(kin[2]), _bits(k2[2]))
        G = nat.getGrm()
        nat.computePcaGrm(2)                                # Lanczos at 600: the GRM stays
        assert np.array_equal(_bits(nat.getGrm()), _bits(G))
        with pytest.raises(native.VpcaError) as e:          # a GRM solve leaves no U
            nat.loadingsBed(2, rows[:10])
        assert e.value.code == native.VPCA_ERR_STATE
        nat.computePca(2)                                   # the carrier solve may overwrite d_C
        for call in (nat.getGrm, lambda: nat.computePcaGrm(2), nat.grmFinalize, lambda: nat.grmBed(rows[:1])):
            with pytest.raises(native.VpcaError) as e:
                call()
            assert e.value.code == native.VPCA_ERR_STATE
        nat.reset()
        nat.grmBed(rows)
        assert nat.grmFinalize() == m
        assert np.array_equal(_bits(nat.getGrm()), _bits(G))


def test_grm_direct_solve_consumes_the_grm():
    n = 300
    rows = _cohort(23, n, 1500)
    with native.NativePca(n) as nat:
        nat.grmBed(rows)
        nat.grmFinalize()
        nat.computePcaGrm(2)
        with pytest.raises(native.VpcaError) as e:
            nat.getGrm()
        assert e.value.code == native.VPCA_ERR_STATE


def test_grm_refusals():
    n = 100
    rows = _cohort(25, n, 50)
    with native.NativePca(n) as nat:
        lib, h = nat._lib, nat._h
        assert lib.vpca_grm_bed(h, None, 5, 25) == native.VPCA_ERR_BAD_ARG
        assert lib.vpca_grm_bed(h, rows.ctypes.data, -1, 25) == native.VPCA_ERR_BAD_ARG
        assert lib.vpca_grm_bed(h, rows.ctypes.data, 5, 24) == native.VPCA_ERR_BAD_ARG
        assert lib.vpca_grm_bed(None, rows.ctypes.data, 5, 25) == native.VPCA_ERR_BAD_ARG
        assert lib.vpca_get_grm(h, None) == native.VPCA_ERR_BAD_ARG
        with pytest.raises(native.VpcaError) as e:
            nat.computePcaGrm(17)
        assert e.value.code == native.VPCA_ERR_BAD_ARG
        with pytest.raises(native.VpcaError) as e:
            nat.computePcaGrm(2)
        assert e.value.code == native.VPCA_ERR_STATE
        mono = np.zeros((3, 25), np.uint8)                 # M = 0
        nat.grmBed(mono)
        with pytest.raises(native.VpcaError) as e:
            nat.grmFinalize()
        assert e.value.code == native.VPCA_ERR_STATE
        with pytest.raises(native.VpcaError) as e:
            nat.grmBed(rows)
        assert e.value.code == native.VPCA_ERR_STATE
        nat.reset()
        nat.grmBed(rows)
        assert nat.grmFinalize() > 0
    with native.NativePca(65536) as nat:
        with pytest.raises(native.VpcaError) as e:
            nat.grmBed(np.zeros((1, 16384), np.uint8))
        assert e.value.code == native.VPCA_ERR_UNSUPPORTED


# ---- 5. the driver end to end ------------------------------------------------------------------------------------------
def _fileset(prefix, n, nv, seed):
    rng = np.random.default_rng(seed)
    code = grm_ref.balding_nichols(rng, n, nv, pops=4, miss=0.01)
    code[rng.random(nv) < 0.1] = 3                          # some monomorphic variants for --maf to drop
    d = np.select([code == 0, code == 2, code == 3], [2, 1, 0], -1).T
    plink.write_fileset(prefix, d, fam=[(f"F{i % 7}", f"I{i}") for i in range(n)])
    return d


def test_driver_filtered_run_equals_a_plain_run_on_the_filtered_fileset(tmp_path, capsys):
    n, nv = 700, 3000
    src = str(tmp_path / "src")
    d = _fileset(src, n, nv, 31)
    kept = [i for i in range(n) if i % 5 != 3]
    fam = [(f"F{i % 7}", f"I{i}") for i in kept]
    (tmp_path / "keep.id").write_text("".join(f"{f}\t{i}\n" for f, i in fam))
    P = str(tmp_path / "filt")
    variants_pca.main(["--bed-path", src, "--keep", str(tmp_path / "keep.id"), "--maf", "0.01", "--ld-prune", "0.2", "--grm",
           "--make-rel", "--num-pc", "4", "--output-path", P])
    got = capsys.readouterr().out
    bim = plink.read_bim(src)
    ids = {b.id: j for j, b in enumerate(bim)}
    keep_v = np.zeros(nv, bool)
    keep_v[[ids[x] for x in open(P + ".prune.in").read().split()]] = True
    assert 0 < keep_v.sum() < nv
    plain = str(tmp_path / "plain")
    plink.write_fileset(plain, d[kept][:, keep_v], fam=fam)
    Q = str(tmp_path / "plainout")
    variants_pca.main(["--bed-path", plain, "--grm", "--make-rel", "--num-pc", "4", "--output-path", Q])
    want = capsys.readouterr().out
    line = [ln for ln in got.splitlines() if ln.startswith("GRM: ")]
    assert len(line) == 1 and line == [ln for ln in want.splitlines() if ln.startswith("GRM: ")]
    assert f" of {int(keep_v.sum())} variants used" in line[0]
    for suffix in (".eigenvec", ".eigenval", ".rel.bin", ".rel.id"):
        assert open(P + suffix, "rb").read() == open(Q + suffix, "rb").read(), suffix
    G = np.fromfile(P + ".rel.bin", dtype="<f8").reshape(len(kept), len(kept))
    vecs = np.array([[float(x) for x in ln.split("\t")[2:]] for ln in open(P + ".eigenvec").read().splitlines()[1:]])
    evals = np.array([float(x) for x in open(P + ".eigenval").read().split()])
    _pcs_check(vecs, evals, G, 4)
    lines = {ln.split("\t")[0]: ln.split("\t") for ln in got.splitlines() if ln.count("\t") == 3}
    assert len(lines) == len(kept)


def test_driver_king_table_rides_along_unchanged(tmp_path, capsys):
    n, nv = 300, 800
    src = str(tmp_path / "src")
    _fileset(src, n, nv, 37)
    variants_pca.main(["--bed-path", src, "--make-king-table", str(tmp_path / "a.kin0")])
    variants_pca.main(["--bed-path", src, "--grm", "--make-king-table", str(tmp_path / "b.kin0"), "--output-path",
           str(tmp_path / "g")])
    capsys.readouterr()
    assert (tmp_path / "a.kin0").read_bytes() == (tmp_path / "b.kin0").read_bytes()
    assert (tmp_path / "g.eigenvec").exists()
