"""Sample QC on the GPU (vpca_sample_missing_bed, vpca_subset_bed_samples; DESIGN.md 11): per-sample missing counts
bit-exact against numpy from 2 to 100 000 samples (every N mod 32 around the word boundaries, padding garbage, wide
strides, all-missing and no-missing rows, staging-chunk and grid edges, any split of the rows), subset bytes against
numpy for many keep patterns, bad arguments, the state left alone, and the driver end to end against plain runs on a
fileset of the kept samples."""
import os

import numpy as np
import pytest

import sample_qc_ref
from kinship_ref import dosage_codes
from spark_examples_b200 import native, plink, variants_pca
from spark_examples_b200.conf import PcaConf
from spark_examples_b200.variants_pca import VariantsPcaDriver, check_ld_flags

pytestmark = pytest.mark.gpu

STAGE_BYTES = 64 << 20   # both calls stage this many row bytes per chunk


def _bits(a):
    return np.ascontiguousarray(a, np.float64).view(np.int64)


def _random_rows(rng, n, nv, extra=0):
    """Random bytes (every code, random padding bits, `extra` junk bytes past ceil(n / 4)); row 1 all missing, row 2 no
    missing call, when there are enough rows."""
    rows = rng.integers(0, 256, size=(nv, (n + 3) // 4 + extra), dtype=np.uint8)
    if nv >= 3:
        rows[1, :] = 0x55
        rows[2, :] = 0xFF
    return rows


def _check_missing(nat, rows, n):
    got = nat.sampleMissingBed(rows, n)
    assert got.dtype == np.int32 and got.shape == (n,)
    np.testing.assert_array_equal(got, sample_qc_ref.missing_counts(rows, n))
    return got


def test_missing_counts_are_exact():
    rng = np.random.default_rng(1)
    sizes = list(range(2, 100)) + [129, 1000, 2504, 100000]
    with native.NativePca(2) as nat:                                    # the rows' own n, whatever the context
        for n in sizes:
            nv = 37 if n < 1000 else 300 if n < 100000 else 64
            nb = (n + 3) // 4
            for extra in (0, 5, (-nb) % 4, (-nb) % 4 + 4):               # tight, odd and 4-byte-aligned strides
                rows = _random_rows(rng, n, nv, extra)
                got = _check_missing(nat, rows, n)
                assert got[0] <= nv and np.all(got >= 1)                # row 1 is all missing
            # any split of the rows into calls gives the same counts
            rows = _random_rows(rng, n, nv)
            whole = nat.sampleMissingBed(rows, n)
            parts = [nat.sampleMissingBed(rows[a:b], n) for a, b in ((0, 1), (1, 20), (20, nv))]
            np.testing.assert_array_equal(parts[0] + parts[1] + parts[2], whole)
        # all missing / nothing missing, and no rows at all
        for n in (2, 17, 1000):
            nb = (n + 3) // 4
            np.testing.assert_array_equal(nat.sampleMissingBed(np.full((300, nb), 0x55, np.uint8), n), np.full(n, 300))
            np.testing.assert_array_equal(nat.sampleMissingBed(np.full((300, nb), 0xAA, np.uint8), n), np.zeros(n))
            np.testing.assert_array_equal(nat.sampleMissingBed(np.zeros((0, nb), np.uint8), n), np.zeros(n))


@pytest.mark.parametrize("n", [2504, 100000])
def test_missing_counts_across_staging_chunks(n):
    rng = np.random.default_rng(7)
    stride = (n + 3) // 4
    per_chunk = STAGE_BYTES // stride
    with native.NativePca(2) as nat:
        for nv in (per_chunk - 1, per_chunk, per_chunk + 1, 2 * per_chunk + 3):
            _check_missing(nat, _random_rows(rng, n, nv), n)


def test_missing_counts_past_the_grid_rows():
    # 4 samples, one byte per row: a 64 MB chunk holds 9e6 rows, more slabs of 1020 rows than 8192 grid rows
    rng = np.random.default_rng(8)
    rows = rng.integers(0, 256, size=(9_000_000, 1), dtype=np.uint8)
    with native.NativePca(2) as nat:
        _check_missing(nat, rows, 4)
        _check_missing(nat, rows, 3)


def _patterns(rng, n):
    """name -> strictly increasing kept indices."""
    p = {"all": np.arange(n), "first": np.array([0]), "last": np.array([n - 1]), "single": np.array([n // 2]),
         "every_other": np.arange(0, n, 2), "odd": np.arange(1, n, 2),
         "runs": np.flatnonzero((np.arange(n) // max(1, n // 7)) % 2 == 0),
         "random10": np.flatnonzero(rng.random(n) < 0.1), "random90": np.flatnonzero(rng.random(n) < 0.9)}
    for r in range(4):                                                 # m mod 4 = 0..3
        m = max(1, min(n, (n // 2) - ((n // 2) % 4) + r))
        p[f"mod4_{r}"] = np.sort(rng.choice(n, size=m, replace=False))
    return {k: v for k, v in p.items() if len(v) >= 1}


def _check_subset(nat, rows, n, keep):
    got = nat.subsetBedSamples(rows, n, keep)
    want = sample_qc_ref.subset_rows(rows, n, keep)
    assert got.shape == want.shape == (rows.shape[0], (len(keep) + 3) // 4)
    np.testing.assert_array_equal(got, want)


@pytest.mark.parametrize("n", [2, 3, 5, 16, 17, 33, 64, 65, 129, 1000, 2504, 100000])
def test_subset_bytes_match_the_reference(n):
    rng = np.random.default_rng(100 + n)
    nv = 41 if n < 100000 else 24
    with native.NativePca(2) as nat:
        for extra in (0, 3):
            rows = _random_rows(rng, n, nv, extra)                      # garbage in the padding and past ceil(n / 4)
            for name, keep in _patterns(rng, n).items():
                _check_subset(nat, rows, n, keep)
        # the subset of a fileset's rows is that fileset's subset, padding bits zero
        keep = np.flatnonzero(rng.random(n) < 0.6)
        keep = keep if len(keep) else np.array([n - 1])
        d = rng.integers(-1, 3, size=(n, nv))
        full = sample_qc_ref._pack(dosage_codes(d))
        np.testing.assert_array_equal(nat.subsetBedSamples(full, n, keep), sample_qc_ref._pack(dosage_codes(d[keep])))


def test_subset_across_chunks_and_grid_rows():
    rng = np.random.default_rng(5)
    with native.NativePca(2) as nat:
        for n in (2504, 100000):
            per_chunk = STAGE_BYTES // ((n + 3) // 4)
            for nv in (per_chunk + 1, 2 * per_chunk + 1):                # two and three chunks: both buffers reused
                rows = _random_rows(rng, n, nv)
                _check_subset(nat, rows, n, np.flatnonzero(rng.random(n) < 0.9))
        # 16 samples: 600 000 rows, more slabs of 64 rows than 8192 grid rows
        rows = rng.integers(0, 256, size=(600_000, 4), dtype=np.uint8)
        _check_subset(nat, rows, 16, np.array([0, 3, 4, 9, 15]))


def test_subset_leaves_the_rest_of_a_wide_out_row():
    rng = np.random.default_rng(6)
    L = native.load_library()
    with native.NativePca(2) as nat:
        for n, m in ((10, 5), (37, 16), (2504, 2253), (100000, 90001)):
            nv = 30
            rows = _random_rows(rng, n, nv, 2)
            keep = np.sort(rng.choice(n, size=m, replace=False)).astype(np.int32)
            mb = (m + 3) // 4
            for wide in (mb + 1, mb + 7, mb + 64):
                out = np.full((nv, wide), 0xA5, np.uint8)
                assert L.vpca_subset_bed_samples(nat._h, rows.ctypes.data, nv, rows.shape[1], n, keep.ctypes.data, m,
                                                 out.ctypes.data, wide) == native.VPCA_OK
                np.testing.assert_array_equal(out[:, :mb], sample_qc_ref.subset_rows(rows, n, keep))
                assert np.all(out[:, mb:] == 0xA5)


def test_bad_arguments():
    L = native.load_library()
    n = 10
    rows = np.zeros((4, 3), np.uint8)
    with native.NativePca(2) as nat:
        out = np.full(n, -7, np.int32)

        def miss(r=rows.ctypes.data, nv=4, stride=3, nn=n, o=out.ctypes.data):
            return L.vpca_sample_missing_bed(nat._h, r, nv, stride, nn, o)
        for kw in ({"r": None}, {"o": None}, {"nv": -1}, {"nn": 0}, {"nn": -3}, {"stride": 2}):
            assert miss(**kw) == native.VPCA_ERR_BAD_ARG, kw
            assert np.all(out == -7)
        assert miss(nv=2 ** 31) == native.VPCA_ERR_OVERFLOW                # refused before any row is read
        assert np.all(out == -7)
        assert miss(r=None, nv=0) == native.VPCA_OK and np.all(out == 0)   # nv = 0: zeros
        assert miss(r=None, o=None, nv=0) == native.VPCA_OK
        assert miss() == native.VPCA_OK and np.all(out == 0)
        with pytest.raises(native.VpcaError):
            nat.sampleMissingBed(rows, 13)                                  # stride 3 < ceil(13 / 4)

        sub = np.full((4, 8), 0x5A, np.uint8)

        def subset(keep, m=None, r=rows.ctypes.data, nv=4, stride=3, nn=n, o=sub.ctypes.data, os_=8, null_keep=False):
            k = np.ascontiguousarray(keep, np.int32)
            return L.vpca_subset_bed_samples(nat._h, r, nv, stride, nn, None if null_keep else k.ctypes.data,
                                             len(k) if m is None else m, o, os_)
        bad = [dict(keep=[0, 2, 2]), dict(keep=[3, 1]), dict(keep=[-1, 2]), dict(keep=[0, 10]), dict(keep=[0], m=0),
               dict(keep=[0, 1, 2, 3, 4], os_=1), dict(keep=[0], r=None), dict(keep=[0], o=None),
               dict(keep=[0], null_keep=True), dict(keep=[0], nv=-1), dict(keep=[0], nn=0), dict(keep=[0], stride=2)]
        for kw in bad:
            assert subset(**kw) == native.VPCA_ERR_BAD_ARG, kw
            assert np.all(sub == 0x5A)
        assert subset([0], r=None, o=None, nv=0) == native.VPCA_OK
        assert subset([0, 1, 2, 3, 4]) == native.VPCA_OK                      # 2 bytes of each 8-byte out row
        assert np.all(sub[:, :2] == 0) and np.all(sub[:, 2:] == 0x5A)
        with pytest.raises(native.VpcaError):
            nat.subsetBedSamples(rows, n, [])


def _planted(rng, n, v, block=6, copy=0.85, missing=0.02):
    d = np.empty((n, v), np.int64)
    for b0 in range(0, v, block):
        founder = rng.binomial(2, rng.uniform(0.02, 0.5), size=n)
        for j in range(b0, min(v, b0 + block)):
            own = rng.binomial(2, rng.uniform(0.005, 0.5), size=n)
            d[:, j] = np.where(rng.random(n) < copy, founder, own)
    d[rng.random((n, v)) < missing] = -1
    return d


def test_leaves_gram_kinship_and_ld_alone():
    rng = np.random.default_rng(14)
    n, v = 150, 900
    rows = sample_qc_ref._pack(dosage_codes(_planted(rng, n, v)))
    other = _random_rows(rng, 1000, 200)
    lo = np.maximum(0, np.arange(v) - 50)
    with native.NativePca(n, num_pc=3) as nat:
        nat.kinshipBed(rows)
        nat.accumulateBed(0, rows, plink.COUNT_A1)
        nat.commit(0)
        nat.finalizeGram()
        nat.computePca(3)
        S0, (ids0, c0, k0) = nat.getGram(), nat.kinshipPairs()
        w0, _ = nat.loadingsBed(3, rows, plink.COUNT_A1)
        ld0 = nat.ldPruneBed(rows, lo, 0.2, max_pairs=10 ** 6)
        q0, p0 = nat.variantQcBed(rows)
        m1 = nat.sampleMissingBed(rows, n)
        s1 = nat.subsetBedSamples(rows, n, np.arange(0, n, 3))
        nat.sampleMissingBed(other, 1000)                                   # rows of another sample count
        nat.subsetBedSamples(other, 1000, np.arange(5, 1000, 2))
        S1, (ids1, c_1, k1) = nat.getGram(), nat.kinshipPairs()
        w1, _ = nat.loadingsBed(3, rows, plink.COUNT_A1)
        ld1 = nat.ldPruneBed(rows, lo, 0.2, max_pairs=10 ** 6)
        q1, p1 = nat.variantQcBed(rows)
    np.testing.assert_array_equal(m1, sample_qc_ref.missing_counts(rows, n))
    np.testing.assert_array_equal(s1, sample_qc_ref.subset_rows(rows, n, np.arange(0, n, 3)))
    np.testing.assert_array_equal(S0, S1)
    np.testing.assert_array_equal(ids0, ids1)
    np.testing.assert_array_equal(c0, c_1)
    np.testing.assert_array_equal(_bits(k0), _bits(k1))
    np.testing.assert_array_equal(_bits(w0), _bits(w1))
    for a, b in zip(ld0, ld1):
        np.testing.assert_array_equal(a, b)
    np.testing.assert_array_equal(q0, q1)
    np.testing.assert_array_equal(_bits(p0), _bits(p1))


# ---- the driver, end to end ------------------------------------------------------------------------------------------
def _layout(rng, v, contigs=2):
    names = np.repeat([str(c + 1) for c in range(contigs)], -(-v // contigs))[:v].tolist()
    pos = np.maximum.accumulate(np.cumsum(rng.integers(200, 3000, size=v))) + 1
    return names, pos


def _cohort(tmp_path, rng, n=240, v=3000):
    d = _planted(rng, n, v, block=5)
    d[: n // 2] = np.where(d[: n // 2] >= 0, np.minimum(2, d[: n // 2] + (rng.random((n // 2, v)) < 0.2)), -1)
    for s, share in ((5, 0.3), (11, 0.12), (40, 0.06), (77, 0.2), (n - 40, 0.5)):   # samples with poor call rates
        d[s] = np.where(rng.random(v) < share, -1, d[s])
    d[7] = d[3]                                                                  # relatives for KING
    d[150] = np.where(rng.random(v) < 0.5, d[151], d[150])
    contigs, pos = _layout(rng, v)
    fam = [(f"F{i % 5}", f"S{i:03d}") for i in range(n)]
    prefix = str(tmp_path / "all")
    plink.write_fileset(prefix, d, fam=fam, contigs=contigs, positions=pos)
    return prefix, d, fam, contigs, pos


def _sub_fileset(tmp_path, name, d, fam, contigs, pos, kept):
    prefix = str(tmp_path / name)
    plink.write_fileset(prefix, d[kept], fam=[fam[k] for k in kept], contigs=contigs, positions=pos)
    return prefix


def _sample_lines(text):
    return {ln.split("\t")[0]: ln for ln in text.splitlines() if ln.count("\t") == 3}


def _from_matrix_size(text):
    lines = text.splitlines()
    start = next(i for i, ln in enumerate(lines) if ln.startswith("Matrix size:"))
    return [ln for ln in lines[start:] if not ln.startswith("GPU stats:")]


def _run(capsys, argv):
    variants_pca.main(argv)
    return capsys.readouterr().out


def _same_file(a, b):
    assert open(a, "rb").read() == open(b, "rb").read(), (a, b)


def _same_npz(a, b):
    with np.load(a) as x, np.load(b) as y:
        assert sorted(x.files) == sorted(y.files)
        for k in x.files:
            if x[k].dtype.kind == "f":
                np.testing.assert_array_equal(_bits(x[k]), _bits(y[k]))
            else:
                np.testing.assert_array_equal(x[k], y[k])


def _driver_gram(argv):
    conf = PcaConf(argv)
    driver = VariantsPcaDriver(conf)
    calls = driver.getCallsRdd(driver.getData)
    qc = driver.variantQc(calls) if conf.maf.isDefined else None
    if conf.ldPrune.isDefined:
        driver.ldPrune(calls, check_ld_flags(conf, plink.read_bim(conf.bedPath())), qc)
    S = driver.getSimilarityMatrix(calls).toArray().copy()
    driver.stop()
    return S


def _ids(path, lines):
    with open(path, "w", encoding="utf-8") as fh:
        fh.write("".join(lines))
    return path


def test_driver_matches_a_run_on_the_kept_samples(tmp_path, capsys):
    rng = np.random.default_rng(31)
    prefix, d, fam, contigs, pos = _cohort(tmp_path, rng)
    n, v = d.shape
    keep_file = _ids(str(tmp_path / "keep.txt"), ["#FID\tIID\n"] + [f"{f} {i}\n" for f, i in fam[::-1] if i != "S013"]
                     + ["\n", "NOPE NOPE\n"])
    remove_file = _ids(str(tmp_path / "remove.txt"), ["S020\n", "F1 S021\n", "S200\n"])
    mind = 0.1
    miss = (d == -1).sum(1)
    kept = [k for k in range(n) if fam[k][1] not in ("S013", "S020", "S021", "S200") and miss[k] / v <= mind]
    m = len(kept)
    assert m < n - 5
    sub = _sub_fileset(tmp_path, "kept", d, fam, contigs, pos, kept)
    common = ["--variants-per-partition", "700", "--num-pc", "3"]
    qc = ["--maf", "0.05", "--geno", "0.02", "--hwe", "1e-6"]
    ld = ["--ld-prune", "0.2", "--ld-window-kb", "120"]
    sel = ["--keep", keep_file, "--remove", remove_file, "--mind", str(mind)]
    a, b = str(tmp_path / "a"), str(tmp_path / "b")
    extra = lambda p: ["--output-path", p, "--make-king-table", p + ".kin0", "--save-loadings", p + ".npz"]  # noqa: E731
    got = _run(capsys, ["--bed-path", prefix] + sel + qc + ld + extra(a) + common)
    want = _run(capsys, ["--bed-path", sub] + qc + ld + extra(b) + common)
    assert f"--keep {keep_file}: 1 IDs match no sample." in got
    n_mind = sum(1 for k in range(n) if fam[k][1] not in ("S013", "S020", "S021", "S200") and miss[k] / v > mind)
    assert n_mind >= 3
    assert f"Sample QC: {m} of {n} samples kept (1 by --keep, 3 by --remove, {n_mind} by --mind {mind!r} removed)." in got
    assert f"Matrix size: {m}." in got and got.index("Sample QC:") < got.index("Matrix size:")
    assert _from_matrix_size(got) == _from_matrix_size(want)
    assert len(_sample_lines(got)) == m and _sample_lines(got) == _sample_lines(want)
    for suffix in (".kin0", ".afreq", ".vmiss", ".hardy", ".prune.in", ".prune.out"):
        _same_file(a + suffix, b + suffix)
    _same_npz(a + ".npz", b + ".npz")
    smiss = open(a + ".smiss").read().splitlines()
    assert len(smiss) == 1 + n - 4 and smiss[0] == "#FID\tIID\tMISSING_CT\tOBS_CT\tF_MISS"
    assert [int(ln.split("\t")[2]) for ln in smiss[1:]] == [int(miss[k]) for k in range(n)
                                                           if fam[k][1] not in ("S013", "S020", "S021", "S200")]
    np.testing.assert_array_equal(_driver_gram(["--bed-path", prefix] + sel + qc + ld + common),
                                  _driver_gram(["--bed-path", sub] + qc + ld + common))
    capsys.readouterr()
    # --remove P.mindrem.id: the same run as --mind alone, but for the attribution and --mind's own files
    c, e = str(tmp_path / "c"), str(tmp_path / "e")
    by_mind = _run(capsys, ["--bed-path", prefix, "--mind", str(mind)] + qc + ld + extra(c) + common)
    listed = _run(capsys, ["--bed-path", prefix, "--remove", c + ".mindrem.id"] + qc + ld + extra(e) + common)
    assert f"Sample QC: {n - n_mind - 1} of {n} samples kept ({n_mind + 1} by --mind {mind!r} removed)." in by_mind
    assert f"Sample QC: {n - n_mind - 1} of {n} samples kept ({n_mind + 1} by --remove removed)." in listed
    assert _sample_lines(listed) == _sample_lines(by_mind) and _from_matrix_size(listed) == _from_matrix_size(by_mind)
    for suffix in (".kin0", ".afreq", ".vmiss", ".hardy", ".prune.in", ".prune.out"):
        _same_file(c + suffix, e + suffix)
    _same_npz(c + ".npz", e + ".npz")
    assert not os.path.exists(e + ".smiss") and not os.path.exists(e + ".mindrem.id")


def test_king_cutoff_and_the_keep_round_trip(tmp_path, capsys):
    rng = np.random.default_rng(32)
    prefix, d, fam, contigs, pos = _cohort(tmp_path, rng, n=200, v=2500)
    n, v = d.shape
    remove_file = _ids(str(tmp_path / "rm.txt"), [f"{fam[k][0]} {fam[k][1]}\n" for k in (0, 1, 2, 199)])
    kept = [k for k in range(n) if k not in (0, 1, 2, 199)]
    sub = _sub_fileset(tmp_path, "kept", d, fam, contigs, pos, kept)
    common = ["--variants-per-partition", "600", "--num-pc", "4"]
    a, b = str(tmp_path / "a"), str(tmp_path / "b")
    kc = ["--king-cutoff", "0.1", "--make-king-table"]
    got = _run(capsys, ["--bed-path", prefix, "--remove", remove_file, "--output-path", a] + kc + [a + ".kin0"] +
               ["--save-loadings", a + ".npz"] + common)
    want = _run(capsys, ["--bed-path", sub, "--output-path", b] + kc + [b + ".kin0"] + ["--save-loadings", b + ".npz"]
                + common)
    assert "Sample QC: 196 of 200 samples kept (4 by --remove removed)." in got
    assert _from_matrix_size(got) == _from_matrix_size(want)
    assert _sample_lines(got) == _sample_lines(want)
    for suffix in (".kin0", ".king.cutoff.in.id", ".king.cutoff.out.id"):
        _same_file(a + suffix, b + suffix)
    _same_npz(a + ".npz", b + ".npz")
    out_ids = open(a + ".king.cutoff.out.id").read().splitlines()[1:]
    assert len(out_ids) >= 1
    # --keep P.king.cutoff.in.id: the PCs of the unrelated set, bit for bit as the kept rows of the --king-cutoff run
    rt = _run(capsys, ["--bed-path", prefix, "--keep", a + ".king.cutoff.in.id"] + common)
    lines, cut_lines = _sample_lines(rt), _sample_lines(got)
    gone = {ln.split("\t")[1] for ln in out_ids}
    assert len(lines) == 196 - len(gone)
    assert lines == {k: ln for k, ln in cut_lines.items() if k not in gone}


def test_project_loadings_of_the_kept_samples(tmp_path, capsys):
    rng = np.random.default_rng(33)
    prefix, d, fam, contigs, pos = _cohort(tmp_path, rng, n=180, v=2000)
    n = d.shape[0]
    common = ["--variants-per-partition", "500", "--num-pc", "3"]
    ref = str(tmp_path / "ref.npz")
    _run(capsys, ["--bed-path", prefix, "--save-loadings", ref] + common)
    keep = np.flatnonzero(rng.random(n) < 0.3)
    keep_file = _ids(str(tmp_path / "k.txt"), [f"{fam[k][1]}\n" for k in keep])     # bare IIDs
    sub = _sub_fileset(tmp_path, "kept", d, fam, contigs, pos, keep)
    got = _run(capsys, ["--bed-path", prefix, "--keep", keep_file, "--project-loadings", ref] + common)
    want = _run(capsys, ["--bed-path", sub, "--project-loadings", ref] + common)
    assert len(_sample_lines(got)) == len(keep) and _sample_lines(got) == _sample_lines(want)
