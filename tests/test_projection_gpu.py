"""GPU tests of variant loadings and projection (vpca_loadings_* / vpca_project_*, DESIGN.md 6): loadings against numpy
with U from the GPU's own computePca, bit-identical loadings across input forms, self-projection, held-out samples,
partial overlap, reproducibility, status codes, and the --save-loadings / --project-loadings driver flags."""
import os
import socket

import numpy as np
import pytest

from projection_ref import dense_to_csr, np_loadings, np_project

pytestmark = pytest.mark.gpu

P = 1024   # panel width of the device-resident inputs below
# component counts that launch every KMAX instantiation of project.cu (2, 4, 8, 16) at and past its lower and upper
# bound; at KMAX 16 loadings_kernel runs 2 variants per thread (VT) instead of 4, and project_kernel stages w in
# 256-variant tiles from KMAX 8 on
KS = (1, 2, 4, 5, 8, 9, 16)


def _cohort(oracle, n, nv, seed=20240901):
    return oracle.c_synth_dense(seed, n, 0, nv, 0).astype(np.int64)          # binary carriers, population structure


def _reference(native, X, k=4, dtype=0):
    """A context that accumulated X and ran computePca(k): (ctx, U, evals)."""
    n = X.shape[0]
    nat = native.NativePca(n, dtype=dtype, num_pc=k)
    off, idx = dense_to_csr(X)
    nat.accumulateCalls(0, off, idx)
    nat.commit(0)
    nat.finalizeGram()
    U, evals, _ = nat.computePca(k)
    return nat, U, evals


def _bed_rows(tmp_path, X, name="c"):
    from spark_examples_b200 import plink
    plink.write_fileset(str(tmp_path / name), X)                   # A1 count 1 = het: carrier of A1, 0: hom A2
    bed = plink.BedFile(str(tmp_path / name))
    return bed.rows(0, bed.n_variants)


def _panels(X, dtype, panel=P):
    """(N, V) cells -> device panel layout (torch uint8 buffer) of the dtype, zero cells after V."""
    import torch
    n, nv = X.shape
    npan = (nv + panel - 1) // panel
    Xp = np.zeros((n, npan * panel), np.int64)
    Xp[:, :nv] = X
    pan = np.ascontiguousarray(Xp.reshape(n, npan, panel).transpose(1, 0, 2))     # (panels, n, panel)
    if dtype == 0:
        host = pan.astype(np.int8).view(np.uint8)
    elif dtype == 1:
        host = (pan.astype(np.float32).view(np.uint32) >> 16).astype(np.uint16).view(np.uint8)   # exact for integers
    else:
        codes = (2 * pan).astype(np.uint8)
        host = codes[..., 0::2] | (codes[..., 1::2] << 4)
    return torch.from_numpy(np.ascontiguousarray(host).reshape(-1)).cuda()


def _rel(a, b):
    return np.max(np.abs(a - b), axis=0) / np.max(np.abs(b), axis=0)


@pytest.mark.parametrize("n,nv", [(257, 3000), (1092, 8000), (257, 3001), (1092, 3001)])
@pytest.mark.parametrize("dtype", [0, 1, 2], ids=["int8", "bf16", "e2m1"])
def test_loadings_match_numpy(oracle, n, nv, dtype):
    """Loadings of k' = 1 .. 16 components (KS) from one computePca(16), from CSR calls and from panels 384 and 1024
    variants wide: numpy's X^T U to 1e-12, and every column the same bits whatever k' and input -- each column is summed
    over the samples in order by every KMAX / VT instantiation.  N = 1092 takes U in five 256-sample tiles at KMAX 16,
    the last one partial; nv = 3001 leaves a partial last panel and a thread with one variant of its pair."""
    import torch
    from spark_examples_b200 import native
    X = _cohort(oracle, n, nv)
    nat, U, _ = _reference(native, X, 16, dtype)
    csr = dense_to_csr(X)
    panels = {}
    with nat:
        calls = {k: nat.loadingsCalls(k, *csr) for k in KS}
        for pw in (384, 1024):
            d_x = _panels(X, dtype, pw)                            # the kernel's own decode of each element type
            for k in KS:
                dw = torch.zeros((nv, k), dtype=torch.float64, device="cuda")
                dc = torch.zeros(nv, dtype=torch.int32, device="cuda")
                nat.loadingsPanels(k, d_x.data_ptr(), nv, pw, dw.data_ptr(), dc.data_ptr())
                panels[pw, k] = dw, dc
            nat.synchronize()
    W, C = np_loadings(X, U)
    w16 = calls[16][0]
    assert np.all(_rel(w16, W) <= 1e-12), _rel(w16, W)
    for k in KS:
        w, cnt = calls[k]
        assert np.array_equal(cnt, C), k
        assert np.array_equal(w.view(np.uint64), w16[:, :k].view(np.uint64)), k   # independent of how many are asked for
        for pw in (384, 1024):
            dw, dc = panels[pw, k]
            assert np.array_equal(dc.cpu().numpy(), C), (pw, k)
            assert np.array_equal(dw.cpu().numpy().view(np.uint64), w.view(np.uint64)), (pw, k)


def test_loadings_bit_identical_across_inputs_and_runs(oracle, tmp_path):
    import torch
    from spark_examples_b200 import native
    X = _cohort(oracle, 300, 2500)
    rows = _bed_rows(tmp_path, X)
    nat, U, _ = _reference(native, X, 3)
    with nat:
        a, ca = nat.loadingsCalls(3, *dense_to_csr(X))
        b, cb = nat.loadingsBed(3, rows, 1)
        d_x = _panels(X, 0)
        dw = torch.zeros((X.shape[1], 3), dtype=torch.float64, device="cuda")
        dc = torch.zeros(X.shape[1], dtype=torch.int32, device="cuda")
        nat.loadingsPanels(3, d_x.data_ptr(), X.shape[1], P, dw.data_ptr(), dc.data_ptr())
        nat.synchronize()
        a2, _ = nat.loadingsCalls(3, *dense_to_csr(X))
    assert np.array_equal(a.view(np.uint64), b.view(np.uint64)) and np.array_equal(ca, cb)
    assert np.array_equal(a.view(np.uint64), dw.cpu().numpy().view(np.uint64)) and np.array_equal(ca, dc.cpu().numpy())
    assert np.array_equal(a.view(np.uint64), a2.view(np.uint64))


def test_self_projection_reproduces_the_eigenvectors(oracle):
    """Projecting the reference samples with their own loadings gives U back, at k = 4 and 16 (KMAX 4 and 16)."""
    from spark_examples_b200 import native
    X = _cohort(oracle, 1092, 8000)
    n = X.shape[0]
    nat, U, evals = _reference(native, X, 16)
    off, idx = dense_to_csr(X)
    with nat:
        w, cnt = nat.loadingsCalls(16, off, idx)
    assert np.all(evals > 1e-3 * evals[0])                        # every pair has lambda well above zero
    for k in (4, 16):
        with native.NativePca(n) as proj:
            proj.projectBegin(k)
            proj.projectCalls(off, idx, np.ascontiguousarray(w[:, :k]), cnt / n)
            got = proj.projectGet(evals[:k])
        err = oracle.eigvec_rel_err(got, U[:, :k])
        print(f"self-projection k={k} eigvec_rel_err per component: {err}")
        assert np.all(err <= 1e-6), (k, err)


def test_held_out_samples_match_numpy_through_every_input(oracle, tmp_path):
    """M = 200 held-out samples (not a multiple of 128) projected with k = 3, 5, 8, 9 and 16 components through CSR
    calls, .bed rows and panels 384 (one 256- and one 128-variant tile of w from KMAX 8 on) and 1024 variants wide:
    numpy to 1e-10, and each component the same bits whatever k -- every column is summed in the same order."""
    import torch
    from spark_examples_b200 import native
    X = _cohort(oracle, 900, 5000)
    n1 = 700
    R, Y = X[:n1], X[n1:]
    m = Y.shape[0]
    nat, U, evals = _reference(native, R, 16)
    with nat:
        loadings = {k: nat.loadingsCalls(k, *dense_to_csr(R)) for k in (3, 5, 8, 9, 16)}
    cnt = loadings[16][1]
    mean = cnt / n1
    rows, y_csr, d_y = _bed_rows(tmp_path, Y), dense_to_csr(Y), {pw: _panels(Y, 0, pw) for pw in (384, 1024)}
    outs = {}
    with native.NativePca(m) as proj:
        for k, (w, _) in loadings.items():
            proj.projectBegin(k)
            proj.projectCalls(*y_csr, w, mean)
            outs[k, "calls"] = proj.projectGet(evals[:k])
            proj.projectBegin(k)
            proj.projectBed(rows, w, mean, 1)
            outs[k, "bed"] = proj.projectGet(evals[:k])
            dw, dm = torch.from_numpy(w).cuda(), torch.from_numpy(mean).cuda()
            for pw in (384, 1024):
                proj.projectBegin(k)
                proj.projectPanels(d_y[pw].data_ptr(), Y.shape[1], pw, dw.data_ptr(), dm.data_ptr())
                outs[k, f"panels{pw}"] = proj.projectGet(evals[:k])
    want = np_project(Y, loadings[16][0], cnt, n1, evals)
    for (k, name), got in outs.items():
        assert got.shape == (m, k)
        assert np.all(_rel(got, want[:, :k]) <= 1e-10), (k, name, _rel(got, want[:, :k]))
        assert np.array_equal(got.view(np.uint64), outs[16, name][:, :k].view(np.uint64)), (k, name)


def test_partial_overlap_equals_zeroed_rows_and_runs_are_reproducible(oracle):
    from spark_examples_b200 import native
    X = _cohort(oracle, 600, 4000)
    R, Y = X[:450], X[450:]
    nat, U, evals = _reference(native, R, 2)
    with nat:
        w, cnt = nat.loadingsCalls(2, *dense_to_csr(R))
    mean = cnt / 450
    keep = (np.arange(X.shape[1]) % 5) != 2
    wz = w.copy()
    wz[~keep] = 0.0
    with native.NativePca(Y.shape[0]) as proj:
        runs = []
        for _ in range(2):
            proj.projectBegin(2)
            proj.projectCalls(*dense_to_csr(Y), wz, mean)
            runs.append(proj.projectGet(evals))
        proj.projectBegin(2)
        proj.projectCalls(*dense_to_csr(Y[:, keep]), w[keep], mean[keep])
        only = proj.projectGet(evals)
    assert np.array_equal(runs[0].view(np.uint64), runs[1].view(np.uint64))
    assert np.all(_rel(runs[0], only) <= 1e-12)
    assert np.all(_rel(only, np_project(Y[:, keep], w[keep], cnt[keep], 450, evals)) <= 1e-10)


def test_status_codes(oracle):
    from spark_examples_b200 import native
    X = _cohort(oracle, 200, 600)
    off, idx = dense_to_csr(X)
    with native.NativePca(200) as nat:
        nat.accumulateCalls(0, off, idx)
        nat.commit(0)
        nat.finalizeGram()
        with pytest.raises(native.VpcaError) as e:
            nat.loadingsCalls(2, off, idx)                          # no computePca yet
        assert e.value.code == native.VPCA_ERR_STATE
        nat.computePca(3)
        for k in (0, 17, 4):                                        # outside [1, 16] / more than computePca computed
            with pytest.raises(native.VpcaError) as e:
                nat.loadingsCalls(k, off, idx)
            assert e.value.code == native.VPCA_ERR_BAD_ARG
        with pytest.raises(native.IndexOutOfRange):
            nat.loadingsCalls(2, np.array([0, 1]), np.array([200], np.int32))
        with pytest.raises(native.VpcaError) as e:
            nat.loadingsPanels(2, 256, 10, 100, 256, 256)          # panel width not a multiple of 128
        assert e.value.code == native.VPCA_ERR_BAD_ARG
        nat.loadingsCalls(2, off, idx)
        nat.reset()                                                 # U no longer valid
        with pytest.raises(native.VpcaError) as e:
            nat.loadingsCalls(2, off, idx)
        assert e.value.code == native.VPCA_ERR_STATE
        w = np.zeros((1, 2))
        m = np.zeros(1)
        with pytest.raises(native.VpcaError) as e:
            nat.projectCalls(np.array([0, 1]), np.array([3], np.int32), w, m)   # before projectBegin
        assert e.value.code == native.VPCA_ERR_STATE
        for k in (0, 17):
            with pytest.raises(native.VpcaError) as e:
                nat.projectBegin(k)
            assert e.value.code == native.VPCA_ERR_BAD_ARG
        nat.projectBegin(2)
        with pytest.raises(native.IndexOutOfRange):
            nat.projectCalls(np.array([0, 1]), np.array([200], np.int32), w, m)
        with pytest.raises(native.VpcaError) as e:
            nat.projectPanels(256, 10, 100, 256, 256)
        assert e.value.code == native.VPCA_ERR_BAD_ARG
        nat.reset()                                                 # drops the projection
        with pytest.raises(native.VpcaError) as e:
            nat.projectGet(np.ones(2))
        assert e.value.code == native.VPCA_ERR_STATE
    with native.NativePca(256, gram_band=(0, 128)) as band:
        for call in (lambda: band.projectBegin(2), lambda: band.loadingsCalls(2, off, idx)):
            with pytest.raises(native.VpcaError) as e:
                call()
            assert e.value.code == native.VPCA_ERR_UNSUPPORTED


def _tsv(lines):
    return {ln.split("\t")[0]: np.array([float(x) for x in ln.split("\t")[2:]]) for ln in lines}


def test_cli_save_then_project_bed(oracle, tmp_path, capsys):
    """--save-loadings then --project-loadings through the driver, with --num-pc 2 (the default) and 16 (the most
    components loadings hold)."""
    for num_pc in (2, 16):
        (tmp_path / f"pc{num_pc}").mkdir()
        _cli_save_then_project_bed(oracle, tmp_path / f"pc{num_pc}", capsys, num_pc)


def _cli_save_then_project_bed(oracle, tmp_path, capsys, num_pc):
    from spark_examples_b200 import plink, variants_pca
    d = oracle.c_synth_dense(7, 400, 0, 3000, 1).astype(np.int64)   # dosage 0/1/2
    n, nv = d.shape
    plink.write_fileset(str(tmp_path / "ref"), d)
    lpath = str(tmp_path / "ref.loadings.npz")
    variants_pca.main(["--bed-path", str(tmp_path / "ref"), "--variants-per-partition", "1000", "--save-loadings", lpath,
                       "--num-pc", str(num_pc)])
    first = _tsv([ln for ln in capsys.readouterr().out.splitlines() if ln.count("\t") == 3])
    variants_pca.main(["--bed-path", str(tmp_path / "ref"), "--variants-per-partition", "700", "--project-loadings", lpath])
    again = _tsv([ln for ln in capsys.readouterr().out.splitlines() if ln.count("\t") == 3])
    assert first.keys() == again.keys()
    for name in first:
        assert np.all(np.abs(first[name] - again[name]) <= 1e-6), name
    # a sample subset, variants shuffled and partly missing, in a second fileset
    f = np.load(lpath)
    assert f["loadings"].shape == (nv, num_pc) and f["eigenvalues"].shape == (num_pc,)
    rng = np.random.default_rng(3)
    subset = np.sort(rng.choice(n, 120, replace=False))
    cols = rng.permutation(nv)[: nv - 400]
    sub = d[subset][:, cols]
    prefix = str(tmp_path / "new")
    plink.write_fileset(prefix, sub, fam=[("synth", f"S{i:06d}") for i in subset])
    with open(prefix + ".bim", "w") as fh:                          # keep each column's own .bim identity
        for j in cols:
            fh.write(f"17\trs{j + 1}\t0\t{41196311 + j}\tA\tG\n")
    variants_pca.main(["--bed-path", prefix, "--project-loadings", lpath])
    got = _tsv([ln for ln in capsys.readouterr().out.splitlines() if ln.count("\t") == 3])
    want = np_project((sub > 0).astype(np.int64), f["loadings"][cols], f["count"][cols], int(f["n_samples"]),
                      f["eigenvalues"])
    for r, i in enumerate(subset):
        g = got[f"S{i:06d}"]
        assert np.all(np.abs(g - want[r, :2]) <= 1e-10 * np.max(np.abs(want[:, :2]), axis=0)), (i, g, want[r])


def _ngpu():
    try:
        import torch
        return torch.cuda.device_count()
    except Exception:
        return 0


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _rank_main(rank, world, port, argv):
    from spark_examples_b200 import variants_pca
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world),
                      LOCAL_RANK=str(rank))
    variants_pca.main(argv)


@pytest.mark.skipif(_ngpu() < 2, reason="needs 2 GPUs")
def test_two_rank_loadings_and_projection_equal_one_rank(oracle, tmp_path):
    import torch.multiprocessing as mp
    from spark_examples_b200 import plink, variants_pca
    d = oracle.c_synth_dense(11, 500, 0, 6000, 1).astype(np.int64)
    plink.write_fileset(str(tmp_path / "c"), d)
    base = ["--bed-path", str(tmp_path / "c"), "--variants-per-partition", "1024"]
    variants_pca.main(base + ["--save-loadings", str(tmp_path / "one.npz")])
    variants_pca.main(base + ["--project-loadings", str(tmp_path / "one.npz"), "--output-path", str(tmp_path / "p1")])
    mp.spawn(_rank_main, args=(2, _free_port(), base + ["--save-loadings", str(tmp_path / "two.npz")]), nprocs=2, join=True)
    mp.spawn(_rank_main, args=(2, _free_port(), base + ["--project-loadings", str(tmp_path / "two.npz"), "--output-path",
                                                        str(tmp_path / "p2")]), nprocs=2, join=True)
    one, two = np.load(tmp_path / "one.npz"), np.load(tmp_path / "two.npz")
    assert np.array_equal(one["keys"], two["keys"]) and np.array_equal(one["count"], two["count"])
    assert np.all(_rel(two["loadings"], one["loadings"]) <= 1e-10)
    read = lambda p: {ln.split("\t")[0]: np.array([float(x) for x in ln.split("\t")[1:3]])
                      for ln in (tmp_path / p / "part-00000").read_text().splitlines()}
    a, b = read("p1-pca.tsv"), read("p2-pca.tsv")
    scale = np.max(np.abs(np.array(list(a.values()))), axis=0)
    for name in a:
        assert np.all(np.abs(a[name] - b[name]) <= 1e-10 * scale), name
