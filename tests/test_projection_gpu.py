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


def _panels(X, dtype):
    """(N, V) cells -> device panel layout (torch uint8 buffer) of the dtype, zero cells after V."""
    import torch
    n, nv = X.shape
    npan = (nv + P - 1) // P
    Xp = np.zeros((n, npan * P), np.int64)
    Xp[:, :nv] = X
    pan = np.ascontiguousarray(Xp.reshape(n, npan, P).transpose(1, 0, 2))     # (panels, n, P)
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


@pytest.mark.parametrize("n,nv", [(257, 3000), (1092, 8000)])
@pytest.mark.parametrize("dtype", [0, 1, 2], ids=["int8", "bf16", "e2m1"])
def test_loadings_match_numpy(oracle, n, nv, dtype):
    from spark_examples_b200 import native
    X = _cohort(oracle, n, nv)
    import torch
    nat, U, _ = _reference(native, X, 4, dtype)
    with nat:
        w, cnt = nat.loadingsCalls(4, *dense_to_csr(X))
        w2, _ = nat.loadingsCalls(2, *dense_to_csr(X))
        d_x = _panels(X, dtype)                                    # the kernel's own decode of each element type
        dw = torch.zeros((nv, 4), dtype=torch.float64, device="cuda")
        dc = torch.zeros(nv, dtype=torch.int32, device="cuda")
        nat.loadingsPanels(4, d_x.data_ptr(), nv, P, dw.data_ptr(), dc.data_ptr())
        nat.synchronize()
    W, C = np_loadings(X, U)
    assert np.array_equal(cnt, C) and np.array_equal(dc.cpu().numpy(), C)
    assert np.array_equal(dw.cpu().numpy().view(np.uint64), w.view(np.uint64))
    assert np.all(_rel(w, W) <= 1e-12), _rel(w, W)
    assert np.array_equal(w2, w[:, :2])                            # a column does not depend on how many are asked for


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
    from spark_examples_b200 import native
    X = _cohort(oracle, 1092, 8000)
    n = X.shape[0]
    nat, U, evals = _reference(native, X, 4)
    off, idx = dense_to_csr(X)
    with nat:
        w, cnt = nat.loadingsCalls(4, off, idx)
    with native.NativePca(n) as proj:
        proj.projectBegin(4)
        proj.projectCalls(off, idx, w, cnt / n)
        got = proj.projectGet(evals)
    err = oracle.eigvec_rel_err(got, U)
    print(f"self-projection eigvec_rel_err per component: {err}")
    assert np.all(err <= 1e-6)


def test_held_out_samples_match_numpy_through_every_input(oracle, tmp_path):
    import torch
    from spark_examples_b200 import native
    X = _cohort(oracle, 900, 5000)
    n1 = 700
    R, Y = X[:n1], X[n1:]
    m = Y.shape[0]
    nat, U, evals = _reference(native, R, 3)
    with nat:
        w, cnt = nat.loadingsCalls(3, *dense_to_csr(R))
    want = np_project(Y, w, cnt, n1, evals)
    mean = cnt / n1
    outs = {}
    with native.NativePca(m) as proj:
        proj.projectBegin(3)
        proj.projectCalls(*dense_to_csr(Y), w, mean)
        outs["calls"] = proj.projectGet(evals)
        proj.projectBegin(3)
        proj.projectBed(_bed_rows(tmp_path, Y), w, mean, 1)
        outs["bed"] = proj.projectGet(evals)
        proj.projectBegin(3)
        d_y = _panels(Y, 0)
        dw, dm = torch.from_numpy(w).cuda(), torch.from_numpy(mean).cuda()
        proj.projectPanels(d_y.data_ptr(), Y.shape[1], P, dw.data_ptr(), dm.data_ptr())
        outs["panels"] = proj.projectGet(evals)
    for name, got in outs.items():
        assert np.all(_rel(got, want) <= 1e-10), (name, _rel(got, want))


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
    from spark_examples_b200 import plink, variants_pca
    d = oracle.c_synth_dense(7, 400, 0, 3000, 1).astype(np.int64)   # dosage 0/1/2
    n, nv = d.shape
    plink.write_fileset(str(tmp_path / "ref"), d)
    lpath = str(tmp_path / "ref.loadings.npz")
    variants_pca.main(["--bed-path", str(tmp_path / "ref"), "--variants-per-partition", "1000", "--save-loadings", lpath])
    first = _tsv([ln for ln in capsys.readouterr().out.splitlines() if ln.count("\t") == 3])
    variants_pca.main(["--bed-path", str(tmp_path / "ref"), "--variants-per-partition", "700", "--project-loadings", lpath])
    again = _tsv([ln for ln in capsys.readouterr().out.splitlines() if ln.count("\t") == 3])
    assert first.keys() == again.keys()
    for name in first:
        assert np.all(np.abs(first[name] - again[name]) <= 1e-6), name
    # a sample subset, variants shuffled and partly missing, in a second fileset
    f = np.load(lpath)
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
