"""Principal coordinates of a subset of the samples (vpca_compute_pca_subset, DESIGN.md 8) and --king-cutoff: kept rows
bit for bit against an M-sample context holding S[K, K], removed rows against the FP64 formula and against a projection
of their genotypes, masked loadings bit for bit against an M-sample context, the state rules, and the driver end to
end on a planted pedigree."""
import numpy as np
import pytest

from kinship_ref import dosage_codes, king_pairs, pack_codes
from spark_examples_b200 import native, plink, variants_pca

pytestmark = pytest.mark.gpu


def _bits(a):
    return np.ascontiguousarray(a, np.float64).view(np.int64)


def _keep_patterns(n, rng):
    out = {"all": np.ones(n, bool)}
    first = np.ones(n, bool)
    first[0] = False
    last = np.ones(n, bool)
    last[-1] = False
    out["first"], out["last"] = first, last
    if n >= 8:
        block = np.ones(n, bool)
        block[n // 3:n // 3 + max(2, n // 10)] = False
        out["block"] = block
        rnd = rng.random(n) >= 0.1
        rnd[:2] = True
        out["random"] = rnd
    return out


def _gram(rng, n, nv=3000):
    p = rng.uniform(0.05, 0.6, size=nv)
    pop = (np.arange(n) % 3)[:, None]                                # three populations: a few clear axes
    x = (rng.random((n, nv)) < p * (1 + 0.5 * pop)).astype(np.int64)
    return (x @ x.T).astype(np.int32)


def _removed_ref(S, keep, u, evals):
    K, R = np.flatnonzero(keep), np.flatnonzero(~keep)
    rho = S[np.ix_(K, K)].astype(np.float64).sum(axis=1)
    return (S[np.ix_(R, K)].astype(np.float64) @ u - (rho @ u) / len(K)) / evals


@pytest.mark.parametrize("eig", ["direct", "lanczos", "auto"])
@pytest.mark.parametrize("n", [3, 129, 1000, 2504])
def test_kept_rows_bit_identical_and_removed_rows_by_formula(monkeypatch, n, eig):
    if eig != "auto":
        monkeypatch.setenv("VPCA_EIG", eig)
    rng = np.random.default_rng(n)
    S = _gram(rng, n)
    ks = [1, 2, 5, 16] if n < 2504 else [2, 16]
    with native.NativePca(n) as nat:
        nat.setGram(S)
        for name, keep in _keep_patterns(n, rng).items():
            K = np.flatnonzero(keep)
            m = len(K)
            with native.NativePca(m) as ref:
                ref.setGram(S[np.ix_(K, K)])
                for k in [k for k in ks if k <= m]:
                    vecs, evals, nz = nat.computePcaSubset(keep, k)
                    method = nat.stats()["eig_method"]
                    rv, re, rnz = ref.computePca(k)
                    assert method == ref.stats()["eig_method"], (name, k)
                    np.testing.assert_array_equal(_bits(vecs[K]), _bits(rv), err_msg=f"{name} k={k}")
                    np.testing.assert_array_equal(_bits(evals), _bits(re))
                    assert nz == rnz
                    if keep.all():
                        av, ae, anz = nat.computePca(k)
                        np.testing.assert_array_equal(_bits(vecs), _bits(av))
                        np.testing.assert_array_equal(_bits(evals), _bits(ae))
                        assert nz == anz
                    else:
                        want = _removed_ref(S, keep, rv, re)
                        # a null eigenvalue (M = 2 has rank 1 after centring) is rounding noise, and the projection
                        # divides by it: there the column's own size sets the scale
                        scale = np.maximum(np.abs(rv).max(axis=0), np.abs(want).max(axis=0))
                        assert (np.abs(vecs[~keep] - want) <= 1e-12 * scale).all(), (name, k)


def _cohort(rng, n, nv):
    p = rng.uniform(0.05, 0.95, size=nv)[:, None]
    d = (rng.random((nv, n)) < p).astype(np.int64) + (rng.random((nv, n)) < p)
    d[rng.random((nv, n)) < 0.01] = -1
    return dosage_codes(d.T)                                          # (nv, n) codes


def _csr(has):
    off = np.zeros(has.shape[0] + 1, np.int64)
    np.cumsum(has.sum(axis=1), out=off[1:])
    return off, np.nonzero(has)[1].astype(np.int32)


def _bed_context(n, rows):
    nat = native.NativePca(n)
    nat.accumulateBed(0, rows)
    nat.commit(0)
    nat.finalizeGram()
    return nat


@pytest.mark.parametrize("dtype", [native.DTYPE_I8, native.DTYPE_BF16])
def test_masked_loadings_and_projection_of_the_removed(dtype):
    rng = np.random.default_rng(77)
    n, nv, k = 300, 6000, 5
    codes = _cohort(rng, n, nv)
    keep = rng.random(n) >= 0.1
    K, R = np.flatnonzero(keep), np.flatnonzero(~keep)
    rows = pack_codes(codes)
    with native.NativePca(n, dtype=dtype) as nat, native.NativePca(len(K), dtype=dtype) as ref:
        nat.accumulateBed(0, rows)
        nat.commit(0)
        nat.finalizeGram()
        ref.accumulateBed(0, pack_codes(codes[:, K]))
        ref.commit(0)
        ref.finalizeGram()
        vecs, evals, _ = nat.computePcaSubset(keep, k)
        rv, re, _ = ref.computePca(k)
        np.testing.assert_array_equal(_bits(vecs[K]), _bits(rv))
        w, cnt = nat.loadingsBed(k, rows)
        rw, rcnt = ref.loadingsBed(k, pack_codes(codes[:, K]))
        np.testing.assert_array_equal(_bits(w), _bits(rw))
        np.testing.assert_array_equal(cnt, rcnt)
        has = plink.decode_rows(rows, n)                               # (nv, n) carriers of A1
        np.testing.assert_array_equal(cnt, has[:, K].sum(axis=1))
        off, idx = _csr(has)
        roff, ridx = _csr(has[:, K])                                   # the same rows, kept columns only
        cw, ccnt = nat.loadingsCalls(k, off, idx)
        rcw, rccnt = ref.loadingsCalls(k, roff, ridx)
        np.testing.assert_array_equal(_bits(cw), _bits(rcw))
        np.testing.assert_array_equal(ccnt, rccnt)
    with native.NativePca(len(R), dtype=dtype) as proj:
        proj.projectBegin(k)
        proj.projectBed(pack_codes(codes[:, R]), w, cnt / len(K))
        P = proj.projectGet(evals)
    scale = np.abs(vecs[K]).max(axis=0)
    assert (np.abs(vecs[R] - P) <= 1e-12 * scale).all()


def test_state_rules_and_refusals():
    rng = np.random.default_rng(5)
    n, nv = 200, 4000
    codes = _cohort(rng, n, nv)
    rows = pack_codes(codes)
    keep = np.ones(n, bool)
    keep[::7] = False
    with native.NativePca(n) as fresh:
        with pytest.raises(native.VpcaError) as e:
            fresh.computePcaSubset(keep, 2)                          # not finalized
        assert e.value.code == native.VPCA_ERR_STATE
    nat = _bed_context(n, rows)
    with nat, _bed_context(n, rows) as plain:
        nat.kinshipBed(rows)
        S0, kin0 = nat.getGram(), nat.kinshipPairs()
        pv, _, _ = plain.computePca(3)
        pw, pc = plain.loadingsBed(3, rows)
        nat.computePcaSubset(keep, 3)
        st = nat.stats()
        assert st["eig_method"] == 1 and st["eig_iterations"] == 0   # 172 kept samples: the direct solver
        with pytest.raises(native.VpcaError) as e:
            nat.getTridiagonal()
        assert e.value.code == native.VPCA_ERR_STATE
        mw, mc = nat.loadingsBed(3, rows)
        assert (mc <= pc).all() and (mc < pc).any()                  # counts over the kept samples only
        v, _, _ = nat.computePca(3)                                  # the next full solve ends the mask
        np.testing.assert_array_equal(_bits(v), _bits(pv))
        w, c = nat.loadingsBed(3, rows)
        np.testing.assert_array_equal(_bits(w), _bits(pw))
        np.testing.assert_array_equal(c, pc)
        nat.computePcaSubset(keep, 3)
        np.testing.assert_array_equal(nat.getGram(), S0)             # the Gram and the kinship counts are only read
        ids, counts, kin = nat.kinshipPairs()
        np.testing.assert_array_equal(ids, kin0[0])
        np.testing.assert_array_equal(counts, kin0[1])
        np.testing.assert_array_equal(_bits(kin), _bits(kin0[2]))
        L = native.load_library()
        out = np.zeros(n * 16)
        for bad_keep, k in [(np.zeros(n, bool), 1), (np.eye(1, n, 5, dtype=bool)[0], 1), (keep, 0), (keep, 17),
                            (np.r_[np.ones(4, bool), np.zeros(n - 4, bool)], 5)]:
            with pytest.raises(native.VpcaError) as e:
                nat.computePcaSubset(bad_keep, k)
            assert e.value.code == native.VPCA_ERR_BAD_ARG, (bad_keep.sum(), k)
        assert L.vpca_compute_pca_subset(nat._h, None, 2, out.ctypes.data, None, None) == native.VPCA_ERR_BAD_ARG
        nat.reset()
        with pytest.raises(native.VpcaError) as e:
            nat.loadingsBed(3, rows)                                   # reset ends U and the mask
        assert e.value.code == native.VPCA_ERR_STATE
        with pytest.raises(native.VpcaError) as e:
            nat.computePcaSubset(keep, 2)
        assert e.value.code == native.VPCA_ERR_STATE
    with native.NativePca(64, gram_band=(0, 32)) as band:
        with pytest.raises(native.VpcaError) as e:
            band.computePcaSubset(np.ones(64, bool), 2)                # arguments, then state, as vpca_compute_pca
        assert e.value.code == native.VPCA_ERR_STATE
        band.finalizeGram()
        with pytest.raises(native.VpcaError) as e:
            band.computePcaSubset(np.ones(64, bool), 2)
        assert e.value.code == native.VPCA_ERR_UNSUPPORTED
        with pytest.raises(native.VpcaError) as e:
            band.computePcaSubset(np.ones(64, bool), 0)
        assert e.value.code == native.VPCA_ERR_BAD_ARG


@pytest.mark.parametrize("eig", ["direct", "lanczos"])
def test_more_than_sixteen_components(monkeypatch, eig):
    """num_pc = 20 admits k up to 20: kept rows bit for bit against an M-sample context with the same num_pc, removed rows
    by the formula in every column, and loadings of the first 16 columns after the solve."""
    monkeypatch.setenv("VPCA_EIG", eig)
    rng = np.random.default_rng(2020)
    n = 700
    codes = _cohort(rng, n, 4000)
    rows = pack_codes(codes)
    keep = rng.random(n) >= 0.1
    K = np.flatnonzero(keep)
    with native.NativePca(n, num_pc=20) as nat, native.NativePca(len(K), num_pc=20) as ref:
        nat.accumulateBed(0, rows)
        nat.commit(0)
        nat.finalizeGram()
        ref.accumulateBed(0, pack_codes(codes[:, K]))
        ref.commit(0)
        ref.finalizeGram()
        S = nat.getGram()
        for k in [17, 20]:
            vecs, evals, nz = nat.computePcaSubset(keep, k)
            rv, re, rnz = ref.computePca(k)
            assert vecs.shape == (n, k)
            np.testing.assert_array_equal(_bits(vecs[K]), _bits(rv))
            np.testing.assert_array_equal(_bits(evals), _bits(re))
            assert nz == rnz
            want = _removed_ref(S, keep, rv, re)
            scale = np.maximum(np.abs(rv).max(axis=0), np.abs(want).max(axis=0))
            assert (np.abs(vecs[~keep] - want) <= 1e-12 * scale).all(), k
        w, cnt = nat.loadingsBed(16, rows)
        rw, rcnt = ref.loadingsBed(16, pack_codes(codes[:, K]))
        np.testing.assert_array_equal(_bits(w), _bits(rw))
        np.testing.assert_array_equal(cnt, rcnt)
        with pytest.raises(native.VpcaError) as e:
            nat.computePcaSubset(keep, 21)
        assert e.value.code == native.VPCA_ERR_BAD_ARG


def _pedigree(rng, nv):
    p = rng.uniform(0.1, 0.9, size=nv)
    hap = {}

    def founder(name):
        hap[name] = (rng.random(nv) < p, rng.random(nv) < p)

    def child(name, mother, father):
        pick = lambda who: np.where(rng.random(nv) < 0.5, hap[who][0], hap[who][1])
        hap[name] = (pick(mother), pick(father))

    for f in ["F1", "F2", "F3", "F4", "U1", "U2", "U3", "U4", "U5", "U6"]:
        founder(f)
    child("C1", "F1", "F2")          # parent-offspring trio F1, F2, C1; C2 a full sib of C1
    child("C2", "F1", "F2")
    child("C3", "F3", "F4")
    hap["D1"] = hap["U1"]            # duplicate of U1
    hap["D3"] = hap["C3"]            # duplicate of C3
    names = list(hap)
    return names, np.stack([hap[s][0].astype(np.int64) + hap[s][1] for s in names])


def _sample_lines(text):
    return {ln.split("\t")[0]: ln for ln in text.splitlines() if ln.count("\t") == 3}


def test_driver_end_to_end_on_a_planted_pedigree(tmp_path, capsys):
    rng = np.random.default_rng(31)
    nv = 8000
    names, dosage = _pedigree(rng, nv)
    extra = (rng.random((60, nv)) < 0.3).astype(np.int64) + (rng.random((60, nv)) < 0.3)
    dosage = np.concatenate([dosage, extra])
    dosage[rng.random(dosage.shape) < 0.01] = -1
    n = dosage.shape[0]
    names = names + [f"X{i:02d}" for i in range(60)]
    fam = [(f"fam{i % 4}", s) for i, s in enumerate(names)]
    prefix = str(tmp_path / "cohort")
    plink.write_fileset(prefix, dosage, fam=fam)
    out = str(tmp_path / "run")
    variants_pca.main(["--bed-path", prefix, "--king-cutoff", "0.0884", "--output-path", out])
    text = capsys.readouterr().out
    ids, _, kin = king_pairs(dosage_codes(dosage), -np.inf)
    keep = variants_pca.king_cutoff_keep(n, ids, kin, 0.0884)
    removed = [names[s] for s in np.flatnonzero(~keep)]
    assert {"D1", "D3"} <= set(removed) and "C1" in removed and not {"F1", "F2"} & set(removed)
    assert all(names.index(s) < 15 for s in removed)                   # only the pedigree has relatives
    m = int(keep.sum())
    assert f"KING cutoff 0.0884: {m} of {n} samples kept, {n - m} projected." in text
    lines = open(out + ".king.cutoff.out.id").read().splitlines()
    assert lines == ["#FID\tIID"] + [f"{fam[s][0]}\t{fam[s][1]}" for s in np.flatnonzero(~keep)]
    got = _sample_lines(text)
    assert len(got) == n
    kept_prefix, rem_prefix = str(tmp_path / "kept"), str(tmp_path / "rem")
    plink.write_fileset(kept_prefix, dosage[keep], fam=[fam[s] for s in np.flatnonzero(keep)])
    plink.write_fileset(rem_prefix, dosage[~keep], fam=[fam[s] for s in np.flatnonzero(~keep)])
    loadings = str(tmp_path / "kept.npz")
    variants_pca.main(["--bed-path", kept_prefix, "--save-loadings", loadings])
    plain = _sample_lines(capsys.readouterr().out)
    for s in np.flatnonzero(keep):
        assert got[names[s]] == plain[names[s]]                        # textually identical: the same bits
    variants_pca.main(["--bed-path", rem_prefix, "--project-loadings", loadings])
    proj = _sample_lines(capsys.readouterr().out)
    pcs = lambda ln: np.array([float(x) for x in ln.split("\t")[2:4]])
    scale = np.abs(np.array([pcs(plain[names[s]]) for s in np.flatnonzero(keep)])).max(axis=0)
    for name in removed:
        assert (np.abs(pcs(got[name]) - pcs(proj[name])) <= 1e-12 * scale).all(), name
    with np.load(loadings) as f:
        assert int(f["n_samples"]) == m
    # --save-loadings in the cutoff run writes the same kept-set loadings as the kept-only run
    both = str(tmp_path / "both.npz")
    variants_pca.main(["--bed-path", prefix, "--king-cutoff", "0.0884", "--save-loadings", both])
    capsys.readouterr()
    with np.load(loadings) as a, np.load(both) as b:
        assert int(b["n_samples"]) == m
        np.testing.assert_array_equal(_bits(a["loadings"]), _bits(b["loadings"]))
        np.testing.assert_array_equal(a["count"], b["count"])
        np.testing.assert_array_equal(_bits(a["eigenvalues"]), _bits(b["eigenvalues"]))
