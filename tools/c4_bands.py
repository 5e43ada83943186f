#!/usr/bin/env python
"""BASELINE configs[3] on all GPUs of one box (two forms, --mode): 100 000 samples x 500 000 variants, the 40 GB int32 Gram held ONCE across the
box as row bands (rank q allocates only the rows it owns: 5 GB at 8 GPUs), variants sharded over the GPUs
(`for (c1 <- callset; c2 <- callset) matrix(c1, c2) += 1`, VariantsPca.scala:186-188, one partition matrix per GPU, with the
sizing note of :176-177 answered by never materialising a second copy).  One process drives every GPU -- the process model of
the reference's `local[*]` driver JVM (VariantsPca.scala:38-50) -- through vpca_gram_set_peers_local: every Gram kernel's
epilogue adds its tile straight into the band of the rank that owns the row (red.relaxed.sys over NVLink), so there is no
reduce step and no gather; the bands ARE the result.  `--mode owner-computes` is the other form SURVEY 8e names: every GPU
holds ALL variants (50 GB of int8 genotypes) and its Gram kernel enumerates only the tiles of the rows it stores -- no peers,
no traffic between the GPUs at all.

Times the Gram launches with CUDA events per device (max over devices = the job), and checks without an N x N oracle:
  * diag(S) = carrier counts of the whole cohort, per band;
  * whole sampled rows of every band (its first, its last and random ones: the lower-triangle part, columns 0..row) and
    random 256 x 256 blocks against an exact fp32 matmul of the same shards (0/1 cells, counts < 2^24, TF32 off).
`--pca K` then computes the top K principal coordinates straight from the bands (vpca_compute_pca_bands: Lanczos with the
mat-vec sharded over the band contexts; no replica of S, no N x N FP64 matrix, no 65 535-sample limit) and reports
`pca_ms` (host clock around the call, which synchronises), `lanczos_steps`, and checks computed from the genotype shards,
not from S: the residual ||J X X^T J u_c - lambda_c u_c|| / lambda_1 of every pair in FP64 (panel by panel), and the
orthonormality of U.
`--loadings` (with --pca) then has every rank compute the variant loadings w = X^T U of the variants it holds
(vpca_loadings_panels on its band-only context, which holds U after the band solve; owner-computes ranks split the panels
between them), timed with CUDA events per rank, checked against FP64 X^T U from the genotype shards, and projects 4096
sampled reference samples in an ordinary 4096-sample context with those loadings: they must come back to their rows of U.

`--gpus N` sets the number of band contexts (ranks); with fewer visible devices they share them round robin (8 band
contexts on one H100 hold the 40 GB Gram of config 4, but not its 50 GB of genotypes as well: lower --variants there)."""
import argparse
import json
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
import numpy as np
import torch
from spark_examples_b200 import native


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--samples", type=int, default=100_000)
    ap.add_argument("--variants", type=int, default=500_000, help="whole cohort; split evenly over the GPUs")
    ap.add_argument("--gpus", type=int, default=0, help="band contexts (ranks); 0 = one per visible device; more than the "
                    "visible devices share them round robin")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--panel", type=int, default=8192)
    ap.add_argument("--check-rows", type=int, default=3, help="sampled whole rows per band checked against fp32 matmul")
    ap.add_argument("--mode", choices=["owner-flush", "owner-computes"], default="owner-flush",
                    help="owner-flush: every GPU holds a variant shard and its kernel adds each tile into the band of the row's "
                         "owner over NVLink; owner-computes: every GPU holds ALL variants and computes only its own band (no "
                         "traffic between GPUs at all; 50 GB of genotypes per GPU)")
    ap.add_argument("--pca", type=int, default=0, help="K > 0: also compute the top K principal coordinates from the bands "
                    "(vpca_compute_pca_bands) and check them against the genotype shards")
    ap.add_argument("--loadings", action="store_true", help="with --pca: every rank computes the loadings of its variants; "
                    "checked against FP64 X^T U, and 4096 sampled reference samples projected back onto U")
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    if args.loadings and args.pca <= 0:
        ap.error("--loadings needs --pca K")
    world = args.gpus or torch.cuda.device_count()
    ndev = torch.cuda.device_count()
    devs = [r % ndev for r in range(world)]
    n, P = args.samples, args.panel
    computes = args.mode == "owner-computes"
    per = args.variants if computes else (args.variants + world - 1) // world
    bands = native.ownerRowBands(n, world)
    ctxs, bufs, streams = [], [], []
    total_v = per if computes else per * world
    report = {"config": f"{n} samples x {total_v} variants, {world} band context(s) on {len(set(devs))} GPU(s), one process, "
                        f"band-only Grams, {args.mode}",
              "n": n, "variants_per_gpu": per, "world": world, "panel": P,
              "band_rows": [b[1] for b in bands], "band_gb": [round(b[1] * n * 4 / 2 ** 30, 2) for b in bands]}
    try:
        for r in range(world):
            torch.cuda.set_device(devs[r])
            s = torch.cuda.Stream(device=devs[r])
            streams.append(s)
            ctxs.append(native.NativePca(n, device=devs[r], stream=s.cuda_stream, max_multiplicity=1, num_pc=max(2, args.pca),
                                         gram_band=bands[r]))
        if not computes:
            native.setPeersLocal(ctxs, "owner_rows")
        for r, c in enumerate(ctxs):
            torch.cuda.set_device(devs[r])
            buf = torch.zeros(c.panelBytes(per, P), dtype=torch.uint8, device=f"cuda:{devs[r]}")
            # the zeros are written on torch's stream, the cells on the context's own non-blocking stream: without this
            # wait the two race, and zeros landing after the cells leave the ranks' copies of the cohort different
            torch.cuda.synchronize(devs[r])
            bufs.append(buf)
            c.synthPanelsDevice(20240901, 0 if computes else r * per, per, 0, buf.data_ptr(), P)
        for c in ctxs:
            c.synchronize()
        times = []
        for rep in range(args.reps + 1):
            for c in ctxs:
                c.reset()
            for c in ctxs:
                c.synchronize()       # every band is zero before any rank adds into it
            ev = []
            for r, c in enumerate(ctxs):
                torch.cuda.set_device(devs[r])
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                with torch.cuda.stream(streams[r]):
                    a.record()
                    c.accumulatePanels(bufs[r].data_ptr(), per, P)
                    b.record()
                ev.append((a, b))
            if not computes:
                for c in ctxs:
                    c.gatherGram()    # closing all-rank barrier on every stream: all remote adds have landed
            for c in ctxs:
                c.synchronize()
            per_dev = [a.elapsed_time(b) for a, b in ev]
            if rep:
                times.append(per_dev)
        ms_dev = np.median(np.array(times), axis=0)
        ms = float(ms_dev.max())
        ops = float(n) * (n + 1) * total_v
        st = [c.stats() for c in ctxs]
        report.update({
            "gram_ms_per_device_median": [round(float(x), 2) for x in ms_dev],
            "gram_ms_job": round(ms, 2),
            "cells_per_s": n * total_v / (ms * 1e-3),
            "syrk_tops_per_gpu": round(ops / world / (ms * 1e-3) / 1e12, 1),
            "frac_of_nominal_int8_4500": round(ops / world / (ms * 1e-3) / 1e12 / 4500.0, 3),
            "resident_schedule": [s["gram_resident"] for s in st],
            # lower triangle of S, minus the part whose owner is the writer itself, crosses NVLink once per rank
            "remote_red_bytes_per_gpu_upper_bound": 0 if computes else int(n * (n + 1) // 2 * 4 * (world - 1) / world),
            "genotype_bytes_per_gpu": int(n) * int(per),
        })
        print(json.dumps(dict(report, checks="pending")), flush=True)     # the timings survive a failure in the checks below
        if args.out:
            Path(args.out).write_text(json.dumps(dict(report, checks="pending")) + "\n")
        # ---- checks: the rows of X on one device as fp32 (6.25 GB per 62 500-variant shard would be 25 GB as fp32, so
        #      the reference values are computed shard by shard from the int8 panels)
        npan = (per + P - 1) // P

        def shard_rows(r, rows):
            """int8 panels of shard r restricted to `rows` -> (len(rows), npan * P) fp32 on device r"""
            x = bufs[r].view(torch.int8)[: npan * n * P].view(npan, n, P)
            sel = x[:, rows, :]                                            # slice or index list
            return sel.permute(1, 0, 2).reshape(sel.shape[1], npan * P).to(torch.float32)

        shard_devs = [0] if computes else list(range(world))     # owner-computes: every rank holds the whole cohort
        carriers = torch.zeros(n, dtype=torch.int64)
        for r in shard_devs:
            x = bufs[r].view(torch.int8)[: npan * n * P].view(npan, n, P)
            for p_ in range(npan):                                   # panel by panel: the int64 sum of a whole shard would not fit
                carriers += (x[p_] != 0).sum(dim=1).cpu()
        ok_diag, ok_rows, ok_blocks = True, True, True
        rng = np.random.default_rng(7)
        for q, c in enumerate(ctxs):
            row0, rows = bands[q]
            pick = sorted({row0, row0 + rows - 1} | set(int(v) for v in rng.integers(row0, row0 + rows, args.check_rows)))
            got = {row: c.gramBand(row, 1)[0] for row in pick}
            for row in pick:
                ok_diag = ok_diag and int(got[row][row]) == int(carriers[row])
            want = {row: torch.zeros(row + 1, dtype=torch.float64) for row in pick}
            for r in shard_devs:
                torch.cuda.set_device(devs[r])
                xr = shard_rows(r, pick)                                   # (len(pick), K)
                for r0 in range(0, max(pick) + 1, 8192):             # columns beyond the last sampled row are never needed
                    r1 = min(n, r0 + 8192)
                    blk = (xr @ shard_rows(r, slice(r0, r1)).t()).to(torch.float64).cpu()   # exact: counts < 2^24
                    for i, row in enumerate(pick):
                        hi = min(r1, row + 1)
                        if hi > r0:
                            want[row][r0:hi] += blk[i, : hi - r0]
            for row in pick:
                ok_rows = ok_rows and bool(np.array_equal(got[row][: row + 1].astype(np.int64), want[row].numpy().astype(np.int64)))
            # one random 256 x 256 block strictly inside the band's lower-triangle part
            br = int(rng.integers(row0, max(row0 + 1, row0 + rows - 256)))
            bc = int(rng.integers(0, max(1, br - 256)))
            gb = c.gramBand(br, min(256, row0 + rows - br))[:, bc:bc + 256].astype(np.int64)
            wb = torch.zeros(gb.shape, dtype=torch.float64)
            for r in shard_devs:
                torch.cuda.set_device(devs[r])
                wb += (shard_rows(r, slice(br, br + gb.shape[0])) @ shard_rows(r, slice(bc, bc + gb.shape[1])).t()).to(torch.float64).cpu()
            ok_blocks = ok_blocks and bool(np.array_equal(gb, wb.numpy().astype(np.int64)))
        report["checks"] = {"diag_equals_carrier_counts": ok_diag, "sampled_rows_exact_vs_fp32_matmul": ok_rows,
                            "random_256_blocks_exact": ok_blocks, "rows_checked_per_band": args.check_rows + 2}
        if args.pca > 0:
            pcs, vecs, evals = principal_coordinates(args.pca, ctxs, bufs, devs, shard_devs, n, per, P)
            report.update(pcs)
            if args.loadings:
                report.update(loadings_and_projection(min(args.pca, 16), ctxs, bufs, devs, streams, computes, n, per, P,
                                                      vecs, evals))
    finally:
        for c in ctxs:
            try:
                c.synchronize()
            except Exception:
                pass
        for c in ctxs:
            c.close()
    line = json.dumps(report)
    print(line, flush=True)
    if args.out:
        Path(args.out).write_text(line + "\n")


def principal_coordinates(k, ctxs, bufs, devs, shard_devs, n, per, P):
    """Top-k PCs from the bands, timed on the host around the (synchronising) call, and checked against the genotypes:
    with JX the column-centred cells, (J X X^T J) U = JX ((JX)^T U) is accumulated in FP64, 1024 variants at a time."""
    import time
    for c in ctxs:
        c.finalizeGram()              # a band stays a band of the lower triangle: nothing is mirrored
    torch.cuda.set_device(devs[0])
    t0 = time.perf_counter()
    vecs, evals, nz = native.computePcaBands(ctxs, k)
    pca_ms = (time.perf_counter() - t0) * 1e3
    st = ctxs[0].stats()
    out = {"pca_k": k, "pca_ms": round(pca_ms, 1), "pca_device_ms": round(st["last_eig_ms"], 1),
           "lanczos_steps": st["eig_iterations"], "eigenvalues": [float(x) for x in evals], "non_zero_rows": nz}
    npan = (per + P - 1) // P
    CU = torch.zeros((n, k), dtype=torch.float64, device=f"cuda:{devs[0]}")
    for r in shard_devs:
        dev = f"cuda:{devs[r]}"
        torch.cuda.set_device(devs[r])
        U = torch.from_numpy(vecs).to(dev)
        acc = torch.zeros((n, k), dtype=torch.float64, device=dev)
        x = bufs[r].view(torch.int8)[: npan * n * P].view(npan, n, P)
        for p_ in range(npan):
            width = min(P, per - p_ * P)                              # cells of this panel that hold variants
            for b0 in range(0, width, 1024):
                b1 = min(b0 + 1024, width)
                xb = x[p_, :, b0:b1].to(torch.float64)
                xb -= xb.mean(dim=0, keepdim=True)                    # J X: every variant column centred over the samples
                acc += xb @ (xb.t() @ U)
        CU += acc.to(CU.device)
    torch.cuda.set_device(devs[0])
    U = torch.from_numpy(vecs).to(CU.device)
    lam = torch.from_numpy(evals).to(CU.device)
    res = (torch.linalg.vector_norm(CU - U * lam[None, :], dim=0) / lam[0]).cpu().numpy()
    orth = float((U.t() @ U - torch.eye(k, dtype=torch.float64, device=CU.device)).abs().max())
    out["pca_checks"] = {"residual_over_lambda1": [float(x) for x in res], "residuals_below_1e-9": bool(np.all(res <= 1e-9)),
                         "max_abs_UtU_minus_I": orth, "orthonormal_to_1e-10": orth <= 1e-10,
                         "descending_eigenvalues": bool(np.all(np.diff(evals) <= 0))}
    return out, vecs, evals


def loadings_and_projection(k, ctxs, bufs, devs, streams, computes, n, per, P, vecs, evals, m=4096):
    """Every rank's loadings of the variants it holds (owner-computes: panels split evenly between the ranks), the second
    of two launches timed with CUDA events on the rank's stream; FP64 X^T U of the same panels as the reference; then m sampled reference samples
    projected with the loadings in an ordinary m-sample context on device 0."""
    world = len(ctxs)
    npan = (per + P - 1) // P
    # (buffer rank, first panel, end panel) of the variants each rank computes
    if computes:
        parts = [(r, r * npan // world, (r + 1) * npan // world) for r in range(world)]
    else:
        parts = [(r, 0, npan) for r in range(world)]
    outs, ev = [], []
    for r, c in enumerate(ctxs):
        b, p0, p1 = parts[r]
        nv = max(0, min(per, p1 * P) - p0 * P)
        torch.cuda.set_device(devs[r])
        dev = f"cuda:{devs[r]}"
        w = torch.empty((max(nv, 1), k), dtype=torch.float64, device=dev)      # every row is written on the ctx stream
        cnt = torch.empty(max(nv, 1), dtype=torch.int32, device=dev)
        a, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        with torch.cuda.stream(streams[r]):
            # one untimed launch first: the first launch of a kernel in a process also loads its module
            c.loadingsPanels(k, bufs[b].data_ptr() + p0 * n * P, nv, P, w.data_ptr(), cnt.data_ptr())
            a.record()
            c.loadingsPanels(k, bufs[b].data_ptr() + p0 * n * P, nv, P, w.data_ptr(), cnt.data_ptr())
            e.record()
        outs.append((w[:nv], cnt[:nv], nv))
        ev.append((a, e))
    for c in ctxs:
        c.synchronize()
    ms = [a.elapsed_time(e) for a, e in ev]
    out = {"loadings_k": k, "loadings_ms_per_rank": [round(x, 2) for x in ms], "loadings_ms_job": round(max(ms), 2),
           "loadings_variants_per_rank": [o[2] for o in outs]}
    rel, counts_ok = 0.0, True
    rng = np.random.default_rng(11)
    pick = torch.from_numpy(np.sort(rng.choice(n, m, replace=False)))
    torch.cuda.set_device(devs[0])
    with native.NativePca(m, device=devs[0], max_multiplicity=1) as proj:
        proj.projectBegin(k)
        for r in range(world):
            b, p0, p1 = parts[r]
            w, cnt, nv = outs[r]
            if nv == 0:
                continue
            torch.cuda.set_device(devs[b])
            x = bufs[b].view(torch.int8)[: npan * n * P].view(npan, n, P)[p0:p1]
            U = torch.from_numpy(np.ascontiguousarray(vecs[:, :k])).to(x.device)
            want = torch.cat([x[q, :, b0:b0 + 1024].to(torch.float64).t() @ U                 # 1024 variants at a time
                              for q in range(p1 - p0) for b0 in range(0, P, 1024)])[:nv]
            cw = torch.cat([(x[q] != 0).sum(dim=0) for q in range(p1 - p0)])[:nv]
            got = w.to(want.device)
            rel = max(rel, float(((got - want).abs().amax(dim=0) / want.abs().amax(dim=0)).max()))
            counts_ok = counts_ok and bool(torch.equal(cnt.to(cw.device).to(torch.int64), cw.to(torch.int64)))
            y = x[:, pick.to(x.device), :].contiguous().to("cuda:%d" % devs[0])     # the sampled rows, same panels
            torch.cuda.set_device(devs[0])
            wy = got.to(y.device).contiguous()
            mean = (cnt.to(y.device).to(torch.float64) / n).contiguous()
            torch.cuda.synchronize()                          # the inputs are ready before the projection's own stream reads them
            proj.projectPanels(y.data_ptr(), nv, P, wy.data_ptr(), mean.data_ptr())
            proj.synchronize()
            del y, wy, mean
        P_got = proj.projectGet(evals[:k])
    u = vecs[pick.numpy(), :k]
    err = np.max(np.abs(P_got - u), axis=0) / np.max(np.abs(vecs[:, :k]), axis=0)
    out["loadings_checks"] = {"max_rel_err_vs_fp64_XtU": rel, "loadings_within_1e-12": rel <= 1e-12,
                              "counts_exact": counts_ok, "projected_samples": m,
                              "self_projection_err_over_max_u": [float(x) for x in err],
                              "self_projection_within_1e-9": bool(np.all(err <= 1e-9))}
    return out


main()
