#!/usr/bin/env python
"""Time the loadings and projection kernels alone on device-resident cohorts, one workload on each side of the loadings'
split threshold (65 535 samples), int8 cells in the panel layout (8192-variant panels), k = 2 and k = 16:
  * 2504 samples x 1 M variants (U from vpca_compute_pca of the same cells): loadings and projection;
  * 100 000 samples x 62 500 variants -- one owner-flush rank's share of configs[3] -- with U from a band solve
    (vpca_compute_pca_bands on two owner-computes band contexts whose Gram holds a 20-population cohort of 2048 variants,
    so that 16 components are separated): loadings only (projection runs in an ordinary context of the new cohort).
Both loadings kernels are timed at both sizes (VPCA_LOADINGS_KERNEL=whole|split; "default" is what the library picks).
Prints one JSON line per workload: card, power limit and max SM clock, median kernel ms from CUDA events over warmed
launches, GB/s of genotype cells read against the 3.35 TB/s data-sheet HBM3 figure, and output checksums (sums of the
outputs; equal between runs, the kernels sum in a fixed order)."""
import json
import os
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

import numpy as np
import torch

from spark_examples_b200 import native

PEAK_GBS = 3350.0
PANEL = 8192


def _card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = [x.strip() for x in q.split(",")]
        return name, power, clock
    except Exception:
        return torch.cuda.get_device_name(0), "unknown", "unknown"


def _median_ms(fn, reps, warmup):
    for _ in range(warmup):
        fn()
    times = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b))
    return float(np.median(times))


def _put(out, key, ms, cell_bytes):
    gbs = cell_bytes / (ms * 1e-3) / 1e9
    out[f"{key}_ms"] = round(ms, 4)
    out[f"{key}_gbs"] = round(gbs, 1)
    out[f"{key}_of_peak"] = round(gbs / PEAK_GBS, 3)


def _time_loadings(nat, X, nv, k, reps, warmup, out, cell_bytes):
    """both kernels and the default; the default's output is kept for the checksum, and must equal its kernel's bits"""
    w = torch.empty((nv, k), dtype=torch.float64, device="cuda")
    cnt = torch.empty(nv, dtype=torch.int32, device="cuda")
    bits = {}
    for kind in ("whole", "split", "default"):
        if kind == "default":
            os.environ.pop("VPCA_LOADINGS_KERNEL", None)
        else:
            os.environ["VPCA_LOADINGS_KERNEL"] = kind
        ms = _median_ms(lambda: nat.loadingsPanels(k, X.data_ptr(), nv, PANEL, w.data_ptr(), cnt.data_ptr()), reps, warmup)
        nat.synchronize()
        bits[kind] = w.clone()
        _put(out, f"loadings_{kind}_k{k}", ms, cell_bytes)
    os.environ.pop("VPCA_LOADINGS_KERNEL", None)
    out[f"default_kernel_k{k}"] = "split" if torch.equal(bits["default"], bits["split"]) else "whole"
    out[f"whole_vs_split_max_rel_k{k}"] = float(((bits["whole"] - bits["split"]).abs().amax(dim=0) /
                                                 bits["split"].abs().amax(dim=0)).max())
    return w, cnt


def small(name, power, clock, reps, warmup):
    n, nv, ks = 2504, 1 << 20, (2, 16)
    out = {"workload": "small", "card": name, "power_limit": power, "max_sm_clock": clock, "n_samples": n, "variants": nv,
           "dtype": "int8", "panel": PANEL, "launches_timed": reps, "peak_gbs": PEAK_GBS}
    cell_bytes = n * ((nv + PANEL - 1) // PANEL) * PANEL
    ts = torch.cuda.current_stream()
    with native.NativePca(n, stream=ts.cuda_stream, num_pc=16) as nat:
        X = torch.empty(nat.panelBytes(nv, PANEL), dtype=torch.uint8, device="cuda")
        nat.synthPanelsDevice(20240901, 0, nv, 0, X.data_ptr(), PANEL)
        nat.accumulatePanels(X.data_ptr(), nv, PANEL)
        nat.finalizeGram()
        _, evals, _ = nat.computePca(16)
        with native.NativePca(n, stream=ts.cuda_stream) as proj:
            for k in ks:
                w, cnt = _time_loadings(nat, X, nv, k, reps, warmup, out, cell_bytes)
                mean = cnt.double() / n
                proj.projectBegin(k)
                ms_p = _median_ms(lambda: proj.projectPanels(X.data_ptr(), nv, PANEL, w.data_ptr(), mean.data_ptr()),
                                  reps, warmup)
                _put(out, f"project_k{k}", ms_p, cell_bytes)
                proj.projectBegin(k)
                proj.projectPanels(X.data_ptr(), nv, PANEL, w.data_ptr(), mean.data_ptr())
                Pr = proj.projectGet(evals[:k])
                out[f"checksum_k{k}"] = [float(w.sum().item()), int(cnt.sum().item()), float(np.sum(Pr))]
    print(json.dumps(out), flush=True)


def _structured_panels(n, nv, pops, seed):
    """(n samples, nv variants) carriers of `pops` populations (shares 1.12^i, allele frequencies drawn independently
    per population from U(0.05, 0.5)) in the panel layout on cuda:0"""
    g = torch.Generator(device="cuda").manual_seed(seed)
    share = 1.12 ** torch.arange(pops, dtype=torch.float64)
    ends = torch.round(torch.cumsum(share, 0) / share.sum() * n).long().tolist()
    freq = 0.05 + 0.45 * torch.rand((pops, nv), generator=g, device="cuda", dtype=torch.float64)
    X = torch.empty((n, nv), dtype=torch.int8, device="cuda")
    row = 0
    for i, end in enumerate(ends):
        carrier = 1.0 - (1.0 - freq[i]) ** 2
        X[row:end] = (torch.rand((end - row, nv), generator=g, device="cuda", dtype=torch.float64) < carrier).to(torch.int8)
        row = end
    npan = -(-nv // PANEL)
    buf = torch.zeros((npan, n, PANEL), dtype=torch.int8, device="cuda")
    for p in range(npan):
        v1 = min(nv, (p + 1) * PANEL)
        buf[p, :, : v1 - p * PANEL] = X[:, p * PANEL:v1]
    return buf.view(torch.uint8).reshape(-1)


def large(name, power, clock, reps, warmup):
    n, nv, ks, world = 100_000, 62_500, (2, 8, 16), 2
    out = {"workload": "large", "card": name, "power_limit": power, "max_sm_clock": clock, "n_samples": n, "variants": nv,
           "dtype": "int8", "panel": PANEL, "launches_timed": reps, "peak_gbs": PEAK_GBS,
           "u_from": "vpca_compute_pca_bands, 2 owner-computes bands, 20 populations x 2048 variants"}
    free = torch.cuda.mem_get_info()[0]
    if free < 50 * 2 ** 30:
        out["skipped"] = f"needs 50 GB of free HBM, {free / 2 ** 30:.1f} GB free"
        print(json.dumps(out), flush=True)
        return
    cell_bytes = n * ((nv + PANEL - 1) // PANEL) * PANEL
    ts = torch.cuda.current_stream()
    bands = native.ownerRowBands(n, world)
    ctxs = []
    try:
        G = _structured_panels(n, 2048, 20, 7)
        for b in bands:
            ctxs.append(native.NativePca(n, stream=ts.cuda_stream, max_multiplicity=1, num_pc=16, gram_band=b))
        for c in ctxs:
            c.accumulatePanels(G.data_ptr(), 2048, PANEL)
            c.finalizeGram()
        del G
        _, evals, _ = native.computePcaBands(ctxs, 16)
        out["band_solve_lanczos_steps"] = ctxs[0].stats()["eig_iterations"]
        nat = ctxs[0]                                                 # a band-only context (rank 0 of the solve)
        X = torch.empty(nat.panelBytes(nv, PANEL), dtype=torch.uint8, device="cuda")
        nat.synthPanelsDevice(20240901, 0, nv, 0, X.data_ptr(), PANEL)
        for k in ks:
            w, cnt = _time_loadings(nat, X, nv, k, reps, warmup, out, cell_bytes)
            out[f"checksum_k{k}"] = [float(w.sum().item()), int(cnt.sum().item())]
    finally:
        for c in ctxs:
            c.close()
    print(json.dumps(out), flush=True)


def main():
    reps, warmup = int(os.environ.get("PB_REPS", "20")), 3
    torch.cuda.set_stream(torch.cuda.Stream())        # the contexts run on torch's current stream, events time it
    name, power, clock = _card()
    which = os.environ.get("PB_WORKLOADS", "small,large").split(",")
    if "small" in which:
        small(name, power, clock, reps, warmup)
    if "large" in which:
        large(name, power, clock, reps, warmup)


if __name__ == "__main__":
    main()
