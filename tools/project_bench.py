#!/usr/bin/env python
"""Time the loadings and projection kernels alone on a device-resident cohort: 2504 samples x 1 M int8 variants in
the panel layout (8192-variant panels), k = 2 and k = 16.  Prints one JSON line: card, power limit, median kernel ms
from CUDA events over warmed launches, GB/s of genotype cells read against the 3.35 TB/s data-sheet HBM3 figure, and
an output checksum (sum of the outputs; equal between runs, the kernels sum in a fixed order)."""
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


def main():
    n = int(os.environ.get("PB_N", "2504"))
    nv = int(os.environ.get("PB_V", str(1 << 20)))
    reps, warmup, panel = int(os.environ.get("PB_REPS", "20")), 3, 8192
    ks = [int(x) for x in os.environ.get("PB_K", "2,16").split(",")]
    ts = torch.cuda.Stream()
    torch.cuda.set_stream(ts)
    name, power, clock = _card()
    out = {"card": name, "power_limit": power, "max_sm_clock": clock, "n_samples": n, "variants": nv, "dtype": "int8",
           "panel": panel, "launches_timed": reps, "peak_gbs": PEAK_GBS}
    cell_bytes = n * ((nv + panel - 1) // panel) * panel
    with native.NativePca(n, stream=ts.cuda_stream, num_pc=16) as nat:
        X = torch.empty(nat.panelBytes(nv, panel), dtype=torch.uint8, device="cuda")
        nat.synthPanelsDevice(20240901, 0, nv, 0, X.data_ptr(), panel)
        nat.accumulatePanels(X.data_ptr(), nv, panel)
        nat.finalizeGram()
        _, evals, _ = nat.computePca(16)
        with native.NativePca(n, stream=ts.cuda_stream) as proj:
            for k in ks:
                w = torch.empty((nv, k), dtype=torch.float64, device="cuda")
                cnt = torch.empty(nv, dtype=torch.int32, device="cuda")
                ms_l = _median_ms(lambda: nat.loadingsPanels(k, X.data_ptr(), nv, panel, w.data_ptr(), cnt.data_ptr()),
                                  reps, warmup)
                mean = cnt.double() / n
                proj.projectBegin(k)
                ms_p = _median_ms(lambda: proj.projectPanels(X.data_ptr(), nv, panel, w.data_ptr(), mean.data_ptr()),
                                  reps, warmup)
                proj.projectBegin(k)
                proj.projectPanels(X.data_ptr(), nv, panel, w.data_ptr(), mean.data_ptr())
                P = proj.projectGet(evals[:k])
                for kind, ms in (("loadings", ms_l), ("project", ms_p)):
                    gbs = cell_bytes / (ms * 1e-3) / 1e9
                    out[f"{kind}_k{k}_ms"] = round(ms, 4)
                    out[f"{kind}_k{k}_gbs"] = round(gbs, 1)
                    out[f"{kind}_k{k}_of_peak"] = round(gbs / PEAK_GBS, 3)
                out[f"checksum_k{k}"] = [float(w.sum().item()), int(cnt.sum().item()), float(np.sum(P))]
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
