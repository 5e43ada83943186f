#!/usr/bin/env python
"""Time vpca_compute_pca_subset (DESIGN.md 8) on a synthetic Gram (the device generator's binary carriers, 8192 variants)
with a seeded 10 % of the samples removed.  One warm-up call per workload, then REPS timed calls: CUDA events on the
context's stream around each call, and torch.profiler's device time of every kernel, summed per stage -- the Gram gather
(subset_gather_kernel), the placement of the samples (subset_scatter / _rho / _relatives_kernel) and the subset solve
(every other kernel of the call: centring and eigensolver).  Workloads "N" from KCB_SAMPLES (default 2504,21845), k from
KCB_K (default 2,16).  Prints one JSON line per (N, k) with the card and its power limit."""
import json
import os
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

import numpy as np
import torch
from torch.profiler import ProfilerActivity, profile

from spark_examples_b200 import native

REPS = 5


def _card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [x.strip() for x in q.split(",")]
        return name, power
    except Exception:
        return torch.cuda.get_device_name(0), "unknown"


def _stage(kernel_name):
    if "subset_gather_kernel" in kernel_name:
        return "gather"
    if "subset_" in kernel_name:
        return "place"
    return "solve"


def run(n, ks, name, power, nv=8192, panel=8192):
    stream = torch.cuda.Stream()
    keep = np.random.default_rng(n).random(n) >= 0.1
    m = int(keep.sum())
    with native.NativePca(n, stream=stream.cuda_stream) as nat:
        buf = torch.empty(nat.panelBytes(nv, panel), dtype=torch.uint8, device="cuda")
        nat.synthPanelsDevice(20240901, 0, nv, 0, buf.data_ptr(), panel)
        nat.accumulatePanels(buf.data_ptr(), nv, panel)
        nat.finalizeGram()
        nat.synchronize()
        del buf
        for k in ks:
            nat.computePcaSubset(keep, k)                               # warm-up: workspace, graphs, module load
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            call_ms = []
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(REPS):
                    e0.record(stream)
                    nat.computePcaSubset(keep, k)
                    e1.record(stream)
                    e1.synchronize()
                    call_ms.append(e0.elapsed_time(e1))
            stages = {"gather": 0.0, "place": 0.0, "solve": 0.0}
            for ev in prof.key_averages():
                if ev.device_type == torch.autograd.DeviceType.CUDA and not ev.key.startswith("Memcpy") \
                        and not ev.key.startswith("Memset"):
                    stages[_stage(ev.key)] += ev.device_time_total / 1e3 / REPS
            st = nat.stats()
            print(json.dumps({"card": name, "power_limit": power, "n_samples": n, "kept": m, "removed": n - m, "k": k,
                              "call_ms_median": round(float(np.median(call_ms)), 3),
                              "gather_ms": round(stages["gather"], 3), "solve_ms": round(stages["solve"], 3),
                              "place_ms": round(stages["place"], 3), "eig_method": st["eig_method"],
                              "eig_iterations": st["eig_iterations"]}), flush=True)


def main():
    name, power = _card()
    ks = [int(x) for x in os.environ.get("KCB_K", "2,16").split(",")]
    for n in os.environ.get("KCB_SAMPLES", "2504,21845").split(","):
        run(int(n), ks, name, power)


if __name__ == "__main__":
    main()
