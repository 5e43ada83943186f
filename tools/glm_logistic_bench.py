#!/usr/bin/env python
"""Time the logistic association tests (vpca_glm_logistic_bed) on the workloads of tools/glm_bench.py: the seeded
Balding-Nichols .bed rows of tools/grm_bench.py at 2504 x 1 048 576 and 21 845 x 65 536, each at q = 11 and q = 32 with
1 % of the calls missing, and at q = 11 with 30 % missing; a case/control phenotype with a 30 % case rate (cases drawn at
random, so almost every variant is null) and q - 1 N(0, 1) covariates beside the intercept.  Per workload: one warm-up
call, then the host clock around glmLogisticBed (it synchronises before it returns, and includes the H2D copy of the
rows from pageable memory), repeated; a separate torch.profiler run of the same call for the per-kernel times; the mean
and largest Newton passes per variant; and the FP64 floor, sum over variants of passes N ((q + 1)(q + 2) / 2 + 2 (q + 1))
FMAs at the H100 SXM data sheet's 34 TFLOP/s (FP64 without tensor cores), with the Newton kernel's share of it.  Prints
one JSON line with the card and its power limit, read in the same run."""
import json
import sys
import time
from collections import defaultdict
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tools"))

import numpy as np
import torch

from glm_bench import with_missing
from grm_bench import _card, bn_rows
from spark_examples_b200 import native

FP64_TFLOPS = 34.0   # H100 SXM data sheet, dense FP64 (no tensor cores)


def kernel_of(name):
    for key in ("glm_count_kernel", "glm_logistic_kernel", "glm_logistic_finish_kernel", "Memcpy HtoD", "Memcpy DtoH"):
        if key in name:
            return key.replace("Memcpy ", "memcpy_").lower()
    return "other"


def phenotype(n, q, seed=5):
    rng = np.random.default_rng(seed)
    return (rng.random(n) < 0.3).astype(np.float64), rng.normal(size=(n, q - 1))


def workload(rows, n, q, repeats=2):
    y, covar = phenotype(n, q)
    with native.NativePca(n) as nat:
        nat.glmLogisticBegin(y, covar)
        _, err, passes = nat.glmLogisticBed(rows)                                      # warm-up
        times = []
        for _ in range(repeats):
            t0 = time.perf_counter()
            nat.glmLogisticBed(rows)
            times.append(time.perf_counter() - t0)
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            nat.glmLogisticBed(rows)
        per = defaultdict(float)
        for ev in prof.events():
            if ev.device_type == torch.autograd.DeviceType.CUDA:
                per[kernel_of(ev.name)] += getattr(ev, "device_time_total", 0.0) / 1e3
    kernels = sum(v for key, v in per.items() if key.startswith("glm_"))
    fmas = float(passes.astype(np.int64).sum()) * n * ((q + 1) * (q + 2) / 2 + 2 * (q + 1))
    floor_ms = 2.0 * fmas / (FP64_TFLOPS * 1e12) * 1e3
    fitted = passes[passes > 0]
    return {"n_samples": n, "variants": rows.shape[0], "q": q, "call_s": [round(t, 4) for t in times],
            "kernel_ms": {key: round(v, 3) for key, v in sorted(per.items())},
            "kernels_total_ms": round(kernels, 3),
            "passes_mean": round(float(fitted.mean()), 3) if len(fitted) else 0.0,
            "passes_max": int(passes.max()) if len(passes) else 0,
            "fp64_floor_ms": round(floor_ms, 3),
            "floor_share_of_newton_kernel": round(floor_ms / per["glm_logistic_kernel"], 3)
            if per["glm_logistic_kernel"] else None,
            "errcodes": np.bincount(np.asarray(err), minlength=6).tolist()}


def main():
    name, power, clock = _card()
    out = {"card": name, "power_limit": power, "max_sm_clock": clock}
    for n, nv in ((2504, 1 << 20), (21845, 1 << 16)):
        rows = bn_rows(n, nv)
        for q in (11, 32):
            out[f"logistic_{n}x{nv}_q{q}"] = workload(rows, n, q)
            print(json.dumps({f"logistic_{n}x{nv}_q{q}": out[f"logistic_{n}x{nv}_q{q}"]}), file=sys.stderr, flush=True)
        key = f"logistic_{n}x{nv}_q11_miss30"
        out[key] = workload(with_missing(rows, n, 0.3), n, 11)
        print(json.dumps({key: out[key]}), file=sys.stderr, flush=True)
        del rows
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
