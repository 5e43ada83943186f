#!/usr/bin/env python
"""Time the linear association tests (vpca_glm_linear_bed) on the seeded Balding-Nichols .bed rows of tools/grm_bench.py
(1 % of the calls missing), with a phenotype of population mean (0, 0.5, 1) plus N(0, 1) noise and q - 1 N(0, 1)
covariates beside the intercept.  Workloads: 2504 x 1 048 576 and 21 845 x 65 536 rows, each at q = 11 and q = 32,
and 21 845 x 65 536 at q = 11 with about 30 % of the calls missing (the solve kernel's missing-call pass walks about
6500 samples per variant there).  Per workload: one warm-up call, then the host clock around glmLinearBed (it synchronises before it returns, and includes the
H2D copy of the rows from pageable memory), repeated; a separate torch.profiler run of the same call for the per-kernel
and H2D times; the FP64 floor N V (q + 1) FMAs at the H100 SXM data sheet's 34 TFLOP/s (FP64 without tensor cores: the
sums are FMA chains) and the byte floor (rows read once, sums written and read, outputs written, at 3.35 TB/s).  Prints
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

from grm_bench import _card, bn_rows
from spark_examples_b200 import native

FP64_TFLOPS = 34.0   # H100 SXM data sheet, dense FP64 (no tensor cores)
HBM_TBS = 3.35       # H100 SXM data sheet, HBM3
SUMS_DOUBLES = native.GLM_MAX_Q + 4


def kernel_of(name):
    for key in ("glm_count_kernel", "glm_sums_kernel", "glm_solve_kernel", "glm_finish_kernel", "Memcpy HtoD", "Memcpy DtoH"):
        if key in name:
            return key.replace("Memcpy ", "memcpy_").lower()
    return "other"


def with_missing(rows, n, rate, seed=9, block=4096):
    """rows with a further `rate` of the calls set missing (code 01) at random, on the GPU in blocks of variants."""
    gen = torch.Generator(device="cuda").manual_seed(seed)
    out = np.empty_like(rows)
    for v0 in range(0, rows.shape[0], block):
        r = torch.from_numpy(rows[v0:v0 + block]).cuda()
        for e in range(4):
            hit = (torch.rand(r.shape, generator=gen, device="cuda") < rate).to(torch.uint8)
            r = (r & ~(hit * (3 << (2 * e))).to(torch.uint8)) | (hit << (2 * e))
        out[v0:v0 + block] = r.cpu().numpy()
    return out


def phenotype(n, q, seed=5):
    rng = np.random.default_rng(seed)
    share = 1.12 ** np.arange(3)
    pop = np.minimum(np.searchsorted(np.cumsum(share / share.sum()) * n, np.arange(n), side="right"), 2)
    return np.array([0.0, 0.5, 1.0])[pop] + rng.normal(size=n), rng.normal(size=(n, q - 1))


def workload(rows, n, q, repeats=3):
    y, covar = phenotype(n, q)
    nv = rows.shape[0]
    with native.NativePca(n) as nat:
        nat.glmBegin(y, covar)
        _, err = nat.glmLinearBed(rows)                                                # warm-up
        times = []
        for _ in range(repeats):
            t0 = time.perf_counter()
            nat.glmLinearBed(rows)
            times.append(time.perf_counter() - t0)
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            nat.glmLinearBed(rows)
        per = defaultdict(float)
        for ev in prof.events():
            if ev.device_type == torch.autograd.DeviceType.CUDA:
                per[kernel_of(ev.name)] += getattr(ev, "device_time_total", 0.0) / 1e3
    kernels = sum(v for key, v in per.items() if key.startswith("glm_"))
    fmas = n * nv * (q + 1)
    nbytes = nv * ((n + 3) // 4) + nv * SUMS_DOUBLES * 8 * 2 + nv * (6 * 8 + 4)
    call = min(times)
    return {"n_samples": n, "variants": nv, "q": q, "call_s": [round(t, 4) for t in times],
            "kernel_ms": {key: round(v, 3) for key, v in sorted(per.items())},
            "kernels_total_ms": round(kernels, 3), "kernel_share_of_call": round(kernels * 1e-3 / call, 3),
            "fp64_floor_ms": round(2.0 * fmas / (FP64_TFLOPS * 1e12) * 1e3, 3),
            "byte_floor_ms": round(nbytes / (HBM_TBS * 1e12) * 1e3, 3),
            "errcodes": np.bincount(np.asarray(err), minlength=5).tolist()}


def main():
    name, power, clock = _card()
    out = {"card": name, "power_limit": power, "max_sm_clock": clock}
    for n, nv in ((2504, 1 << 20), (21845, 1 << 16)):
        rows = bn_rows(n, nv)
        for q in (11, 32):
            out[f"glm_{n}x{nv}_q{q}"] = workload(rows, n, q)
        if n == 21845:   # the missing-call pass at its widest: about 30 % of the calls missing, N / 2 of them per row
            out[f"glm_{n}x{nv}_q11_miss30"] = workload(with_missing(rows, n, 0.3), n, 11)
        del rows
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
