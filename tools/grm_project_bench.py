#!/usr/bin/env python
"""Time the GRM loadings and projection kernels (vpca_grm_loadings_bed, vpca_grm_project_bed; DESIGN.md 14) on the seeded
Balding-Nichols .bed rows of tools/grm_bench.py.  Workloads: 2504 x 1 048 576 and 21 845 x 65 536 rows, each at k = 2
and k = 16.  U comes from a GRM of the first 65 536 rows (the kernels' work does not depend on U's values).  Per
workload and call: one warm-up call, the host clock around a call (it synchronises before it returns, so this includes
the H2D copy of the rows from pageable memory), and a separate torch.profiler run of one call for the device time of
each kernel and of the H2D copies.  Each kernel time is set against two floors: its bytes (the rows, plus the tables and
w the projection reads) at the 3.35 TB/s HBM3 figure, and its N V k FMAs at the 34 TFLOP/s (17e12 FMA/s) vector FP64
figure of the H100 SXM data sheet.  Prints one JSON line with the card, its power limit and maximum SM clock, read in the
same run."""
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

HBM_BYTES_S = 3.35e12
FP64_FMA_S = 17e12


def kernel_of(name):
    for key in ("grm_loadings_kernel", "grm_project_reduce_kernel", "grm_project_kernel", "grm_table_kernel", "qc_count",
                "Memcpy HtoD", "Memcpy DtoH"):
        if key in name:
            return key.replace("Memcpy ", "memcpy_").lower()
    return "other"


def profiled(fn):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
    per = defaultdict(float)
    for ev in prof.events():
        if ev.device_type == torch.autograd.DeviceType.CUDA:
            per[kernel_of(ev.name)] += getattr(ev, "device_time_total", 0.0) / 1e3
    return per


def timed(fn, repeats=2):
    fn()
    times = []
    for _ in range(repeats):
        t0 = time.perf_counter()
        fn()
        times.append(time.perf_counter() - t0)
    return times


def floors(n, nv, k, extra_bytes=0):
    byte_ms = (nv * ((n + 3) // 4) + extra_bytes) / HBM_BYTES_S * 1e3
    fp64_ms = n * nv * k / FP64_FMA_S * 1e3
    return round(byte_ms, 3), round(fp64_ms, 3)


def workload(n, nv, ks=(2, 16)):
    rows = bn_rows(n, nv)
    out = {"n_samples": n, "variants": nv}
    with native.NativePca(n, num_pc=16) as ref, native.NativePca(n, num_pc=2) as new:
        ref.grmBed(rows[: 1 << 16])
        ref.grmFinalize()
        ref.computePcaGrm(16)
        for k in ks:
            w, tab = ref.grmLoadingsBed(k, rows)

            def project():
                new.projectBegin(k)
                new.projectGrmBed(rows, tab, w)
                new.projectGet(np.ones(k))
            res = {}
            for name, fn, kern, extra in (
                    ("loadings", lambda: ref.grmLoadingsBed(k, rows), "grm_loadings_kernel", 0),
                    ("projection", project, "grm_project_kernel", nv * (k + 4) * 8)):
                host = timed(fn)
                per = profiled(fn)
                kms = per[kern]
                byte_ms, fp64_ms = floors(n, nv, k, extra)
                res[name] = {"call_s": [round(t, 4) for t in host], "kernel_ms": round(kms, 3),
                             "device_ms": {key: round(v, 3) for key, v in sorted(per.items())},
                             "byte_floor_ms": byte_ms, "fp64_floor_ms": fp64_ms,
                             "share_of_fp64_floor": round(fp64_ms / kms, 3) if kms else None,
                             "share_of_byte_floor": round(byte_ms / kms, 3) if kms else None}
            out[f"k{k}"] = res
    return out


def main():
    assert torch.cuda.is_available(), "this benchmark measures the GPU; none is visible"
    name, power, clock = _card()
    out = {"card": name, "power_limit": power, "max_sm_clock": clock,
           "grm_project_2504x1048576": workload(2504, 1 << 20),
           "grm_project_21845x65536": workload(21845, 1 << 16)}
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
