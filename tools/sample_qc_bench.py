#!/usr/bin/env python
"""Time sample QC (vpca_sample_missing_bed, vpca_subset_bed_samples) on seeded data.  Rows are drawn from a pool of random
2-bit .bed rows with 1 % missing calls; 10 % of the samples, chosen at random, are removed by the subset.  Per workload
and call: one warm-up call, then the host clock around the call (which synchronises before it returns), then a separate
torch.profiler run of the same call for the kernel and the copies.  Workloads: 2504 x 1 048 576 and 100 000 x 65 536
rows, both calls on a 2-sample context as the driver runs them.  Prints one JSON line with the card, its power limit and
one entry per workload and call: the call time, the profiled H2D / D2H copy and kernel times, and the bytes moved."""
import json
import subprocess
import sys
import time
from collections import defaultdict
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

import numpy as np
import torch

from spark_examples_b200 import native


def _card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [x.strip() for x in q.split(",")]
        return name, power
    except Exception:
        return torch.cuda.get_device_name(0), "unknown"


def rows_1pct_missing(n, nv, pool, seed=20240901):
    """(nv, ceil(n / 4)) .bed rows, each a random row of a pool of uniform called codes with 1 % missing calls."""
    rng = np.random.default_rng(seed)
    codes = rng.choice(np.array([0, 2, 3], np.uint8), size=(pool, n))
    codes[rng.random((pool, n), dtype=np.float32) < 0.01] = 1
    codes = np.concatenate([codes, np.zeros((pool, (-n) % 4), np.uint8)], axis=1).reshape(pool, -1, 4)
    packed = (codes[:, :, 0] | (codes[:, :, 1] << 2) | (codes[:, :, 2] << 4) | (codes[:, :, 3] << 6)).astype(np.uint8)
    return packed[rng.integers(0, pool, size=nv)]


def stage(name):
    for key in ("sample_missing", "subset_samples", "Memcpy HtoD", "Memcpy DtoH"):
        if key in name:
            return key.replace("Memcpy ", "memcpy_").lower()
    return "other"


def timed(call):
    call()
    t0 = time.perf_counter()
    call()
    t = time.perf_counter() - t0
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        call()
    per = defaultdict(float)
    for ev in prof.events():
        if ev.device_type == torch.autograd.DeviceType.CUDA:
            per[stage(ev.name)] += getattr(ev, "device_time_total", 0.0) / 1e3
    return t, {k: round(v, 3) for k, v in sorted(per.items())}


def workload(n, nv, pool):
    rows = rows_1pct_missing(n, nv, pool)
    rng = np.random.default_rng(3)
    keep = np.sort(rng.choice(n, size=n - n // 10, replace=False))
    out = {"n_samples": n, "variants": nv, "kept": len(keep), "in_bytes": int(rows.nbytes)}
    with native.NativePca(2) as nat:
        t, per = timed(lambda: nat.sampleMissingBed(rows, n))
        miss = nat.sampleMissingBed(rows, n)
        out["missing"] = {"call_s": round(t, 4), "gpu_ms": per, "mean_f_miss": round(float(miss.mean()) / nv, 5)}
        t, per = timed(lambda: nat.subsetBedSamples(rows, n, keep))
        sub = nat.subsetBedSamples(rows, n, keep)
        out["subset"] = {"call_s": round(t, 4), "gpu_ms": per, "out_bytes": int(sub.nbytes),
                         "copy_gb_per_s": round((rows.nbytes + sub.nbytes) / t / 1e9, 2)}
    return out


def main():
    name, power = _card()
    out = {"card": name, "power_limit": power,
           "bed_2504x1048576": workload(2504, 1 << 20, 4096),
           "bed_100000x65536": workload(100000, 1 << 16, 512)}
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
