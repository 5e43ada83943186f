#!/usr/bin/env python
"""Time variant QC (vpca_variant_qc_bed, vpca_hwe_exact) on seeded data.  Rows are drawn from a pool of 2-bit .bed rows
at Hardy-Weinberg proportions (allele frequency uniform in [0.01, 0.5], 1 % missing calls), so the HWE loops have the
length of real common variants.  Per workload: one warm-up call on the first 4096 rows, then the host clock around the
call (which synchronises before it returns), then a separate torch.profiler run of the same call for the count kernel,
the HWE kernel and the copies.  Workloads: 2504 x 1 048 576 and 100 000 x 65 536 rows through NativePca.variantQcBed,
and the HWE kernel alone on 10^6 common-variant counts at N = 10^6 through NativePca.hweExact.  Prints one JSON line with
the card, its power limit and one entry per workload: the call time, the H2D bytes and their rate over the call, and the
kernel times."""
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


def hwe_rows(n, nv, pool, seed=20240901):
    """(nv, ceil(n / 4)) .bed rows, each a random row of a pool drawn at HWE."""
    rng = np.random.default_rng(seed)
    q = rng.uniform(0.01, 0.5, size=(pool, 1)).astype(np.float32)
    u = rng.random((pool, n), dtype=np.float32)
    codes = np.where(u < q * q, 0, np.where(u < q * q + 2 * q * (1 - q), 2, 3)).astype(np.uint8)
    codes[rng.random((pool, n), dtype=np.float32) < 0.01] = 1
    codes = np.concatenate([codes, np.zeros((pool, (-n) % 4), np.uint8)], axis=1).reshape(pool, -1, 4)
    packed = (codes[:, :, 0] | (codes[:, :, 1] << 2) | (codes[:, :, 2] << 4) | (codes[:, :, 3] << 6)).astype(np.uint8)
    return packed[rng.integers(0, pool, size=nv)]


def hwe_counts(n, nv, seed=7):
    """(nv, 4) counts of common variants (allele frequency in [0.05, 0.5]) at HWE, nothing missing."""
    rng = np.random.default_rng(seed)
    q = rng.uniform(0.05, 0.5, size=nv)
    het = rng.binomial(n, 2 * q * (1 - q))
    h2 = rng.binomial(n - het, (1 - q) ** 2 / ((1 - q) ** 2 + q * q))
    return np.stack([n - het - h2, het, h2, np.zeros(nv, np.int64)], axis=1).astype(np.int32)


def stage(name):
    for key in ("qc_count", "qc_hwe", "Memcpy HtoD", "Memcpy DtoH"):
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


def bed_workload(n, nv, pool):
    rows = hwe_rows(n, nv, pool)
    with native.NativePca(n) as nat:
        nat.variantQcBed(rows[:4096])                                       # warm-up: module load
        h2d0 = nat.stats()["h2d_bytes"]
        t, per = timed(lambda: nat.variantQcBed(rows))
        h2d = int(nat.stats()["h2d_bytes"] - h2d0) // 3                    # three calls since h2d0
        c, p = nat.variantQcBed(rows)
    return {"n_samples": n, "variants": nv, "call_s": round(t, 4), "h2d_bytes": h2d, "h2d_gbps": round(h2d / t / 1e9, 2),
            "kernel_ms": per, "hwe_p_below_1e-6": int((p < 1e-6).sum())}


def hwe_workload(n, nv):
    c = hwe_counts(n, nv)
    with native.NativePca(2) as nat:
        nat.hweExact(c[:4096])
        t, per = timed(lambda: nat.hweExact(c))
    return {"n_samples": n, "variants": nv, "call_s": round(t, 4), "kernel_ms": per}


def main():
    name, power = _card()
    out = {"card": name, "power_limit": power,
           "bed_2504x1048576": bed_workload(2504, 1 << 20, 4096),
           "bed_100000x65536": bed_workload(100000, 1 << 16, 512),
           "hwe_1000000x1000000": hwe_workload(10 ** 6, 10 ** 6)}
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
