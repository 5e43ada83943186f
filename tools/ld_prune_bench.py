#!/usr/bin/env python
"""Time LD pruning (vpca_ld_prune_bed) on a seeded .bed with planted LD blocks: every block of 8 variants copies one
founder row of random 2-bit codes (a quarter of them missing) and redraws a fifth of its bytes.  One contig, a variant every
2 kb, a 500 kb window (about 250 variants per window), r2 > 0.2.  One warm-up call on the first 65 536 variants, then the
host clock around NativePca.ldPruneBed (which synchronises before it returns), then a separate torch.profiler run of the
same call for the kernel time of each stage.  Workloads "N x V" from LD_WORKLOADS (default 2504x1048576 and
100000x65536, the second with the sample axis split into pieces).  Prints one JSON line per workload: card, power limit,
the chunk geometry, the plane Gram's SYRK operations R (R + 1) N per chunk (R = 3 C) and their rate over the call, the
H2D bytes, the kept variants and the in-LD pairs."""
import ctypes
import json
import os
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

SPACING_BP, WINDOW_KB, R2, BLOCK = 2000, 500, 0.2, 8


def _card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [x.strip() for x in q.split(",")]
        return name, power
    except Exception:
        return torch.cuda.get_device_name(0), "unknown"


def planted_rows(n, nv, seed=20240901):
    stride = (n + 3) // 4
    step = max(BLOCK, (1 << 26) // stride // BLOCK * BLOCK)       # variants generated at a time (64 MB of rows)
    rng = np.random.default_rng(seed)
    rows = np.empty((nv, stride), np.uint8)
    for v0 in range(0, nv, step):
        v1 = min(nv, v0 + step)
        founders = rng.integers(0, 256, size=((v1 - v0 + BLOCK - 1) // BLOCK, stride), dtype=np.uint8)
        block = founders[(np.arange(v0, v1) - v0) // BLOCK]
        redraw = rng.random((v1 - v0, stride), dtype=np.float32) < 0.2
        block[redraw] = rng.integers(0, 256, size=int(redraw.sum()), dtype=np.uint8)
        rows[v0:v1] = block
    return rows


def geometry(nv, h):
    """Chunk size and count as vpca_ld_prune_bed chooses them (DESIGN.md 9)."""
    c = (max(2 * h, 1024) + 31) // 32 * 32
    if nv <= c:
        return (nv + 31) // 32 * 32, 1
    chunks, s = 1, 0
    while s + c < nv:
        s += c - h
        chunks += 1
    return c, chunks


def stage(name):
    for key in ("ld_planes", "ld_pairs", "ld_row_scan", "ld_sweep", "gram", "memset", "Memset", "Memcpy"):
        if key in name:
            return {"Memset": "memset", "Memcpy": "memcpy"}.get(key, key)
    return "other"


def run(n, nv, name, power):
    rows = planted_rows(n, nv)
    pos = np.arange(nv, dtype=np.int64) * SPACING_BP + 1
    lo = np.searchsorted(pos, pos - WINDOW_KB * 1000, side="left").astype(np.int64)
    h = int(np.max(np.arange(nv) - lo))
    c, chunks = geometry(nv, h)
    R = 3 * c
    ops = float(R) * (R + 1) * n * chunks
    out = {"card": name, "power_limit": power, "n_samples": n, "variants": nv, "window_variants": h, "chunk": c,
           "chunks": chunks, "r2_max": R2, "syrk_ops": ops}
    with native.NativePca(n) as nat:
        w = min(nv, 65536)
        nat.ldPruneBed(rows[:w], lo[:w], R2)                       # warm-up: module load, tile list, stream-K split
        h2d0 = nat.stats()["h2d_bytes"]
        t0 = time.perf_counter()
        keep, _, _ = nat.ldPruneBed(rows, lo, R2)
        t1 = time.perf_counter()
        h2d = int(nat.stats()["h2d_bytes"] - h2d0)
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            nat.ldPruneBed(rows, lo, R2)
        per = defaultdict(float)
        for ev in prof.events():
            if ev.device_type == torch.autograd.DeviceType.CUDA:
                per[stage(ev.name)] += getattr(ev, "device_time_total", 0.0) / 1e3
        t = t1 - t0
        total = ctypes.c_int64(0)
        k = np.zeros(nv, np.uint8)
        rc = native.load_library().vpca_ld_prune_bed(nat._h, rows.ctypes.data, nv, rows.shape[1], lo.ctypes.data, R2,
                                                     k.ctypes.data, 0, None, None, ctypes.byref(total))
        if rc != native.VPCA_OK:
            raise native.VpcaError(rc, "vpca_ld_prune_bed failed")
        out.update({"call_s": round(t, 4), "syrk_tops": round(ops / t / 1e12, 1), "h2d_bytes": h2d,
                    "kept": int(keep.sum()), "ld_pairs": int(total.value),
                    "stage_ms": {k: round(v, 2) for k, v in sorted(per.items())}})
    print(json.dumps(out), flush=True)


def main():
    name, power = _card()
    for wl in os.environ.get("LD_WORKLOADS", "2504x1048576,100000x65536").split(","):
        n, nv = (int(x) for x in wl.split("x"))
        run(n, nv, name, power)


if __name__ == "__main__":
    main()
