#!/usr/bin/env python
"""Time KING-robust kinship (vpca_kinship_bed / vpca_kinship_pairs) on seeded numpy .bed rows (uniform random 2-bit codes,
a quarter of them missing): one warm-up call, then the host clock around NativePca.kinshipBed (which synchronises before it
returns) and around NativePca.kinshipPairs.  Workloads "N x V" from KB_WORKLOADS (default 2504x1048576 and 21845x65536).
Prints one JSON line per workload: card, power limit, the plane Gram's SYRK operations 3N (3N + 1) V and their rate, the
H2D bytes of the rows, the pairs selected at --king-table-filter 0.0442 and the total count of all pairs."""
import ctypes
import json
import os
import subprocess
import sys
import time
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


def run(n, nv, name, power, threshold=0.0442):
    stride = (n + 3) // 4
    rows = np.random.default_rng(20240901).integers(0, 256, size=(nv, stride), dtype=np.uint8)
    ops = 3 * n * (3 * n + 1) * nv
    out = {"card": name, "power_limit": power, "n_samples": n, "variants": nv, "syrk_ops": float(ops),
           "h2d_bytes": int(nv * stride)}
    with native.NativePca(n) as nat:
        nat.kinshipBed(rows[: min(nv, 65536)])                     # warm-up: module load, tile list, stream-K split
        nat.kinshipPairs(threshold)
        nat.reset()
        h2d0 = nat.stats()["h2d_bytes"]
        t0 = time.perf_counter()
        nat.kinshipBed(rows)
        t1 = time.perf_counter()
        ids, _, _ = nat.kinshipPairs(threshold)
        t2 = time.perf_counter()
        total = ctypes.c_int64(0)
        rc = native.load_library().vpca_kinship_pairs(nat._h, float("-inf"), 0, None, None, None, ctypes.byref(total))
        t3 = time.perf_counter()
        if rc != native.VPCA_OK:
            raise native.VpcaError(rc, "count-only vpca_kinship_pairs failed")
        out.update({"kinship_bed_s": round(t1 - t0, 4), "syrk_tops": round(ops / (t1 - t0) / 1e12, 1),
                    "kinship_pairs_s": round(t2 - t1, 4), "pairs_selected": int(len(ids)), "filter": threshold,
                    "count_all_pairs_s": round(t3 - t2, 4), "all_pairs": int(total.value),
                    "h2d_bytes_counted": int(nat.stats()["h2d_bytes"] - h2d0)})
    print(json.dumps(out), flush=True)


def main():
    name, power = _card()
    for w in os.environ.get("KB_WORKLOADS", "2504x1048576,21845x65536").split(","):
        n, nv = (int(x) for x in w.split("x"))
        run(n, nv, name, power)


if __name__ == "__main__":
    main()
