#!/usr/bin/env python
"""Time the Firth-penalized logistic tests (vpca_glm_firth_bed) in both modes.  Workloads: those of
tools/glm_logistic_bench.py (seeded Balding-Nichols rows at 2504 x 1 048 576 and 21 845 x 65 536, q = 11 and 32 with 1 %
of the calls missing, q = 11 with 30 % missing, a 30 % case rate drawn at random), and a rare-variant workload on the
same rows: 30 % of them replaced by rows with 1 to 5 copies of A2 (on an A1 background) and a 10 % case rate, at q = 11
and 32.  Per workload and mode: one warm-up call, then the host clock around one glmFirthBed call (it synchronises before
it returns, and includes the H2D copy of the rows from pageable memory); a separate torch.profiler run for the per-kernel
times; the mean and largest passes of the Firth fits; and the FP64 floor of the Firth kernel, sum over its variants of
passes N ((q + 1)(q + 2) + 3 (q + 1)) FMAs (walk A's H and eta, walk B's hat diagonal, eta and score; a backtracked pass
runs walk A alone, so this is an upper bound of the work) at the H100 SXM data sheet's 34 TFLOP/s (FP64 without tensor
cores).  Prints one JSON line with the card, its power limit and its maximum SM clock, read in the same run."""
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
KERNELS = ("glm_count_kernel", "glm_logistic_kernel", "glm_firth_select_kernel", "glm_firth_kernel",
           "glm_logistic_finish_kernel")


def kernel_of(name):
    for key in KERNELS[::-1] + ("Memcpy HtoD", "Memcpy DtoH"):
        if key in name:
            return key.replace("Memcpy ", "memcpy_").lower()
    return "other"


def rare(rows, n, share=0.3, seed=3):
    """rows with `share` of them (at random) replaced by 1 to 5 A2 copies, as hets, on a HOM_A1 background."""
    rng = np.random.default_rng(seed)
    out = rows.copy()
    sel = np.flatnonzero(rng.random(rows.shape[0]) < share)
    out[sel] = 0
    k = rng.integers(1, 6, len(sel))
    s = rng.integers(0, n, (len(sel), 5))
    for j in range(5):
        on = k > j
        np.bitwise_or.at(out, (sel[on], s[on, j] >> 2), (2 << (2 * (s[on, j] & 3))).astype(np.uint8))
    return out


def workload(rows, n, q, rate, mode):
    rng = np.random.default_rng(5)
    y, covar = (rng.random(n) < rate).astype(np.float64), rng.normal(size=(n, q - 1))
    with native.NativePca(n) as nat:
        nat.glmLogisticBegin(y, covar)
        nat.glmFirthBed(rows, mode=mode)                                                  # warm-up
        t0 = time.perf_counter()
        _, err, passes, firth = nat.glmFirthBed(rows, mode=mode)
        call = time.perf_counter() - t0
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            nat.glmFirthBed(rows, mode=mode)
        per = defaultdict(float)
        for ev in prof.events():
            if ev.device_type == torch.autograd.DeviceType.CUDA:
                per[kernel_of(ev.name)] += getattr(ev, "device_time_total", 0.0) / 1e3
    fp = passes[firth == 1].astype(np.int64)
    fmas = float(fp.sum()) * n * ((q + 1) * (q + 2) + 3 * (q + 1))
    floor_ms = 2.0 * fmas / (FP64_TFLOPS * 1e12) * 1e3
    return {"n_samples": n, "variants": rows.shape[0], "q": q, "case_rate": rate, "mode": mode, "call_s": round(call, 4),
            "kernel_ms": {key: round(v, 3) for key, v in sorted(per.items())},
            "firth_fits": int(fp.size),
            "firth_passes_mean": round(float(fp.mean()), 3) if fp.size else 0.0,
            "firth_passes_max": int(fp.max()) if fp.size else 0,
            "firth_fp64_floor_ms": round(floor_ms, 3),
            "floor_share_of_firth_kernel": round(floor_ms / per["glm_firth_kernel"], 3)
            if per["glm_firth_kernel"] else None,
            "errcodes": np.bincount(np.asarray(err), minlength=7).tolist()}


def main():
    import argparse
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--n", type=int, choices=(2504, 21845), help="run only the workloads of this many samples")
    args = ap.parse_args()
    name, power, clock = _card()
    out = {"card": name, "power_limit": power, "max_sm_clock": clock}

    def run(key, rows, n, q, rate):
        for mode in ("always", "fallback"):
            out[f"{key}_{mode}"] = workload(rows, n, q, rate, mode)
            print(json.dumps({f"{key}_{mode}": out[f"{key}_{mode}"]}), file=sys.stderr, flush=True)
    for n, nv in ((2504, 1 << 20), (21845, 1 << 16)):
        if args.n not in (None, n):
            continue
        rows = bn_rows(n, nv)
        for q in (11, 32):
            run(f"firth_{n}x{nv}_q{q}", rows, n, q, 0.3)
        run(f"firth_{n}x{nv}_q11_miss30", with_missing(rows, n, 0.3), n, 11, 0.3)
        rr = rare(rows, n)
        for q in (11, 32):
            run(f"firth_{n}x{nv}_q{q}_rare", rr, n, q, 0.1)
        del rows, rr
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
