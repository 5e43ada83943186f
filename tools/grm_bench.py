#!/usr/bin/env python
"""Time the variance-standardized relationship matrix (vpca_grm_bed + vpca_grm_finalize, vpca_compute_pca_grm) on seeded
Balding-Nichols .bed rows: three populations (shares 1 : 1.12 : 1.25, F_ST 0.20 / 0.12 / 0.04), ancestral allele
frequency 0.05 + 0.45 u, 1 % of the calls missing.  Workloads: 2504 x 262 144 and 21 845 x 65 536 rows.  Per workload:
one warm-up pass, then the host clock around grmBed + grmFinalize (both synchronise before they return), repeated; a
separate torch.profiler run of the same pass for the per-kernel times; the achieved FP64 rate N (N + 1) / 2 * M * 2 flops
over the SYRK kernel time against the 67 TFLOP/s FP64-tensor figure of the H100 SXM data sheet; the host clock around
computePcaGrm(2) (the two axes of the three populations); and, as a yardstick, torch.matmul in float64 (cuBLAS, the whole N x N product: twice the multiply
work) of the same expanded Z, timed with CUDA events.  Prints one JSON line with the card and its power limit, read in
the same run."""
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

FP64_TENSOR_TFLOPS = 67.0   # H100 SXM data sheet, dense FP64 tensor core


def _card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = [x.strip() for x in q.split(",")]
        return name, power, clock
    except Exception:
        return torch.cuda.get_device_name(0), "unknown", "unknown"


def bn_rows(n, nv, seed=20261018, block=8192):
    """(nv, ceil(n / 4)) .bed rows of the cohort described above, drawn on the GPU in blocks of variants."""
    rng = np.random.default_rng(seed)
    gen = torch.Generator(device="cuda").manual_seed(seed)
    share = 1.12 ** np.arange(3)
    pop = np.minimum(np.searchsorted(np.cumsum(share / share.sum()) * n, np.arange(n), side="right"), 2)
    pop_d = torch.from_numpy(pop).cuda()
    out = np.empty((nv, (n + 3) // 4), np.uint8)
    for v0 in range(0, nv, block):
        b = min(block, nv - v0)
        anc = 0.05 + 0.45 * rng.random(b)
        P = np.stack([rng.beta(anc * (1 - f) / f, (1 - anc) * (1 - f) / f) for f in (0.20, 0.12, 0.04)], axis=1)
        p = torch.from_numpy(P).cuda()[:, pop_d]                                        # (b, n)
        d = (torch.rand((b, n), generator=gen, device="cuda", dtype=torch.float64) < p).to(torch.uint8) + \
            (torch.rand((b, n), generator=gen, device="cuda", dtype=torch.float64) < p).to(torch.uint8)
        code = torch.where(d == 2, 0, torch.where(d == 1, 2, 3)).to(torch.uint8)
        code[torch.rand((b, n), generator=gen, device="cuda") < 0.01] = 1
        code = torch.nn.functional.pad(code, (0, (-n) % 4)).view(b, -1, 4)
        packed = code[:, :, 0] | (code[:, :, 1] << 2) | (code[:, :, 2] << 4) | (code[:, :, 3] << 6)
        out[v0:v0 + b] = packed.cpu().numpy()
    return out


def expanded_z(rows, n):
    """The used variants' z columns on the device, (n, M) float64, from the same counts and table operations."""
    r = torch.from_numpy(rows).cuda()
    code = torch.stack([(r >> s) & 3 for s in (0, 2, 4, 6)], dim=-1).reshape(r.shape[0], -1)[:, :n].long()   # (V, n)
    cnt = torch.stack([(code == c).sum(1) for c in (0, 2, 3)], dim=1).double()
    nn, a = cnt.sum(1), 2 * cnt[:, 0] + cnt[:, 1]
    used = (a > 0) & (a < 2 * nn)
    a1 = a <= 2 * nn - a
    rr = torch.where(a1, a, 2 * nn - a)
    nn1 = torch.where(used, nn, torch.ones_like(nn))
    mu = rr / nn1
    s = 1.0 / torch.sqrt(mu * (1.0 - rr / (2.0 * nn1)))
    tab = torch.stack([(torch.where(a1, 2.0, 0.0) - mu) * s, torch.zeros_like(mu), (1.0 - mu) * s,
                       (torch.where(a1, 0.0, 2.0) - mu) * s], dim=1)
    Zt = torch.gather(tab[used], 1, code[used])
    return Zt.T.contiguous()


def kernel_of(name):
    for key in ("grm_syrk", "grm_expand", "grm_table", "grm_compact", "grm_finish", "qc_count", "Memcpy HtoD"):
        if key in name:
            return key.replace("Memcpy ", "memcpy_").lower()
    return "other"


def workload(n, nv, k=2, repeats=3):
    rows = bn_rows(n, nv)
    with native.NativePca(n, num_pc=k) as nat:
        def grm_pass():
            nat.reset()
            nat.grmBed(rows)
            return nat.grmFinalize()
        M = grm_pass()                                                                  # warm-up
        times = []
        for _ in range(repeats):
            t0 = time.perf_counter()
            grm_pass()
            times.append(time.perf_counter() - t0)
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            grm_pass()
        per = defaultdict(float)
        for ev in prof.events():
            if ev.device_type == torch.autograd.DeviceType.CUDA:
                per[kernel_of(ev.name)] += getattr(ev, "device_time_total", 0.0) / 1e3
        grm_pass()
        t0 = time.perf_counter()
        nat.computePcaGrm(k)
        solve_s = time.perf_counter() - t0
        method = nat.stats()["eig_method"]
    flops = n * (n + 1) / 2 * M * 2
    syrk_ms = per["grm_syrk"]
    Z = expanded_z(rows, n)
    assert Z.shape[1] == M
    torch.matmul(Z, Z.T)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(repeats):
        torch.matmul(Z, Z.T)
    e1.record()
    torch.cuda.synchronize()
    mm_ms = e0.elapsed_time(e1) / repeats
    del Z
    torch.cuda.empty_cache()
    return {"n_samples": n, "variants": nv, "used": M, "grm_pass_s": [round(t, 4) for t in times],
            "kernel_ms": {key: round(v, 3) for key, v in sorted(per.items())},
            "syrk_tflops": round(flops / (syrk_ms * 1e-3) / 1e12, 2),
            "syrk_share_of_67tflops": round(flops / (syrk_ms * 1e-3) / 1e12 / FP64_TENSOR_TFLOPS, 3),
            "datasheet_floor_ms": round(flops / (FP64_TENSOR_TFLOPS * 1e12) * 1e3, 2),
            "solve_k2_s": round(solve_s, 4), "eig_method": method,
            "torch_matmul_f64_ms": round(mm_ms, 2)}


def main():
    name, power, clock = _card()
    out = {"card": name, "power_limit": power, "max_sm_clock": clock,
           "grm_2504x262144": workload(2504, 1 << 18),
           "grm_21845x65536": workload(21845, 1 << 16)}
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
