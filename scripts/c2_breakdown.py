#!/usr/bin/env python
"""Where the time of one C2 step goes: per-kernel table and scoring counters.

    python scripts/c2_breakdown.py --out DIR [--warmup 3]

Builds the C2 inputs exactly as bench.py does (same seed, sizes and build()), runs warm-up steps, then ONE step under
torch.profiler with CUDA activities.  Writes to DIR:
  kernels.csv     kernel name, launches, total device ms (sorted by time)
  summary.json    the table plus the counters of that step: tile products executed / full (stats [5], [6]), exact
                  rescorings per user (stats [1]), the fused kernel's own time (CUDA events inside the library), the GPU
                  name and its power limit
and prints both as markdown.  Needs a GPU; bench.py stays the timing reference (the profiler slows the host).
"""
from __future__ import annotations

import argparse
import csv
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def gpu_info(index=0):
    q = "name,power.limit,clocks.max.sm"
    try:
        txt = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader", "-i", str(index)],
                             capture_output=True, text=True, timeout=10).stdout.strip()
        name, power, clk = [x.strip() for x in txt.split("\n")[0].split(",")]
        return {"name": name, "power_limit": power, "sm_max_clock": clk}
    except Exception as exc:                                       # noqa: BLE001
        import torch
        return {"name": torch.cuda.get_device_name(index), "power_limit": "unknown (%s)" % exc, "sm_max_clock": None}


def kernel_table(prof):
    from torch.autograd import DeviceType
    rows = []
    for evt in prof.key_averages():
        if getattr(evt, "device_type", None) != DeviceType.CUDA:
            continue
        us = getattr(evt, "self_device_time_total", None)
        if us is None:
            us = getattr(evt, "self_cuda_time_total", 0.0)
        rows.append({"kernel": evt.key, "launches": int(evt.count), "total_ms": float(us) / 1e3})
    rows.sort(key=lambda r: -r["total_ms"])
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--users", type=int, default=1_000_000)
    ap.add_argument("--items", type=int, default=100_000)
    ap.add_argument("--nnz", type=int, default=100_000_000)
    ap.add_argument("--rank", type=int, default=50)
    ap.add_argument("--topk", type=int, default=10)
    args = ap.parse_args()

    import numpy as np
    import torch
    from torch.profiler import ProfilerActivity, profile
    import bench
    from polara_b200 import _build
    from polara_b200 import dist as pdist
    from polara_b200.engine import DeviceCSR, get_engine
    from polara_b200.host import ArrayData
    from polara_b200.models import B200SVDModel

    if not torch.cuda.is_available():
        raise SystemExit("c2_breakdown needs a GPU")
    torch.cuda.set_device(0)
    dev = torch.device("cuda", 0)
    _build.build()
    eng = get_engine(0)

    # the inputs of bench.py's C2 step (one GPU): same generator, seed and nnz correction, build() from the device CSR
    indptr_d, indices_d, values_d = bench.synth_csr_torch(args.users, args.items, args.nnz, 20260924, dev)
    nnz = int(indices_d.shape[0])
    if nnz < 0.97 * args.nnz:
        del indptr_d, indices_d, values_d
        indptr_d, indices_d, values_d = bench.synth_csr_torch(args.users, args.items,
                                                              int(args.nnz * (args.nnz / nnz) ** 1.15), 20260924, dev)
    shape = (args.users, args.items)
    data = ArrayData(np.zeros((1, 2), dtype=np.int64), np.ones(1), shape)
    data.train_csr = (indptr_d, indices_d, values_d, shape)
    model = B200SVDModel(data)
    model.verbose = False
    model.rank = args.rank
    model.topk = args.topk
    model.build()
    p_dev = DeviceCSR(indptr_d, indices_d, values_d, shape)
    v_dev = model._device_factor("itemid")
    step = pdist.make_step(eng, p_dev, v_dev, args.rank, args.topk, None)
    for _ in range(args.warmup):
        step()
    torch.cuda.synchronize()

    s0 = eng.stats()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        step()
        torch.cuda.synchronize()
    s1 = eng.stats()
    fused_ms = eng.last_score_kernel_ms()
    rows = kernel_table(prof)

    executed, full = s1[5] - s0[5], s1[6] - s0[6]
    summary = {
        "gpu": gpu_info(0),
        "config": {"users": args.users, "items": args.items, "nnz": int(indices_d.shape[0]), "rank": args.rank,
                   "topk": args.topk, "warmup": args.warmup},
        "tile_products_executed": int(executed), "tile_products_full": int(full),
        "executed_share": executed / max(full, 1),
        "rescored_per_user": (s1[1] - s0[1]) / args.users,
        "fused_kernel_ms": fused_ms,
        "kernels_total_ms": sum(r["total_ms"] for r in rows),
        "kernels": rows,
    }
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "kernels.csv"), "w", newline="") as f:
        w = csv.DictWriter(f, fieldnames=["kernel", "launches", "total_ms"])
        w.writeheader()
        w.writerows(rows)
    with open(os.path.join(args.out, "summary.json"), "w") as f:
        json.dump(summary, f, indent=1)

    g = summary["gpu"]
    print("%s, power limit %s" % (g["name"], g["power_limit"]))
    print("| kernel | launches | total ms |\n|---|---|---|")
    for r in rows:
        print("| %s | %d | %.3f |" % (r["kernel"][:90], r["launches"], r["total_ms"]))
    print("| all kernels | %d | %.3f |" % (sum(r["launches"] for r in rows), summary["kernels_total_ms"]))
    print("tile products executed %d of %d (%.2f %%), exact rescorings per user %.1f, fused kernel %.3f ms" % (
        executed, full, 100.0 * summary["executed_share"], summary["rescored_per_user"], fused_ms))


if __name__ == "__main__":
    main()
