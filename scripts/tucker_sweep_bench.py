"""Timing of the Tucker-rank search of a CoFFee model: one tucker_rank_sweep against the reference-style loop it replaces.

    python scripts/tucker_sweep_bench.py [--scale 1.0] [--test-users 100000] [--num-iters 4] [--loop all|corners]

Workload: the C4 shape of ``bench.py --config c4`` (1 M users x 50 K items x 5 feedback levels, nnz 5e7, the same
synthetic tensor), built once at mlrank (60, 60, 4); test data: ``--test-users`` further users of the same generator
(about 50 rated items each) with one holdout item per user, top-10.  The grid is r1, r2 in {20, 40, 60} x r3 in
{2, 3, 4}: 25 triples, the skip rule drops (20, 60, 2) and (60, 20, 2).  One JSON line with:
  * build_s: the HOOI build (``--num-iters`` iterations, growth_tol 0);
  * sweep_ms: one tucker_rank_sweep over the grid (host clock around work that ends in a copy to the host), and the
    per-triple phases of a second, profiled sweep (``profile_phases``): host rounding (host clock), item rotation,
    value rewrite, SpMM and scoring (CUDA events), as the median over the triples and the sum;
  * search_s: find_optimal_tucker_ranks with the default evaluator (hit rate: one holdout item per user) against the reference-style loop on the
    same model and the ``--loop`` triples (``model.mlrank = t``; ``get_recommendations()``; evaluate; factors restored),
    scaled to the grid when the loop runs a subset;
  * lists_equal: of the looped triples, how many have lists equal to the sweep's (all at r2 = 60 by construction;
    below it the rotations differ in the last bit, DESIGN.md section 4).
The device name and its power limit are read in the same run.  Writes nothing but stdout, and progress to stderr.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

GRID = ([20, 40, 60], [20, 40, 60], [2, 3, 4])


def _progress(msg):
    print("tucker_sweep_bench: " + msg, file=sys.stderr, flush=True)


def _device_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = [x.strip() for x in out.split(",")]
        return {"name": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as exc:                       # the torch name still identifies the card
        import torch
        return {"name": torch.cuda.get_device_name(0), "power_limit": "not read (%s)" % exc}


def _data(scale, n_test, dev):
    import pandas as pd
    import torch
    from bench import synth_csr_torch
    from polara_b200.host import ArrayData
    n_users, n_items, nnz_t = int(1_000_000 * scale), int(50_000 * scale), int(50_000_000 * scale)
    indptr, indices, values = synth_csr_torch(n_users + n_test, n_items, int((nnz_t * 1.15) * (1 + n_test / n_users)),
                                              20260924, dev)
    user = torch.repeat_interleave(torch.arange(n_users + n_test, device=dev), torch.diff(indptr))
    idx = torch.stack([user, indices.to(torch.int64), (values - 1).to(torch.int64)], dim=1).cpu().numpy()
    train = idx[idx[:, 0] < n_users]
    test = idx[idx[:, 0] >= n_users]
    test[:, 0] -= n_users
    counts = np.bincount(test[:, 0], minlength=n_test)
    test = test[counts[test[:, 0]] >= 2]                  # every test user keeps a profile beside its holdout item
    test[:, 0] = np.cumsum(counts >= 2)[test[:, 0]] - 1
    rng = np.random.default_rng(1)
    starts = np.r_[0, np.flatnonzero(np.diff(test[:, 0])) + 1]
    pick = starts + (rng.random(len(starts)) * np.diff(np.r_[starts, len(test)])).astype(np.int64)
    hold = np.zeros(len(test), bool)
    hold[pick] = True
    holdout = pd.DataFrame({"userid": test[hold, 0], "itemid": test[hold, 1], "rating": test[hold, 2] + 1.0})
    rest = test[~hold]
    m = int(test[:, 0].max()) + 1
    data = ArrayData(train, np.ones(len(train)), (n_users, n_items, 5), rest[:, 0], rest[:, 1], rest[:, 2],
                     (m, n_items, 5), holdout=holdout, n_feedback=5, holdout_size=1)
    return data, (n_users, n_items, m), len(train), len(rest)


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--scale", type=float, default=1.0)
    ap.add_argument("--test-users", type=int, default=100_000)
    ap.add_argument("--num-iters", type=int, default=4)
    ap.add_argument("--loop", choices=["all", "corners"], default="all",
                    help="triples of the reference-style loop: the whole grid, or r1, r2 in {20, 60} x r3 in {2, 4}")
    args = ap.parse_args()
    import torch
    from polara_b200 import _build
    _build.build()
    from polara_b200 import pipelines
    from polara_b200.models import B200CoffeeModel
    torch.cuda.set_device(0)
    dev = torch.device("cuda", 0)
    info = _device_info()
    _progress("data")
    data, shape, nnz_train, nnz_test = _data(args.scale, int(args.test_users * args.scale), dev)
    model = B200CoffeeModel(data)
    model.verbose = False
    model.mlrank = (60, 60, 4)
    model.seed = 0
    model.growth_tol = 0.0
    model.num_iters = args.num_iters
    model.topk = 10
    _progress("build")
    t0 = time.perf_counter()
    model.build()
    torch.cuda.synchronize()
    build_s = time.perf_counter() - t0
    model._is_ready = True
    grid = pipelines._tucker_grid(GRID)
    _progress("sweep (%d triples)" % len(grid))
    model.tucker_rank_sweep(grid[:2])                     # warm-up: modules, allocator
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    lists = model.tucker_rank_sweep(grid)
    sweep_ms = (time.perf_counter() - t0) * 1e3
    model.profile_phases = True
    model.tucker_rank_sweep(grid)
    model.profile_phases = False
    phases = {k: [t[k] for t in model.last_sweep_timings] for k in
              ("round_ms", "rotate_ms", "rewrite_ms", "spmm_ms", "score_ms")}
    phase_stats = {k: {"median": float(np.median(v)), "sum": float(np.sum(v))} for k, v in phases.items()}
    _progress("search")
    t0 = time.perf_counter()
    best = pipelines.find_optimal_tucker_ranks(model, GRID, "hr", metric_type="relevance")
    search_s = time.perf_counter() - t0
    loop = grid if args.loop == "all" else [t for t in grid if t[0] in (20, 60) and t[1] in (20, 60) and t[2] in (2, 4)]
    _progress("reference-style loop (%d triples)" % len(loop))
    full, full_rank = dict(model.factors), model._mlrank
    equal, equal_full, res = 0, 0, {}
    t0 = time.perf_counter()
    for t in loop:
        model.mlrank = t
        recs = model.get_recommendations()
        model._recommendations = recs
        res[t] = pipelines.evaluate_models(model, "hr", metric_type="relevance")[model.method]
        model._recommendations = None
        model._mlrank, model.factors = full_rank, dict(full)
        same = int(np.array_equal(recs, lists[t]))
        equal += same
        equal_full += same if t[1] == 60 else 0
    loop_s = time.perf_counter() - t0
    loop_best = max(res, key=res.get)
    out = {"workload": "C4 CoFFee Tucker-rank search: %d x %d x 5 tensor, train nnz %d, build mlrank (60, 60, 4), "
                       "%d test users (test nnz %d), top-10, grid %s"
                       % (shape[0], shape[1], nnz_train, shape[2], nnz_test, GRID),
           "device": info, "build_s": build_s, "num_iters": args.num_iters, "triples": len(grid),
           "sweep_ms": sweep_ms, "sweep_ms_per_triple": sweep_ms / len(grid), "phases_ms_per_triple": phase_stats,
           "search_s": search_s, "best": [int(x) for x in best],
           "loop": {"triples": len(loop), "s": loop_s, "s_scaled_to_grid": loop_s * len(grid) / len(loop),
                    "best_of_looped": [int(x) for x in loop_best]},
           "search_speedup_vs_loop": loop_s * len(grid) / len(loop) / search_s,
           "lists_equal": {"equal": equal, "of": len(loop), "equal_at_r2_60": equal_full,
                           "of_at_r2_60": sum(1 for t in loop if t[1] == 60)}}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
