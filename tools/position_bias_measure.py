"""Time the ranking objectives' gradient pass and the position factors' update on one GPU: 10M documents in 100K queries of 100, 8
features, lambdarank (or --objective rank_xendcg), trained without a position field and with P distinct positions (P in 10, 1000,
100000; every query shows its documents at positions drawn from [0, P)).  Per iteration, torch.profiler's CUDA activity gives the device
time of the gradient kernel and of the update's kernels (k_absmax, k_set_scale, k_refit_leaf_sums, k_position_bias_update; the tree
learner runs one k_absmax per tree itself, so the cost of the feature is the difference of the two runs).  The wall time of an
iteration, ending in a device sync, is taken in a separate run without the profiler.  The card's name and power limit are read in the
same run.

    python tools/position_bias_measure.py [--docs 10000000] [--queries 100000] [--positions 10,1000,100000] [--iters 5] [--out FILE]
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

DS_PARAMS = "max_bin=255 bin_construct_sample_cnt=200000 num_threads=0"
KERNELS = ("k_grad_lambdarank", "k_grad_xendcg", "k_absmax", "k_set_scale", "k_refit_leaf_sums", "k_position_bias_update")


def _run(capi, ds, params, iters):
    import torch
    from torch.profiler import ProfilerActivity, profile
    b = capi.Booster(ds, params)
    try:
        for _ in range(2):      # warm-up: first launches, the column copy
            b.update_one_iter()
        b.get_scores()
        t0 = time.perf_counter()
        for _ in range(iters):
            b.update_one_iter()
        b.get_scores()      # ends in a stream sync
        wall = (time.perf_counter() - t0) / iters
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(iters):
                b.update_one_iter()
            b.get_scores()
            torch.cuda.synchronize()
        us = {k: 0.0 for k in KERNELS}
        for e in prof.events():
            for k in KERNELS:
                if k in e.name and e.device_type.name == "CUDA":
                    us[k] += e.device_time_total / iters
        _, f = b.position_bias()
        return dict(iteration_ms=wall * 1e3, kernel_us_per_iter=us, grad_and_update_us=sum(us.values()), factors=len(f),
                    factor_range=[float(f.min()), float(f.max())] if len(f) else None)
    finally:
        b.free()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--docs", type=int, default=10_000_000)
    ap.add_argument("--queries", type=int, default=100_000)
    ap.add_argument("--positions", default="10,1000,100000")
    ap.add_argument("--objective", default="lambdarank")
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch  # noqa: F401  (before the engine's library, which brings its own NCCL)
    from mmlspark_b200 import capi
    rng = np.random.default_rng(0)
    n, nq = args.docs, args.queries
    X = rng.standard_normal((n, 8), dtype=np.float32)
    y = np.clip(np.round(X[:, 0] + 0.5 * X[:, 1] + 1.5 + 0.5 * rng.standard_normal(n, dtype=np.float32)), 0, 4).astype(np.float32)
    sizes = np.full(nq, n // nq, np.int32)
    sizes[: n - int(sizes.sum())] += 1
    params = "objective=%s learning_rate=0.1 num_leaves=31 min_data_in_leaf=20 verbosity=-1 metric= %s" % (args.objective, DS_PARAMS)
    ds = capi.Dataset.from_mat(X, DS_PARAMS).set_field("label", y).set_field("group", sizes)
    del X
    runs = [dict(positions=0, **_run(capi, ds, params, args.iters))]
    for P in (int(p) for p in args.positions.split(",")):
        ds.set_field("position", rng.integers(0, P, n).astype(np.int32))
        runs.append(dict(positions=P, **_run(capi, ds, params, args.iters)))
    ds.set_field("position", np.zeros(0, np.int32))
    ds.free()
    try:
        gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                             check=True).stdout.strip().splitlines()[0]
    except Exception as e:      # noqa
        gpu = "unknown (%s)" % e
    base = runs[0]["grad_and_update_us"]
    for r in runs[1:]:
        r["added_us"] = r["grad_and_update_us"] - base
    line = json.dumps(dict(gpu=gpu, objective=args.objective, docs=n, queries=nq, iters=args.iters, runs=runs))
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
