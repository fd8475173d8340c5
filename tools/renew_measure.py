"""Device time of the leaf renewal pass (renew_kernel.cuh) for weighted regression_l1 at 10M rows, on one GPU.

A 10M x 16 dense f32 regression_l1 dataset with row weights, 31 leaves.  Two weight sets: float32 weights in [0.5, 2] on a 1/64 grid,
where every add of the cdf scan is exact, and log-uniform weights spanning 1..1e7, where the scan's adds round and each leaf's cdf is
summed in row order.  After `--warmup` iterations, `--iters` iterations run under torch.profiler; the pass is the sum of the device
times of the kernels Renew launches (k_renew_*, and cub's radix sort kernels, which only the renewal uses), per tree.  `--lib` loads
another build of libb200gbm.so, to compare two builds in one run.  The card's name and power limit are read in the same run.

    python tools/renew_measure.py [--rows 10000000] [--iters 5] [--warmup 2] [--lib PATH] [--out FILE]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

DS_PARAMS = "max_bin=255 is_pre_partition=True bin_construct_sample_cnt=200000 num_threads=0"
PARAMS = "objective=regression_l1 metric= learning_rate=0.1 num_leaves=31 min_data_in_leaf=20 verbosity=-1 num_threads=0"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=10_000_000)
    ap.add_argument("--features", type=int, default=16)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--lib", default=None)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile
    from mmlspark_b200 import capi
    if args.lib:
        capi.LIB_PATH = os.path.abspath(args.lib)
    rng = np.random.default_rng(0)
    n = args.rows
    X = rng.standard_normal((n, args.features), dtype=np.float32)
    y = (X[:, 0] * 2 + np.sin(3 * X[:, 1]) + X[:, 2] * X[:, 3] + rng.standard_normal(n, dtype=np.float32)).astype(np.float32)
    weights = {"narrow [0.5, 2]": (0.5 + np.round(rng.uniform(0, 1.5, n) * 64) / 64).astype(np.float32),
               "wide 1..1e7": (10.0 ** rng.uniform(0, 7, n)).astype(np.float32)}
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    res = dict(gpu=gpu, lib=capi.LIB_PATH, rows=n, iters=args.iters, arms={})
    ds = capi.Dataset.from_mat(X, DS_PARAMS).set_field("label", y)
    try:
        for name, w in weights.items():
            ds.set_field("weight", w)
            b = capi.Booster(ds, PARAMS)
            try:
                for _ in range(args.warmup):
                    b.update_one_iter()
                torch.cuda.synchronize()
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    for _ in range(args.iters):
                        b.update_one_iter()
                    torch.cuda.synchronize()
            finally:
                b.free()
            times = {}
            for e in prof.key_averages():
                if "k_renew" in e.key or "RadixSort" in e.key:
                    times[e.key.split("(")[0][:60]] = e.device_time_total / 1e3 / args.iters
            res["arms"][name] = dict(renew_ms_per_tree=sum(times.values()), kernels_ms_per_tree=times)
            print(name, json.dumps(res["arms"][name]), flush=True)
    finally:
        ds.free()
    print(json.dumps(res))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
