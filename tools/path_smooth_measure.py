"""Training speed with path smoothing against without, on one GPU.

The cfg2 shape of bench.py (10M x 256 dense f32 regression, 255 bins, 31 leaves).  Three boosters on the same dataset: plain,
path_smooth=10 (the scans' output-based kMono instantiations with smoothing), and, for the cost of smoothing on top of constraints,
monotone constraints on 16 features (+1 on features 0-7, -1 on 8-15) with and without path_smooth=10.  All are warmed up, then alternated
over `--rounds` rounds of `--iters` timed iterations; each round reports iterations/s per arm.  The card's name and power limit are read
in the same run.

    python tools/path_smooth_measure.py [--rows 10000000] [--features 256] [--iters 20] [--warmup 3] [--out FILE]
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

DS_PARAMS = "max_bin=255 is_pre_partition=True bin_construct_sample_cnt=200000 num_threads=0"
PARAMS = ("metric= boost_from_average=true boosting_type=gbdt num_iterations=1000 learning_rate=0.1 num_leaves=31 max_bin=255 "
          "verbosity=-1 min_data_in_leaf=20 objective=regression num_threads=0")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=10_000_000)
    ap.add_argument("--features", type=int, default=256)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    from mmlspark_b200 import capi
    rng = np.random.default_rng(0)
    X = rng.standard_normal((args.rows, args.features), dtype=np.float32)
    y = (X[:, 0] * 2 + np.sin(3 * X[:, 1]) + X[:, 2] * X[:, 3] + 0.1 * rng.standard_normal(args.rows, dtype=np.float32)).astype(np.float32)
    mono = [1] * 8 + [-1] * 8 + [0] * (args.features - 16)
    mc = " monotone_constraints=" + ",".join(str(m) for m in mono)
    arms = {"plain": PARAMS, "path_smooth_10": PARAMS + " path_smooth=10", "monotone_16": PARAMS + mc,
            "monotone_16_path_smooth_10": PARAMS + mc + " path_smooth=10"}
    ds = capi.Dataset.from_mat(X, DS_PARAMS).set_field("label", y)
    boosters = {k: capi.Booster(ds, p) for k, p in arms.items()}
    res = {k: [] for k in arms}
    try:
        for b in boosters.values():
            for _ in range(args.warmup):
                b.update_one_iter()
        for _ in range(args.rounds):
            for k, b in boosters.items():
                t0 = time.perf_counter()
                for _ in range(args.iters):
                    b.update_one_iter()      # each iteration reads its tree back (a stream sync)
                res[k].append(args.iters / (time.perf_counter() - t0))
    finally:
        for b in boosters.values():
            b.free()
        ds.free()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    out = dict(card=card.splitlines()[0] if card else "unknown", rows=args.rows, features=args.features, iters_per_round=args.iters,
               its_per_s={k: [round(v, 3) for v in vs] for k, vs in res.items()},
               median_ratio_smooth_to_plain=round(float(np.median(res["path_smooth_10"]) / np.median(res["plain"])), 4),
               median_ratio_monotone_smooth_to_monotone=round(float(np.median(res["monotone_16_path_smooth_10"]) / np.median(res["monotone_16"])), 4))
    doc = json.dumps(out, indent=1)
    print(doc)
    if args.out:
        with open(args.out, "w") as f:
            f.write(doc + "\n")


if __name__ == "__main__":
    main()
