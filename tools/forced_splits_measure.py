"""Training speed with a forced split plan against without, on one GPU.

The cfg2 shape of bench.py (10M x 256 dense f32 regression, 255 bins, 31 leaves).  Two boosters on the same dataset: plain, and one whose
every tree starts with a three-node plan (feature 0 at 0, then features 1 and 2 at 0 below it), written to a temporary file.  Both are
warmed up, then alternated over `--rounds` rounds of `--iters` timed iterations; each round reports iterations/s per arm.  The card's
name and power limit are read in the same run.  --extra adds parameters to both arms (e.g. extra_trees=true), --max-bin sets the
dataset's (above 255 every feature is a wide one, scanned by k_scan_wide).

    python tools/forced_splits_measure.py [--rows 10000000] [--features 256] [--iters 20] [--warmup 3] [--max-bin 255] [--extra ""]
                                          [--out FILE]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

DS_PARAMS = "max_bin=%d is_pre_partition=True bin_construct_sample_cnt=200000 num_threads=0"
PARAMS = ("metric= boost_from_average=true boosting_type=gbdt num_iterations=1000 learning_rate=0.1 num_leaves=31 max_bin=%d "
          "verbosity=-1 min_data_in_leaf=20 objective=regression num_threads=0 %s")
PLAN = {"feature": 0, "threshold": 0.0, "left": {"feature": 1, "threshold": 0.0}, "right": {"feature": 2, "threshold": 0.0}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=10_000_000)
    ap.add_argument("--features", type=int, default=256)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--max-bin", type=int, default=255)
    ap.add_argument("--extra", default="")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    from mmlspark_b200 import capi
    rng = np.random.default_rng(0)
    X = rng.standard_normal((args.rows, args.features), dtype=np.float32)
    y = (X[:, 0] * 2 + np.sin(3 * X[:, 1]) + X[:, 2] * X[:, 3] + 0.1 * rng.standard_normal(args.rows, dtype=np.float32)).astype(np.float32)
    with tempfile.TemporaryDirectory() as tmp:
        plan = os.path.join(tmp, "plan.json")
        with open(plan, "w") as f:
            json.dump(PLAN, f)
        params = PARAMS % (args.max_bin, args.extra)
        arms = {"plain": params, "forced_3": params + " forcedsplits_filename=" + plan}
        ds = capi.Dataset.from_mat(X, DS_PARAMS % args.max_bin).set_field("label", y)
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
    out = dict(card=card.splitlines()[0] if card else "unknown", rows=args.rows, features=args.features, max_bin=args.max_bin,
               extra=args.extra, iters_per_round=args.iters,
               its_per_s={k: [round(v, 3) for v in vs] for k, vs in res.items()},
               median_ratio_forced_to_plain=round(float(np.median(res["forced_3"]) / np.median(res["plain"])), 4))
    doc = json.dumps(out, indent=1)
    print(doc)
    if args.out:
        with open(args.out, "w") as f:
            f.write(doc + "\n")


if __name__ == "__main__":
    main()
