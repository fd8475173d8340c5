"""Time LGBM_BoosterRefit on one GPU: a 10M x 64 regression model of 100 trees (255 leaves) is trained, the leaf indices of the training
rows are predicted on the device, and a booster with the model merged into it refits all 100 trees on the same rows.  The refit ends in a
device sync; its time is split into the staging of the 10M x 100 leaf-index matrix (host to device through the pinned row blocks,
transposed and range-checked on the device) and the per-tree work (gradients, per-leaf sums, leaf rule, score update), as the engine reports
them (B200GBM_BoosterGetRefitTiming).  Training the same 100 trees is timed beside it.  The card's name and power limit are read in the
same run.

    python tools/refit_measure.py [--rows 10000000] [--features 64] [--trees 100] [--leaves 255] [--repeats 3] [--out FILE]
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=10_000_000)
    ap.add_argument("--features", type=int, default=64)
    ap.add_argument("--trees", type=int, default=100)
    ap.add_argument("--leaves", type=int, default=255)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    from mmlspark_b200 import capi
    rng = np.random.default_rng(0)
    X = rng.standard_normal((args.rows, args.features), dtype=np.float32)
    y = (X[:, 0] * 2 + np.sin(3 * X[:, 1]) + X[:, 2] * X[:, 3] + 0.1 * rng.standard_normal(args.rows, dtype=np.float32)).astype(np.float32)
    params = "objective=regression learning_rate=0.1 num_leaves=%d min_data_in_leaf=20 verbosity=-1 %s" % (args.leaves, DS_PARAMS)
    ds = capi.Dataset.from_mat(X, DS_PARAMS).set_field("label", y)
    b = capi.Booster(ds, params)
    b.update_one_iter()      # warm-up: first launches, the column copy
    t0 = time.perf_counter()
    for _ in range(args.trees - 1):
        b.update_one_iter()
    b.get_scores()      # ends in a stream sync
    train_s = (time.perf_counter() - t0) * args.trees / (args.trees - 1)
    model = b.save_model_to_string()
    b.free()
    old = capi.Booster(model_str=model)
    leaf = old.predict_device(X, capi.PREDICT_LEAF_INDEX).astype(np.int32)
    old.free()
    del X
    runs = []
    for r in range(args.repeats + 1):      # the first refit is a warm-up
        m = capi.Booster(ds, params + " refit_decay_rate=0.9")
        old = capi.Booster(model_str=model)
        m.merge(old)
        old.free()
        t0 = time.perf_counter()
        m.refit(leaf)
        wall = time.perf_counter() - t0
        t = m.refit_timing()
        m.free()
        if r > 0:
            runs.append(dict(wall_s=wall, stage_s=t["stage_ms"] / 1e3, tree_s=t["tree_ms"] / 1e3, batches=t["batches"], row_blocks=t["blocks"]))
    ds.free()
    try:
        gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                             check=True).stdout.strip().splitlines()[0]
    except Exception as e:      # noqa
        gpu = "unknown (%s)" % e
    res = dict(gpu=gpu, rows=args.rows, features=args.features, trees=args.trees, leaves=args.leaves,
               leaf_matrix_bytes=args.rows * args.trees * 4, train_100_trees_s=train_s, refit=runs)
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
