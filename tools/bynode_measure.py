"""Training speed with per-node feature sampling (feature_fraction_bynode) against without, on one GPU.

Dense f32 regression, 255 bins, 31 leaves: the cfg2 shape of bench.py (10M x 256) by default, or another --rows x --features.  Arms:
the key absent, feature_fraction_bynode=1.0 (which must train the model of the absent key; checked at the end), 0.5 and 0.1 (at 256
features the selection and Floyd's branch of the sampler).  All are warmed up, then alternated over --rounds rounds of --iters timed
iterations; each round reports iterations/s per arm.  The arms grow different trees, so iterations/s alone does not compare the
sampler's cost: each arm also runs once more in a child process with B200GBM_SPLIT_TIMING=1 on --timing-rows rows, and the tool reports
the per-split "scan+pick" time (the scan kernels, the sampler blocks among them, and the pick).  The card's name and power limit are
read in the same run.

    python tools/bynode_measure.py [--rows 10000000] [--features 256] [--iters 20] [--warmup 3] [--rounds 3] [--timing-rows 1000000]
                                   [--out FILE]
"""
import argparse
import json
import os
import re
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

DS_PARAMS = "max_bin=255 is_pre_partition=True bin_construct_sample_cnt=200000 num_threads=0"
PARAMS = ("metric= boost_from_average=true boosting_type=gbdt num_iterations=1000 learning_rate=0.1 num_leaves=31 max_bin=255 "
          "verbosity=-1 min_data_in_leaf=20 objective=regression num_threads=0")
ARMS = {"absent": "", "bynode_1.0": " feature_fraction_bynode=1.0", "bynode_0.5": " feature_fraction_bynode=0.5",
        "bynode_0.1": " feature_fraction_bynode=0.1"}


def _data(rows, features):
    rng = np.random.default_rng(0)
    X = rng.standard_normal((rows, features), dtype=np.float32)
    y = (X[:, 0] * 2 + np.sin(3 * X[:, 1]) + X[:, 2] * X[:, 3] + 0.1 * rng.standard_normal(rows, dtype=np.float32)).astype(np.float32)
    return X, y


def _split_timing(arm, rows, features, iters):
    """one child process: train `iters` iterations with B200GBM_SPLIT_TIMING=1 and return the per-split scan+pick time (us)"""
    env = dict(os.environ, B200GBM_SPLIT_TIMING="1")
    r = subprocess.run([sys.executable, os.path.abspath(__file__), "--child", arm, "--rows", str(rows), "--features", str(features),
                        "--iters", str(iters)], env=env, capture_output=True, text=True, check=True)
    m = re.search(r"scan\+pick=([0-9.]+)us", r.stderr)
    if not m:
        raise RuntimeError("no split timing in the child's output:\n" + r.stderr[-2000:])
    return float(m.group(1))


def _child(arm, rows, features, iters):
    from mmlspark_b200 import capi
    X, y = _data(rows, features)
    ds = capi.Dataset.from_mat(X, DS_PARAMS).set_field("label", y)
    b = capi.Booster(ds, PARAMS + ARMS[arm])
    try:
        for _ in range(iters):
            b.update_one_iter()
    finally:
        b.free()      # the learner prints the split timing when it is freed
        ds.free()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=10_000_000)
    ap.add_argument("--features", type=int, default=256)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--timing-rows", type=int, default=1_000_000)
    ap.add_argument("--child", default=None, help=argparse.SUPPRESS)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if args.child:
        _child(args.child, args.rows, args.features, args.iters)
        return
    from mmlspark_b200 import capi
    X, y = _data(args.rows, args.features)
    ds = capi.Dataset.from_mat(X, DS_PARAMS).set_field("label", y)
    del X
    boosters = {k: capi.Booster(ds, PARAMS + p) for k, p in ARMS.items()}
    res = {k: [] for k in ARMS}
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
        trees = {k: b.save_model_to_string().split("\nparameters:")[0] for k, b in boosters.items()}
        assert trees["bynode_1.0"] == trees["absent"], "feature_fraction_bynode=1.0 must train the model of the absent key"
        assert trees["bynode_0.5"] != trees["absent"]
    finally:
        for b in boosters.values():
            b.free()
        ds.free()
    split_us = {k: _split_timing(k, args.timing_rows, args.features, args.iters) for k in ARMS}
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    out = dict(card=card.splitlines()[0] if card else "unknown", rows=args.rows, features=args.features, iters_per_round=args.iters,
               its_per_s={k: [round(v, 3) for v in vs] for k, vs in res.items()},
               median_ratio={k: round(float(np.median(res[k]) / np.median(res["absent"])), 4) for k in ARMS if k != "absent"},
               timing_rows=args.timing_rows, scan_pick_us_per_split={k: round(v, 2) for k, v in split_us.items()})
    doc = json.dumps(out, indent=1)
    print(doc)
    if args.out:
        with open(args.out, "w") as f:
            f.write(doc + "\n")


if __name__ == "__main__":
    main()
