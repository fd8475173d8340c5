"""Training speed and accuracy of quantised training (use_quantized_grad) against full precision, on one GPU.

Shapes: cfg2 of bench.py (10M x 256 dense f32 regression, 255 bins, 31 leaves), or cfg3's kind (binary, is_unbalance=false).  The
matrix is built in host memory, so cfg3 at its full shape (100M x 512, with the validation rows about 215 GB of float32) runs only on a
host with that much free memory: elsewhere the tool stops before allocating and asks for --rows / --features to scale it down.
Three boosters on the same dataset: full precision, and quantised at B = 4 and B = 16 (num_grad_quant_bins, stochastic rounding).  All are warmed up, then alternated over `--rounds` rounds of `--iters` timed
iterations; each round reports iterations/s per arm and, from a second pass with the histogram events on (B200GBM_BoosterGetTiming), K4
ms per iteration.  Each arm's metric on a held-out validation set (l2 or binary_logloss) after all its iterations is reported beside.
The card's name and power limit are read in the same run.

    python tools/quant_measure.py [--shape cfg2|cfg3] [--rows N] [--features F] [--iters 20] [--warmup 3] [--rounds 3] [--out FILE]
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
BASE = ("boost_from_average=true boosting_type=gbdt num_iterations=1000 learning_rate=0.1 num_leaves=31 max_bin=255 verbosity=-1 "
        "min_data_in_leaf=20 num_threads=0")
SHAPES = {"cfg2": dict(rows=10_000_000, features=256, objective="objective=regression metric=l2"),
          "cfg3": dict(rows=100_000_000, features=512, objective="objective=binary is_unbalance=false metric=binary_logloss")}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shape", default="cfg2", choices=sorted(SHAPES))
    ap.add_argument("--rows", type=int, default=None)
    ap.add_argument("--features", type=int, default=None)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    shape = SHAPES[args.shape]
    rows, features = args.rows or shape["rows"], args.features or shape["features"]
    nvalid = max(rows // 20, 1000)
    need = (rows + nvalid) * features * 4 * 2          # the matrix, and the labels' and datasets' transient copies with margin
    free = os.sysconf("SC_PAGE_SIZE") * os.sysconf("SC_AVPHYS_PAGES")
    if need > free:
        sys.exit("%s at %d x %d needs about %.0f GB of host memory, %.0f GB are free: scale it down with --rows / --features"
                 % (args.shape, rows, features, need / 1e9, free / 1e9))
    from mmlspark_b200 import capi
    rng = np.random.default_rng(0)
    X = rng.standard_normal((rows + nvalid, features), dtype=np.float32)
    z = (X[:, 0] * 2 + np.sin(3 * X[:, 1]) + X[:, 2] * X[:, 3] + 0.1 * rng.standard_normal(rows + nvalid, dtype=np.float32)).astype(np.float32)
    y = z if args.shape == "cfg2" else (z > 0).astype(np.float32)
    params = BASE + " " + shape["objective"]
    arms = {"full": params, "quant_b4": params + " use_quantized_grad=true num_grad_quant_bins=4",
            "quant_b16": params + " use_quantized_grad=true num_grad_quant_bins=16"}
    ds = capi.Dataset.from_mat(X[:rows], DS_PARAMS).set_field("label", y[:rows])
    dv = capi.Dataset.from_mat(X[rows:], DS_PARAMS, reference=ds).set_field("label", y[rows:])
    del X
    boosters = {}
    res = {k: [] for k in arms}
    k4 = {k: [] for k in arms}
    try:
        for k, p in arms.items():
            boosters[k] = capi.Booster(ds, p)
            boosters[k].add_valid(dv)
        for b in boosters.values():
            for _ in range(args.warmup):
                b.update_one_iter()
        for _ in range(args.rounds):
            for k, b in boosters.items():
                t0 = time.perf_counter()
                for _ in range(args.iters):
                    b.update_one_iter()      # each iteration reads its tree back (a stream sync)
                res[k].append(args.iters / (time.perf_counter() - t0))
            for k, b in boosters.items():   # K4 time per iteration, events on, in a pass of its own
                b.set_profile(True)
                b.get_timing(reset=True)
                for _ in range(args.iters):
                    b.update_one_iter()
                k4[k].append(b.get_timing(reset=True)["hist_ms"] / args.iters)
                b.set_profile(False)
        metric = {k: float(b.get_eval(1)[0]) for k, b in boosters.items()}
        trained = {k: b.current_iteration() for k, b in boosters.items()}
    finally:
        for b in boosters.values():
            b.free()
        dv.free()
        ds.free()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    out = dict(card=card.splitlines()[0] if card else "unknown", shape=args.shape, rows=rows, features=features, iters_per_round=args.iters,
               its_per_s={k: [round(v, 3) for v in vs] for k, vs in res.items()},
               k4_ms_per_iter={k: [round(v, 3) for v in vs] for k, vs in k4.items()},
               median_speedup={k: round(float(np.median(res[k]) / np.median(res["full"])), 4) for k in arms},
               valid_metric=metric, iterations_trained=trained)
    doc = json.dumps(out, indent=1)
    print(doc)
    if args.out:
        with open(args.out, "w") as f:
            f.write(doc + "\n")


if __name__ == "__main__":
    main()
