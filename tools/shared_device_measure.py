"""Cost of data-parallel training with R rank-threads on ONE device (the same-device collective of LGBM_NetworkInit).

The cfg2 shape of bench.py (10M x 256 dense f32 regression, 255 bins, 31 leaves) is split into R contiguous shards, R in {1, 2, 4}, every
rank-thread on device 0.  Ranks on one device share one stream, so their kernels run one after another: R ranks cost at least one rank over
all rows, plus the collectives and the smaller per-rank launches.  The "merged" arms train the same R shards as ONE rank over one dataset
built from the R row parts (LGBM_DatasetCreateFromMats, what single-dataset mode does), and report its ingest time next to
LGBM_DatasetCreateFromMat's on the whole matrix.  After a warm-up the script alternates the arms over three rounds of 20 timed iterations
and prints the iterations/s of every round.  A separate run under torch.profiler (R = 2) gives the device time per launch of
k_allreduce_same_device.  The card's name and power limit are read in the same run.

    python tools/shared_device_measure.py [--rows 10000000] [--features 256] [--out FILE]

It prints one JSON document, and also writes it to FILE when --out is given.
"""
import argparse
import json
import os
import subprocess
import sys
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

DS_PARAMS = "max_bin=255 is_pre_partition=True bin_construct_sample_cnt=200000 num_threads=0"


def params(R):
    return ("metric= boost_from_average=true is_pre_partition=True boosting_type=gbdt tree_learner=data_parallel num_iterations=1000 "
            "learning_rate=0.1 num_leaves=31 max_bin=255 bagging_fraction=1.0 bagging_freq=0 feature_fraction=1.0 max_depth=-1 "
            "min_sum_hessian_in_leaf=0.001 num_machines=%d verbosity=-1 lambda_l1=0.0 lambda_l2=0.0 min_gain_to_split=0.0 "
            "max_delta_step=0.0 min_data_in_leaf=20 objective=regression num_threads=0" % R)


def run(X, y, R, warmup, iters, port, on_timed=None):
    """R rank-threads on device 0; returns the wall time of `iters` iterations after `warmup`, all ranks barriered by the collectives"""
    from mmlspark_b200 import capi
    machines = ",".join("127.0.0.1:%d" % (port + r) for r in range(R))
    bounds = np.linspace(0, len(X), R + 1).astype(np.int64)
    ready = threading.Barrier(R)
    secs, errs = [0.0] * R, []

    def task(r):
        try:
            capi.set_device(0)
            if R > 1:
                capi.network_init(machines, port + r, 300, R)
            try:
                sl = slice(int(bounds[r]), int(bounds[r + 1]))
                ds = capi.Dataset.from_mat(X[sl], DS_PARAMS).set_field("label", y[sl])
                b = capi.Booster(ds, params(R))
                for _ in range(warmup):
                    b.update_one_iter()
                b.get_scores()                       # a host read: the warm-up has finished on the device
                ready.wait()
                t0 = time.perf_counter()
                with (on_timed() if on_timed and r == 0 else _Null()):
                    for _ in range(iters):
                        b.update_one_iter()
                    b.get_scores()
                secs[r] = time.perf_counter() - t0
                b.free(); ds.free()
            finally:
                if R > 1:
                    capi.network_free()
        except Exception as e:   # noqa
            errs.append((r, repr(e)))

    ts = [threading.Thread(target=task, args=(r,)) for r in range(R)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    if errs:
        raise RuntimeError(errs)
    return max(secs)


def run_merged(X, y, R, warmup, iters):
    """the R shards of run() as ONE rank (single-dataset mode): one dataset from the R row parts through LGBM_DatasetCreateFromMats;
    returns the wall time of `iters` iterations after `warmup` and the dataset's ingest time in ms"""
    from mmlspark_b200 import capi
    bounds = np.linspace(0, len(X), R + 1).astype(np.int64)
    capi.set_device(0)
    ds = capi.Dataset.from_mats([X[int(bounds[r]):int(bounds[r + 1])] for r in range(R)], DS_PARAMS).set_field("label", y)
    ingest = ds.ingest_ms()
    b = capi.Booster(ds, params(1))
    try:
        for _ in range(warmup):
            b.update_one_iter()
        b.get_scores()
        t0 = time.perf_counter()
        for _ in range(iters):
            b.update_one_iter()
        b.get_scores()
        return time.perf_counter() - t0, ingest
    finally:
        b.free(); ds.free()


def ingest_from_mat(X):
    """ingest time in ms of LGBM_DatasetCreateFromMat on the whole matrix (the concatenation of the shards)"""
    from mmlspark_b200 import capi
    capi.set_device(0)
    ds = capi.Dataset.from_mat(X, DS_PARAMS)
    try:
        return ds.ingest_ms()
    finally:
        ds.free()


class _Null:
    def __enter__(self):
        return self

    def __exit__(self, *a):
        return False


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=10_000_000)
    ap.add_argument("--features", type=int, default=256)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None, help="also write the JSON document to this file")
    a = ap.parse_args()
    # torch first: it brings its own NCCL, and the engine's library would otherwise load the system one torch cannot use
    from torch.profiler import ProfilerActivity, profile
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                          capture_output=True, text=True).stdout.strip()
    rng = np.random.default_rng(2024)
    X = rng.standard_normal((a.rows, a.features), dtype=np.float32)
    y = (X[:, 0] + 0.5 * X[:, 1] * X[:, 2] + np.sin(X[:, 3]) + 0.3 * rng.standard_normal(a.rows, dtype=np.float32)).astype(np.float32)
    rates = {"1": [], "2": [], "4": [], "merged_2": [], "merged_4": []}
    ingest = {"from_mat": [], "from_mats_2": [], "from_mats_4": []}
    port = 27000
    for rnd in range(a.rounds):
        order = ["1", "2", "merged_2", "4", "merged_4"]
        for arm in (order if rnd % 2 == 0 else order[::-1]):
            if arm.startswith("merged_"):
                R = int(arm[len("merged_"):])
                s, ms = run_merged(X, y, R, a.warmup, a.iters)
                ingest["from_mats_%d" % R].append(ms)
            else:
                s = run(X, y, int(arm), a.warmup, a.iters, port)
                port += 10
            rates[arm].append(a.iters / s)
            print("round %d %s: %.2f iters/s" % (rnd, arm, a.iters / s), flush=True)
        ingest["from_mat"].append(ingest_from_mat(X))
    # kernel time of the same-device all-reduce, in a run of its own
    prof_box = {}

    def on_timed():
        p = profile(activities=[ProfilerActivity.CUDA])
        prof_box["p"] = p
        return p

    run(X, y, 2, a.warmup, 5, port, on_timed=on_timed)
    ev = [e for e in prof_box["p"].events() if "k_allreduce_same_device" in e.name]
    us = [e.time_range.elapsed_us() for e in ev]
    per_launch_us = float(np.mean(us)) if us else float("nan")
    out = dict(card=card, rows=a.rows, features=a.features, iters=a.iters,
               iters_per_s={arm: dict(median=float(np.median(v)), runs=[round(x, 3) for x in v]) for arm, v in rates.items()},
               ingest_ms={k: dict(median=float(np.median(v)), runs=[round(x, 1) for x in v]) for k, v in ingest.items()},
               allreduce_same_device=dict(launches=len(ev), mean_us=per_launch_us))
    print(json.dumps(out))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
