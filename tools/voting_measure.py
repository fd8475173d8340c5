"""Data-parallel against voting-parallel training with R rank-threads on ONE device (the same-device collective).

The cfg2 shape of bench.py (10M x 256 dense f32 regression, 255 bins, 31 leaves) is split into R contiguous shards, R in {2, 4}.  For each R
the arms data-parallel, voting top_k=20 and voting top_k=5 are warmed up and then alternated over three rounds of `--iters` timed
iterations.  Each arm reports its iterations/s per round, the histogram and record bytes per split round from B200GBM_BoosterGetCommInfo,
and the per-operation split timing of one extra run with B200GBM_SPLIT_TIMING=1 (a subprocess; its stderr line is kept).  On one device the
"all-reduce" is a pass over device memory and voting adds an all-gather and two launches per split, so this measures voting's overhead,
not the network saving it is built for.  The card's name and power limit are read in the same run.

    python tools/voting_measure.py [--rows 10000000] [--features 256] [--iters 20] [--out FILE]
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
ARMS = [("data_parallel", 20), ("voting", 20), ("voting", 5)]


def params(R, learner, top_k):
    return ("metric= boost_from_average=true boosting_type=gbdt tree_learner=%s top_k=%d num_iterations=1000 learning_rate=0.1 "
            "num_leaves=31 max_bin=255 num_machines=%d verbosity=-1 min_data_in_leaf=20 objective=regression num_threads=0"
            % (learner, top_k, R))


def data(rows, features):
    rng = np.random.default_rng(0)
    X = rng.standard_normal((rows, features), dtype=np.float32)
    y = (X[:, 0] * 2 + np.sin(3 * X[:, 1]) + X[:, 2] * X[:, 3] + 0.1 * rng.standard_normal(rows, dtype=np.float32)).astype(np.float32)
    return X, y


def train_rounds(X, y, R, port, warmup, iters, rounds):
    """every arm's boosters are built once on R rank-threads of device 0; the arms then alternate, `rounds` x `iters` timed iterations"""
    from mmlspark_b200 import capi
    bounds = np.linspace(0, len(X), R + 1).astype(np.int64)
    out = {"%s_k%d" % a: dict(its=[], comm=None) for a in ARMS}
    errs = []
    barrier = threading.Barrier(R)

    def task(r):
        try:
            capi.set_device(0)
            capi.network_init(",".join("127.0.0.1:%d" % (port + q) for q in range(R)), port + r, 600, R)
            try:
                sl = slice(int(bounds[r]), int(bounds[r + 1]))
                ds = capi.Dataset.from_mat(X[sl], DS_PARAMS).set_field("label", y[sl])
                boosters = [capi.Booster(ds, params(R, learner, k)) for learner, k in ARMS]
                for b in boosters:
                    for _ in range(warmup):
                        b.update_one_iter()
                    b.get_scores()
                for _ in range(rounds):
                    for (learner, k), b in zip(ARMS, boosters):
                        c0 = b.get_comm_info()
                        barrier.wait()
                        t0 = time.perf_counter()
                        for _ in range(iters):
                            b.update_one_iter()
                        b.get_scores()
                        dt = time.perf_counter() - t0
                        c1 = b.get_comm_info()
                        if r == 0:
                            arm = out["%s_k%d" % (learner, k)]
                            arm["its"].append(iters / dt)
                            s = c1["splits"] - c0["splits"]
                            arm["comm"] = dict(hist_bytes_per_split=(c1["hist_bytes"] - c0["hist_bytes"]) / s,
                                               record_bytes_per_split=(c1["record_bytes"] - c0["record_bytes"]) / s)
                for b in boosters:
                    b.free()
                ds.free()
            finally:
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
    return out


def split_timing(args, R, learner, k):
    """one run of `iters` iterations with B200GBM_SPLIT_TIMING=1 in a subprocess; returns rank 0's timing line"""
    cmd = [sys.executable, os.path.abspath(__file__), "--child"] + [str(v) for v in (R, learner, k, args.rows, args.features, args.iters)]
    p = subprocess.run(cmd, capture_output=True, text=True, env=dict(os.environ, B200GBM_SPLIT_TIMING="1"), cwd=ROOT)
    lines = [l for l in p.stderr.splitlines() if l.startswith("[b200gbm split timing]")]
    return lines[0] if lines else p.stderr[-500:]


def child(R, learner, k, rows, features, iters):
    from mmlspark_b200 import capi
    X, y = data(rows, features)
    bounds = np.linspace(0, rows, R + 1).astype(np.int64)

    def task(r):
        capi.set_device(0)
        capi.network_init(",".join("127.0.0.1:%d" % (31500 + q) for q in range(R)), 31500 + r, 600, R)
        sl = slice(int(bounds[r]), int(bounds[r + 1]))
        ds = capi.Dataset.from_mat(X[sl], DS_PARAMS).set_field("label", y[sl])
        b = capi.Booster(ds, params(R, learner, k))
        for _ in range(iters):
            b.update_one_iter()
        b.free(); ds.free()
        capi.network_free()

    ts = [threading.Thread(target=task, args=(r,)) for r in range(R)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()


def main():
    if len(sys.argv) > 1 and sys.argv[1] == "--child":
        a = sys.argv[2:]
        child(int(a[0]), a[1], int(a[2]), int(a[3]), int(a[4]), int(a[5]))
        return
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=10_000_000)
    ap.add_argument("--features", type=int, default=256)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    X, y = data(args.rows, args.features)
    res = dict(card=card, rows=args.rows, features=args.features, iters_per_round=args.iters, results={})
    for i, R in enumerate((2, 4)):
        arms = train_rounds(X, y, R, 31000 + 20 * i, 3, args.iters, 3)
        for learner, k in ARMS:
            arms["%s_k%d" % (learner, k)]["split_timing"] = split_timing(args, R, learner, k)
        res["results"]["R%d" % R] = arms
    doc = json.dumps(res, indent=1)
    print(doc)
    if args.out:
        with open(args.out, "w") as f:
            f.write(doc)


if __name__ == "__main__":
    main()
