"""Prediction early stopping (pred_early_stop) on one GPU: rows/s of the device predictor with and without it.

    python tools/pred_early_stop_measure.py [--rows N] [--train-rows T] [--cols F] [--repeats R] [--sample S] [--out PATH]

Two seeded models are trained on T rows x F columns (31 leaves): binary over 2000 iterations and 10-class multiclass over 500.  N rows
of the same problem sit on the device as float32, so each timed call is the predictor's CUDA-event time (kernels and the score
download), not an upload.  Each arm is the median of R calls, after a warm-up, with the arms of one model alternated in every round:
  - "parent": B200GBM_BoosterPredictForMatDevice, the entry point without a parameter, which runs k_predict_raw as before;
  - "off": the entry point with a parameter and pred_early_stop=false, which must run the same kernel at the same speed;
  - "never": early stopping with a margin no row reaches, the cost of k_predict_raw_es when nothing stops;
  - "margin m": early stopping at freq 10 and margin m (binary: 2, 5, 10; multiclass: 2, 5, 10).
For each early-stopping arm the share of (row, tree) walks skipped is computed on the host over S sampled rows, from the NumPy rule
(per-tree leaf values, fp64 sums in model order, the margin after every 10 iterations), and the device's raw scores of those rows are
checked against it bit for bit.  Prints the card's name and power limit, and one JSON document."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

DS = "max_bin=255 is_pre_partition=True num_threads=0"
FREQ = 10


def problem(n, F, classes, seed):
    rng = np.random.default_rng(seed)
    X = rng.standard_normal((n, F)).astype(np.float32)
    w = rng.standard_normal(F) * (rng.random(F) < 0.25)
    z = X @ w + np.sin(2 * X[:, 0]) + 0.5 * rng.standard_normal(n)
    y = np.digitize(z, np.quantile(z, np.arange(1, classes) / classes)).astype(np.float32)
    return X, y


def train(capi, X, y, params, iters):
    ds = capi.Dataset.from_mat(X, DS)
    ds.set_field("label", y)
    b = capi.Booster(ds, params + " num_leaves=31 learning_rate=0.1 min_data_in_leaf=20 verbosity=-1 " + DS)
    for _ in range(iters):
        b.update_one_iter()
    return capi.Booster(model_str=b.save_model_to_string())


def leaf_values(capi, b, X):
    """[rows][trees] the value of the leaf each row reaches in each tree"""
    from mmlspark_b200.modeltext import parse_model
    trees = parse_model(b.save_model_to_string())["trees"]
    leaves = b.predict_device(X, capi.PREDICT_LEAF_INDEX).astype(np.int64)
    out = np.empty(leaves.shape)
    for t, tree in enumerate(trees):
        out[:, t] = np.asarray(tree["leaf_value"], dtype=np.float64)[leaves[:, t]]
    return out


def restated(vals, K, freq, margin):
    """(raw scores, iterations walked) of every row: the early-stopping rule on per-tree leaf values; freq None = off"""
    n, T = vals.shape
    iters = T // K
    sums = np.cumsum(vals.reshape(n, iters, K), axis=1)      # fp64 adds in model order, per class
    walked = np.full(n, iters)
    if freq is not None:
        for it in range(freq, iters + 1, freq):
            s = sums[:, it - 1]
            if K == 1:
                m = 2.0 * np.abs(s[:, 0])
            else:
                top = np.sort(s, axis=1)
                m = top[:, -1] - top[:, -2]
            stop = (walked == iters) & (m > margin)
            walked[stop] = it
    return sums[np.arange(n), walked - 1], walked


def device_predict(capi, b, ptr, n, F, K, parameter, out, old=False):
    """one raw-score call on device-resident float32 rows; returns its CUDA-event milliseconds"""
    n_out, ms = C.c_int64(0), C.c_double(0)
    L = capi.load()
    if old:
        capi.check(L.B200GBM_BoosterPredictForMatDevice(b.handle, ptr, C.c_int(capi.DTYPE_FLOAT32), C.c_int64(n), C.c_int32(F),
                                                        C.c_int(capi.PREDICT_RAW_SCORE), C.c_int(0), C.c_int(-1), C.byref(n_out),
                                                        out.ctypes.data_as(C.POINTER(C.c_double)), C.byref(ms)))
    else:
        capi.check(L.B200GBM_BoosterPredictForMatDeviceWithParameter(b.handle, ptr, C.c_int(capi.DTYPE_FLOAT32), C.c_int64(n), C.c_int32(F),
                                                                     C.c_int(capi.PREDICT_RAW_SCORE), C.c_int(0), C.c_int(-1), parameter.encode(),
                                                                     C.byref(n_out), out.ctypes.data_as(C.POINTER(C.c_double)), C.byref(ms)))
    assert n_out.value == n * K
    return ms.value


def measure(capi, name, b, K, X, buf, margins, repeats, sample):
    n, F = X.shape
    es = lambda m: "pred_early_stop=true pred_early_stop_freq=%d pred_early_stop_margin=%r" % (FREQ, m)
    arms = [("parent", None, True), ("off", "pred_early_stop=false", False), ("never", es(1e300), False)]
    arms += [("margin %g" % m, es(m), False) for m in margins]
    outs = {a: np.zeros(n * K) for a, _, _ in arms}
    for a, p, old in arms:      # warm-up
        device_predict(capi, b, buf.ptr, n, F, K, p, outs[a], old)
    times = {a: [] for a, _, _ in arms}
    for _ in range(repeats):
        for a, p, old in arms:
            times[a].append(device_predict(capi, b, buf.ptr, n, F, K, p, outs[a], old))
    assert np.array_equal(outs["off"], outs["parent"]) and np.array_equal(outs["never"], outs["parent"])
    vals = leaf_values(capi, b, X[:sample])
    T = vals.shape[1]
    full, _ = restated(vals, K, None, 0.0)
    assert np.array_equal(outs["parent"].reshape(n, K)[:sample], full)
    res = {"model": name, "rows": n, "trees": T, "K": K, "arms": []}
    for a, p, _ in arms:
        ms = float(np.median(times[a]))
        arm = {"arm": a, "ms": round(ms, 3), "rows_per_s": round(n / (ms / 1e3)), "spread_ms": [round(min(times[a]), 3), round(max(times[a]), 3)]}
        if a.startswith("margin"):
            m = float(a.split()[1])
            raw, walked = restated(vals, K, FREQ, m)
            assert np.array_equal(outs[a].reshape(n, K)[:sample], raw), a
            arm["walks_skipped"] = round(1.0 - walked.sum() / (len(walked) * (T // K)), 4)
        arm["speedup_vs_parent"] = round(float(np.median(times["parent"])) / ms, 3)
        res["arms"].append(arm)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1_000_000)
    ap.add_argument("--train-rows", type=int, default=200_000)
    ap.add_argument("--cols", type=int, default=64)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--sample", type=int, default=10_000)
    ap.add_argument("--binary-iters", type=int, default=2000)
    ap.add_argument("--multi-iters", type=int, default=500)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    from mmlspark_b200 import capi
    capi.load()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                          capture_output=True, text=True).stdout.strip()
    print("card:", card, flush=True)
    report = {"card": card, "freq": FREQ, "results": []}
    for name, classes, params, iters in (("binary", 2, "objective=binary", a.binary_iters),
                                         ("multiclass10", 10, "objective=multiclass num_class=10", a.multi_iters)):
        Xt, yt = problem(a.train_rows, a.cols, classes, 1)
        b = train(capi, Xt, yt, params, iters)
        X, _ = problem(a.rows, a.cols, classes, 2)
        buf = capi.DeviceBuffer(X.nbytes)
        try:
            capi.memcpy(buf.ptr, X.ctypes.data, X.nbytes)
            r = measure(capi, name, b, b.num_model_per_iteration(), X, buf, (2.0, 5.0, 10.0), a.repeats, min(a.sample, a.rows))
        finally:
            buf.free()
        print(json.dumps(r), flush=True)
        report["results"].append(r)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(report, f, indent=1)


if __name__ == "__main__":
    main()
