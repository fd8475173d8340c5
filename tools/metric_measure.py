"""Time of LGBM_BoosterGetEval for the sort-based metrics average_precision and auc_mu, next to a NumPy / scikit-learn computation on the
same scores downloaded to the host (what a host loop over the scores would cost, the download included).

Shapes: average_precision at 100M rows (binary, weighted), auc_mu at 10M rows x 10 classes with the default matrix and with a dense
custom auc_mu_weights matrix.  Scores come in through init_score and are evaluated before the first iteration.  Every arm is warmed up,
every timed window ends with a device synchronise, and the card's name and power limit are printed with the result (one JSON document).
Run from the repository root after build()."""
import argparse
import json
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, ".")

DS = "max_bin=255 is_pre_partition=True bin_construct_sample_cnt=200000 num_threads=0"
BASE = "num_leaves=15 learning_rate=0.1 verbosity=-1 "


def _booster(capi, params, y, s, w):
    X = np.random.default_rng(1).standard_normal((len(y), 1), dtype=np.float32)      # one feature: the metric does not read it
    ds = capi.Dataset.from_mat(X, DS).set_field("label", y).set_field("init_score", s).set_field("weight", w)
    return capi.Booster(ds, BASE + params), ds


def _time_device(torch, b, warmup, reps):
    for _ in range(warmup):
        v = b.get_eval(0)
    torch.cuda.synchronize()
    ms = []
    for _ in range(reps):
        t0 = time.perf_counter()
        v = b.get_eval(0)
        torch.cuda.synchronize()
        ms.append((time.perf_counter() - t0) * 1e3)
    return float(v[0]), ms


def _host_ap(b, y, w):
    from sklearn.metrics import average_precision_score
    t0 = time.perf_counter()
    s = b.get_scores(0)
    v = average_precision_score(y, s, sample_weight=w)
    return float(v), (time.perf_counter() - t0) * 1e3


def _host_aucmu(b, y, w, K, Wm):
    from sklearn.metrics import roc_auc_score
    t0 = time.perf_counter()
    S = b.get_scores(0).reshape(K, -1)
    Wm = Wm.copy()
    np.fill_diagonal(Wm, 0.0)
    order = np.argsort(y, kind="stable")
    bounds = np.searchsorted(y[order], np.arange(K + 1))
    vals = []
    for i in range(K):
        for j in range(i + 1, K):
            rows = np.concatenate([order[bounds[i]:bounds[i + 1]], order[bounds[j]:bounds[j + 1]]])
            v = Wm[i] - Wm[j]
            d = (v[i] - v[j]) * (v @ S[:, rows])
            vals.append(roc_auc_score(y[rows] == i, d, sample_weight=w[rows]))
    return float(np.mean(vals)), (time.perf_counter() - t0) * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ap-rows", type=int, default=100_000_000)
    ap.add_argument("--mu-rows", type=int, default=10_000_000)
    ap.add_argument("--classes", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--no-host", action="store_true", help="skip the host computations")
    ap.add_argument("--out", default=None, help="also write the JSON document to this file")
    a = ap.parse_args()
    import torch      # first: it brings its own NCCL, and the engine's library would otherwise load the system one torch cannot use
    from mmlspark_b200 import capi
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                          capture_output=True, text=True).stdout.strip()
    rng = np.random.default_rng(7)
    res = {"card": card}

    n = a.ap_rows
    y = (rng.random(n, dtype=np.float32) < 0.1).astype(np.float32)
    s = np.round(rng.standard_normal(n) + 1.5 * y, 3)
    w = (0.5 + rng.random(n, dtype=np.float32)).astype(np.float32)
    b, ds = _booster(capi, "objective=binary metric=average_precision", y, s, w)
    del s
    v, ms = _time_device(torch, b, a.warmup, a.reps)
    res["average_precision"] = {"rows": n, "value": v, "device_ms": ms, "device_ms_median": float(np.median(ms))}
    if not a.no_host:
        hv, hms = _host_ap(b, y, w)
        res["average_precision"].update(host_value=hv, host_ms=hms)
    print(json.dumps({"average_precision": res["average_precision"]}), flush=True)
    b.free(); ds.free()
    del y, w

    n, K = a.mu_rows, a.classes
    y = rng.integers(0, K, n).astype(np.float32)
    S = rng.standard_normal((K, n)) + 1.0 * (np.arange(K)[:, None] == y[None, :].astype(int))
    w = (0.5 + rng.random(n, dtype=np.float32)).astype(np.float32)
    dense = rng.uniform(0.5, 2.0, (K, K))
    np.fill_diagonal(dense, 0.0)
    for name, Wm, key in (("auc_mu_default", np.ones((K, K)), ""),
                          ("auc_mu_dense_matrix", dense, "auc_mu_weights=" + ",".join(repr(float(x)) for x in dense.ravel()))):
        b, ds = _booster(capi, "objective=multiclass num_class=%d metric=auc_mu %s" % (K, key), y, S.ravel(), w)
        v, ms = _time_device(torch, b, a.warmup, a.reps)
        res[name] = {"rows": n, "classes": K, "value": v, "device_ms": ms, "device_ms_median": float(np.median(ms))}
        if not a.no_host:
            hv, hms = _host_aucmu(b, y, w, K, Wm)
            res[name].update(host_value=hv, host_ms=hms)
        print(json.dumps({name: res[name]}), flush=True)
        b.free(); ds.free()
    doc = json.dumps(res)
    print(doc)
    if a.out:
        with open(a.out, "w") as f:
            f.write(doc + "\n")


if __name__ == "__main__":
    main()
