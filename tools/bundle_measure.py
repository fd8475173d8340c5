"""Exclusive feature bundling on one-hot data, one GPU: a seeded CSR dataset of N rows x (B categorical columns one-hot encoded into L
levels each + D dense columns), created and trained with enable_bundle=true and false.

    python tools/bundle_measure.py [--rows N] [--blocks B] [--levels L] [--dense D] [--iters K] [--rounds R]

Prints the card's name and power limit, then per setting: storage columns and bin bytes, ingest time (LGBM_DatasetCreateFromCSR, CUDA
events), iterations/s (timed rounds alternate between the two boosters) and K4 time per iteration (CUDA events around every K4 launch,
in a separate profiled round), and whether both models are identical."""
import argparse
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def one_hot_csr(n, blocks, levels, dense, seed):
    import numpy as np
    rng = np.random.default_rng(seed)
    per_row = blocks + dense
    idx = np.empty((n, per_row), dtype=np.int32)
    val = np.empty((n, per_row), dtype=np.float64)
    # skewed level frequencies, as a categorical column typically has
    p = 1.0 / np.arange(1, levels + 1); p /= p.sum()
    for b in range(blocks):
        idx[:, b] = b * levels + rng.choice(levels, n, p=p)
        val[:, b] = 1.0
    idx[:, blocks:] = blocks * levels + np.arange(dense, dtype=np.int32)[None, :]
    val[:, blocks:] = rng.standard_normal((n, dense))
    w = rng.standard_normal(blocks * levels) * 0.3
    y = w[idx[:, :blocks]].sum(axis=1) + val[:, blocks:blocks + 4].sum(axis=1) + 0.5 * rng.standard_normal(n)
    indptr = (np.arange(n + 1, dtype=np.int64) * per_row).astype(np.int32 if n * per_row < 2**31 else np.int64)
    return indptr, idx.reshape(-1), val.reshape(-1), blocks * levels + dense, (y > np.median(y)).astype(np.float32)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=2_000_000)
    ap.add_argument("--blocks", type=int, default=50)
    ap.add_argument("--levels", type=int, default=200)
    ap.add_argument("--dense", type=int, default=64)
    ap.add_argument("--iters", type=int, default=10, help="iterations per timed round")
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    import numpy as np
    from mmlspark_b200 import capi
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                          capture_output=True, text=True, check=True).stdout.strip()
    print("card: %s" % card)
    indptr, indices, data, F, y = one_hot_csr(args.rows, args.blocks, args.levels, args.dense, 17)
    print("data: %d rows x %d columns (%d one-hot blocks of %d levels + %d dense), %d stored values"
          % (args.rows, F, args.blocks, args.levels, args.dense, len(data)))
    base = "max_bin=255 is_pre_partition=True num_threads=0"
    train = "objective=binary metric=binary_logloss num_leaves=63 learning_rate=0.1"
    sets = {}
    for on in (True, False):
        ds_params = base + (" enable_bundle=false" if not on else "")
        ds = capi.Dataset.from_csr(indptr, indices, data, F, ds_params)
        ds.set_field("label", y)
        ncols, _ = ds.bundles()
        b = capi.Booster(ds, ds_params + " " + train)
        b.update_one_iter()      # warm-up: first launches, column copy
        sets[on] = dict(ds=ds, booster=b, columns=ncols, bin_bytes=((ncols + 31) // 32) * 32 * args.rows, ingest_ms=ds.ingest_ms(), times=[])
    for _ in range(args.rounds):
        for on in (True, False):
            b = sets[on]["booster"]
            t0 = time.perf_counter()
            for _ in range(args.iters):
                b.update_one_iter()
            sets[on]["times"].append(time.perf_counter() - t0)      # UpdateOneIter ends in a device synchronise
    for on in (True, False):
        b = sets[on]["booster"]
        b.set_profile(True); b.get_timing(reset=True)
        for _ in range(args.iters):
            b.update_one_iter()
        t = b.get_timing(reset=True)
        b.set_profile(False)
        s = sets[on]
        s["k4_ms_per_iter"] = t["hist_ms"] / max(t["iterations"], 1)
        s["iters_per_s"] = args.iters * len(s["times"]) / sum(s["times"])
    same = sets[True]["booster"].save_model_to_string().split("\nparameters:")[0] == sets[False]["booster"].save_model_to_string().split("\nparameters:")[0]
    for on in (True, False):
        s = sets[on]
        print("enable_bundle=%s: columns=%d bin_bytes=%.3f GB ingest=%.1f ms iters/s=%.2f (rounds: %s) K4=%.2f ms/iter"
              % (str(on).lower(), s["columns"], s["bin_bytes"] / 1e9, s["ingest_ms"], s["iters_per_s"],
                 ", ".join("%.2f" % (args.iters / x) for x in s["times"]), s["k4_ms_per_iter"]))
    print("trees identical: %s" % same)
    for on in (True, False):
        sets[on]["booster"].free(); sets[on]["ds"].free()


if __name__ == "__main__":
    main()
