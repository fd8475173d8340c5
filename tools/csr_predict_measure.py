"""Batched GPU prediction of CSR rows against the dense batched predictor and the per-row CSR predictor, one GPU.

    python tools/csr_predict_measure.py [--rows N] [--cols F] [--density D] [--iters K] [--leaves L] [--dense-rows M]
                                        [--single-rows S] [--wide-rows W] [--wide-iters KW] [--repeats R]

A seeded sparse binary problem of N rows x F columns with about D*F stored values per row is trained for K iterations of L leaves from
CSR.  Prints the card's name and power limit, then raw-score prediction times, each the median of R timed calls after a warm-up:
  - predict_csr_device over all N rows: CUDA-event time (uploads, kernels, download) and the end-to-end call time;
  - predict_csr_device and predict_device over the first M rows, the latter on those rows densified (float64; all N rows densified
    would not fit in host memory), and whether both outputs are identical;
  - the per-row predict_for_csr_single loop over S sampled rows, scaled to N rows;
  - at 2^18 hashed columns (W rows, KW iterations), where a dense matrix cannot be built, predict_csr_device alone."""
import argparse
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

DS = "max_bin=255 is_pre_partition=True num_threads=0"


def sparse_problem(n, F, per_row, seed):
    """per_row distinct ascending columns per row (one in each of per_row equal column ranges), standard normal values"""
    import numpy as np
    rng = np.random.default_rng(seed)
    width = F // per_row
    cols = rng.integers(0, width, (n, per_row), dtype=np.int32) + (np.arange(per_row, dtype=np.int32) * width)[None, :]
    val = rng.standard_normal((n, per_row))
    w = rng.standard_normal(F) * (rng.random(F) < 0.05)
    y = (w[cols] * val).sum(axis=1) + 0.5 * rng.standard_normal(n)
    indptr = np.arange(n + 1, dtype=np.int64) * per_row
    return indptr, cols.reshape(-1), val.reshape(-1), (y > np.median(y)).astype(np.float32)


def train(capi, indptr, indices, data, F, y, iters, leaves):
    ds = capi.Dataset.from_csr(indptr, indices, data, F, DS)
    ds.set_field("label", y)
    b = capi.Booster(ds, DS + " objective=binary num_leaves=%d learning_rate=0.1 verbosity=-1" % leaves)
    t0 = time.perf_counter()
    for _ in range(iters):
        b.update_one_iter()
    return ds, b, time.perf_counter() - t0


def timed(fn, repeats):
    """median event time (ms, or None) and median wall time (ms) of `repeats` calls after one warm-up; fn returns (out, event_ms)"""
    import numpy as np
    out, _ = fn()
    ev, wall = [], []
    for _ in range(repeats):
        t0 = time.perf_counter()
        out, ms = fn()
        wall.append((time.perf_counter() - t0) * 1e3)
        ev.append(ms)
    return out, (float(np.median(ev)) if ev[0] is not None else None), float(np.median(wall))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1_000_000)
    ap.add_argument("--cols", type=int, default=4000)
    ap.add_argument("--density", type=float, default=0.02)
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--leaves", type=int, default=63)
    ap.add_argument("--dense-rows", type=int, default=100_000)
    ap.add_argument("--single-rows", type=int, default=2000)
    ap.add_argument("--wide-rows", type=int, default=1_000_000)
    ap.add_argument("--wide-iters", type=int, default=50)
    ap.add_argument("--repeats", type=int, default=5)
    args = ap.parse_args()
    import numpy as np
    from mmlspark_b200 import capi
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                          capture_output=True, text=True, check=True).stdout.strip()
    print("card: %s" % card)
    RAW = capi.PREDICT_RAW_SCORE
    n, F, R = args.rows, args.cols, args.repeats
    per_row = max(1, int(round(args.density * F)))
    indptr, indices, data, y = sparse_problem(n, F, per_row, 11)
    ds, b, secs = train(capi, indptr, indices, data, F, y, args.iters, args.leaves)
    print("model: %d iterations x %d leaves, trained from CSR %d rows x %d columns, %d stored values per row (%.1f s)"
          % (args.iters, args.leaves, n, F, per_row, secs))

    _, ev, wall = timed(lambda: b.predict_csr_device(indptr, indices, data, F, RAW, return_ms=True), R)
    print("predict_csr_device, %d rows: %.1f ms CUDA events, %.1f ms end to end = %.2f Mrows/s" % (n, ev, wall, n / wall / 1e3))

    m = min(args.dense_rows, n)
    sub = indptr[:m + 1]
    dense = np.zeros((m, F))
    dense[np.repeat(np.arange(m), per_row), indices[:sub[-1]]] = data[:sub[-1]]
    csr_out, cev, cwall = timed(lambda: b.predict_csr_device(sub, indices, data, F, RAW, return_ms=True), R)
    den_out, dev, dwall = timed(lambda: b.predict_device(dense, RAW, return_ms=True), R)
    print("first %d rows: predict_csr_device %.1f ms events / %.1f ms end to end; predict_device on the densified rows (%.2f GB) "
          "%.1f ms events / %.1f ms end to end; outputs identical: %s"
          % (m, cev, cwall, dense.nbytes / 1e9, dev, dwall, np.array_equal(csr_out, den_out)))
    del dense

    rows = np.random.default_rng(1).choice(n, min(args.single_rows, n), replace=False)
    t0 = time.perf_counter()
    for r in rows:
        b.predict_for_csr_single(indices[indptr[r]:indptr[r + 1]], data[indptr[r]:indptr[r + 1]], F, RAW)
    per = (time.perf_counter() - t0) / len(rows)
    print("predict_for_csr_single loop: %.1f us per row over %d sampled rows, %.1f s for %d rows (scaled)" % (per * 1e6, len(rows), per * n, n))
    b.free(); ds.free()

    W, FW = args.wide_rows, 1 << 18
    rng = np.random.default_rng(29)
    wcols = np.sort(rng.integers(0, 4000, (W, 12), dtype=np.int32), axis=1) + (np.arange(12, dtype=np.int32) * 4000)[None, :]
    wval = rng.standard_normal((W, 12))
    wy = (wval[:, :3].sum(axis=1) > 0).astype(np.float32)
    wptr = np.arange(W + 1, dtype=np.int64) * 12
    ds, b, secs = train(capi, wptr, wcols.reshape(-1), wval.reshape(-1), FW, wy, args.wide_iters, args.leaves)
    _, ev, wall = timed(lambda: b.predict_csr_device(wptr, wcols.reshape(-1), wval.reshape(-1), FW, RAW, return_ms=True), R)
    print("2^18 columns (%d rows, 12 stored values per row, %d iterations x %d leaves; dense would be %.0f GB): predict_csr_device "
          "%.1f ms CUDA events, %.1f ms end to end = %.2f Mrows/s" % (W, args.wide_iters, args.leaves, W * FW * 8 / 1e9, ev, wall, W / wall / 1e3))
    b.free(); ds.free()


if __name__ == "__main__":
    main()
