"""Training rate and gradient-kernel time of rank_xendcg against lambdarank on one GPU, at bench.py's cfg4 shape
(20M rows x 136 features, ~200k query groups of 50-150 documents).

    python tools/xendcg_measure.py [--rows N] [--iters K] [--rounds R] [--query-size Q]

Prints the card's name and power limit, iterations/s of both objectives (timed rounds alternate between them on one dataset), and
the mean time per launch of k_grad_lambdarank and k_grad_xendcg from torch.profiler's CUDA activity in a separate, untimed pass.
--query-size Q replaces cfg4's query groups by groups of Q documents (k_grad_xendcg takes its four sums serially, so long queries
cost it latency; lambdarank runs only when no query has more than 1000 documents)."""
import argparse
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=20_000_000)
    ap.add_argument("--iters", type=int, default=10, help="iterations per timed round")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--query-size", type=int, default=0, help="documents per query group (default: cfg4's 50-150)")
    args = ap.parse_args()
    import numpy as np
    import torch
    import bench
    from mmlspark_b200 import capi
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                          capture_output=True, text=True, check=True).stdout.strip()
    print("card: %s" % card)
    cfg = dict(bench.CONFIGS["cfg4"])
    F = cfg["features"]
    groups = bench.group_sizes(cfg["seed"], args.rows)
    if args.query_size:
        groups = np.full(args.rows // args.query_size, args.query_size, np.int32)
        if args.rows % args.query_size:
            groups = np.append(groups, np.int32(args.rows % args.query_size))
    ds, _, _, _ = bench.build_dataset(capi, cfg, args.rows, F, 0, "device", groups)
    print("data: %d rows x %d features, %d queries" % (args.rows, F, len(groups)))
    params = bench.booster_params(cfg, 1)
    objectives = ("lambdarank", "rank_xendcg") if int(groups.max()) <= 1000 else ("rank_xendcg",)
    boosters = {o: capi.Booster(ds, params.replace("objective=lambdarank", "objective=" + o)) for o in objectives}
    for b in boosters.values():          # warm-up: first launches, allocations
        for _ in range(3):
            b.update_one_iter()
    torch.cuda.synchronize()
    rates = {o: [] for o in boosters}
    for _ in range(args.rounds):
        for o, b in boosters.items():
            t0 = time.perf_counter()
            for _ in range(args.iters):
                b.update_one_iter()
            torch.cuda.synchronize()
            rates[o].append(args.iters / (time.perf_counter() - t0))
    for o, r in rates.items():
        print("%-12s iterations/s per round: %s  (median %.3f)" % (o, " ".join("%.3f" % x for x in r), sorted(r)[len(r) // 2]))
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for b in boosters.values():
            for _ in range(3):
                b.update_one_iter()
        torch.cuda.synchronize()
    for e in prof.key_averages():
        if "k_grad_lambdarank" in e.key or "k_grad_xendcg" in e.key:
            total = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0.0)
            print("kernel %-20s launches %d  mean %.1f us" % ("k_grad_lambdarank" if "lambdarank" in e.key else "k_grad_xendcg", e.count, total / e.count))


if __name__ == "__main__":
    main()
