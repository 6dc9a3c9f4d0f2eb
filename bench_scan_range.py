"""Measure the streaming brute-force range scan (b200vs_scan_range_*) against the top-k scan (b200vs_scan_*) at the
reader's shape: 1 M rows x 768 floats pushed in 2048-row tiles (FLAGS_vector_index_bruteforce_batch_count), L2, for
nq = 1, 64 and 1024 queries.  Two radii: one that keeps about 0.1 % of the rows per query, and one that fills the
1024-hit cap within the first tile (every later push then only uploads its tile and each CTA returns at once).

Per configuration it prints one JSON line: wall time per push (host clock around the synchronous push: upload,
normalise, kernel), device time of all kernels and of the host-to-device copies per push (torch.profiler with CUDA
activities, in a separate pass so tracing does not slow the timed one), rows scanned per second of wall time, and the
mean hits kept per query.  The card name and power limit come first.  Usage: python bench_scan_range.py [--rows N] [--dim D] [--nq 1,64,1024]."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "dingo-store_b200", "python"))
import b200vs  # noqa: E402

TILE = 2048
POOL_TILES = 64  # distinct tiles cycled through the scan (ids stay unique per tile); the hit rate is the data's


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                              text=True, timeout=60).stdout.strip().splitlines()[0]
    except (OSError, IndexError, subprocess.SubprocessError):
        return "unknown"


def radius_for_fraction(pool, xq, frac):
    """L2 radius below which about `frac` of the rows fall, from a sample of queries and rows (float64)."""
    X = pool[: min(len(pool), 32)].reshape(-1, pool.shape[-1]).astype(np.float64)
    Q = xq[:16].astype(np.float64)
    d2 = (X * X).sum(1)[None, :] + (Q * Q).sum(1)[:, None] - 2.0 * Q @ X.T
    return float(np.quantile(d2, frac))


def tiles(pool, rows):
    pushed, t = 0, 0
    while pushed < rows:
        n = min(TILE, rows - pushed)
        yield pool[t % len(pool)][:n], np.arange(pushed, pushed + n, dtype=np.int64)
        pushed += n
        t += 1


def one_pass(make, pool, rows):
    sc = make()
    times = []
    for x, ids in tiles(pool, rows):
        t0 = time.perf_counter()
        sc.push(x, ids)
        times.append(time.perf_counter() - t0)
    out = sc.finish()
    return np.array(times), out


def device_ms(make, pool, rows):
    """(kernel ms, host-to-device copy ms) of one profiled pass: every kernel the scan launches, every upload."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        one_pass(make, pool, rows)
        torch.cuda.synchronize()
    kern = h2d = 0.0
    for e in prof.key_averages():
        us = getattr(e, "device_time_total", 0.0) or getattr(e, "cuda_time_total", 0.0)
        if "Memcpy HtoD" in e.key:
            h2d += us
        elif "Memcpy" not in e.key and "Memset" not in e.key:
            kern += us
    return kern / 1000.0, h2d / 1000.0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1_000_000)
    ap.add_argument("--dim", type=int, default=768)
    ap.add_argument("--nq", default="1,64,1024")
    ap.add_argument("--topk", type=int, default=10)
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "bench_scan_range.py measures on a CUDA device"
    torch.zeros(1, device="cuda")
    print(json.dumps({"card": card(), "rows": args.rows, "dim": args.dim, "tile": TILE}), flush=True)
    rng = np.random.default_rng(0)
    pool = rng.random((POOL_TILES, TILE, args.dim), dtype=np.float32)
    ntiles = -(-args.rows // TILE)
    for nq in [int(v) for v in args.nq.split(",")]:
        xq = rng.random((nq, args.dim), dtype=np.float32)
        runs = [("range 0.1%", radius_for_fraction(pool, xq, 0.001)), ("range cap-fill", 1e30)]
        for name, radius in runs:
            make = lambda r=radius: b200vs.BruteForceRangeScan(b200vs.L2, args.dim, xq, r, 1024)  # noqa: E731
            one_pass(make, pool, 8 * TILE)  # warm-up: module load, allocations
            t, (_, _, C) = one_pass(make, pool, args.rows)
            kms, hms = device_ms(make, pool, args.rows)
            print(json.dumps({"scan": name, "nq": nq, "radius": radius, "pushes": ntiles, "wall_ms_per_push": 1e3 * t.mean(),
                              "wall_ms_per_push_p50": 1e3 * float(np.median(t)), "kernel_ms_per_push": kms / ntiles,
                              "h2d_ms_per_push": hms / ntiles,
                              "rows_per_s": args.rows / t.sum(), "mean_hits_per_query": float(C.mean())}), flush=True)
        make = lambda: b200vs.BruteForceScan(b200vs.L2, args.dim, xq, args.topk)  # noqa: E731
        one_pass(make, pool, 8 * TILE)
        t, _ = one_pass(make, pool, args.rows)
        kms, hms = device_ms(make, pool, args.rows)
        print(json.dumps({"scan": f"top-k k={args.topk}", "nq": nq, "pushes": ntiles, "wall_ms_per_push": 1e3 * t.mean(),
                          "wall_ms_per_push_p50": 1e3 * float(np.median(t)), "kernel_ms_per_push": kms / ntiles,
                          "h2d_ms_per_push": hms / ntiles,
                          "rows_per_s": args.rows / t.sum()}), flush=True)


if __name__ == "__main__":
    main()
