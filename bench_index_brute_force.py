"""Measure brute-force search served from an index's own device rows (b200vs_brute_force_search / _range_search) against
the reader's current path: the same live rows, in ascending id order from host memory, pushed in 2048-row tiles
(FLAGS_vector_index_bruteforce_batch_count) through b200vs_scan_* / b200vs_scan_range_*.  The reader path timed here
starts from decoded host rows, so it leaves out the RocksDB iteration and protobuf decoding the reader also pays.

Indexes: HNSW L2 and IVF-Flat L2 (nlist 1024), rows x 768 uniform floats; nq 1 and 256; top-10, and range with a radius
that keeps about 0.1 % of the rows, max_results 1024.  Every configuration first checks that both paths return the same
ids, distance bits and counts, then prints one JSON line: median wall time of each path (host clock around the
synchronous call, after a warm-up) and the speed-up.  The card name and power limit come first.
Usage: python bench_index_brute_force.py [--rows N] [--hnsw-rows N] [--dim D] [--reps R]"""
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


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                              text=True, timeout=60).stdout.strip().splitlines()[0]
    except (OSError, IndexError, subprocess.SubprocessError):
        return "unknown"


def median_s(fn, reps):
    fn()  # warm-up: module load, scratch sizing
    t = []
    for _ in range(reps):
        t0 = time.perf_counter()
        out = fn()
        t.append(time.perf_counter() - t0)
    return float(np.median(t)), out


def reader_topk(x, ids, xq, k):
    sc = b200vs.BruteForceScan(b200vs.L2, x.shape[1], xq, k)
    for a in range(0, len(ids), TILE):
        sc.push(x[a:a + TILE], ids[a:a + TILE])
    return sc.finish()


def reader_range(x, ids, xq, radius, cap):
    sc = b200vs.BruteForceRangeScan(b200vs.L2, x.shape[1], xq, radius, cap)
    for a in range(0, len(ids), TILE):
        sc.push(x[a:a + TILE], ids[a:a + TILE])
    return sc.finish()


def same(a, b):
    return all(np.array_equal(u.view(np.uint32) if u.dtype == np.float32 else u, v.view(np.uint32) if v.dtype == np.float32 else v)
               for u, v in zip(a, b))


def run(name, ix, x, ids, rng, reps):
    order = np.argsort(ids, kind="stable")
    xs, ids_s = np.ascontiguousarray(x[order]), ids[order]
    for nq in (1, 256):
        xq = rng.random((nq, x.shape[1]), dtype=np.float32)
        s = x[rng.choice(len(x), 4096, replace=False)].astype(np.float64)
        radius = float(np.quantile(((s[None, :, :] - xq[:4, None, :].astype(np.float64)) ** 2).sum(-1), 0.001))
        for mode in ("top-10", "range 0.1%"):
            if mode == "top-10":
                t_ix, r_ix = median_s(lambda: ix.brute_force_search(xq, 10), reps)
                t_rd, r_rd = median_s(lambda: reader_topk(xs, ids_s, xq, 10), max(1, reps // 3))
            else:
                t_ix, r_ix = median_s(lambda: ix.brute_force_range_search(xq, radius, 1024), reps)
                t_rd, r_rd = median_s(lambda: reader_range(xs, ids_s, xq, radius, 1024), max(1, reps // 3))
            print(json.dumps({"index": name, "rows": len(ids), "nq": nq, "search": mode, "parity": same(r_ix, r_rd),
                              "index_ms": 1e3 * t_ix, "reader_scan_ms": 1e3 * t_rd, "speedup": t_rd / t_ix}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1_000_000)
    ap.add_argument("--hnsw-rows", type=int, default=1_000_000)
    ap.add_argument("--dim", type=int, default=768)
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "bench_index_brute_force.py measures on a CUDA device"
    torch.zeros(1, device="cuda")
    print(json.dumps({"card": card(), "dim": args.dim, "tile": TILE}), flush=True)
    rng = np.random.default_rng(0)

    x = rng.random((args.rows, args.dim), dtype=np.float32)
    ids = rng.permutation(args.rows).astype(np.int64)
    iv = b200vs.Index(b200vs.IVF_FLAT, b200vs.L2, args.dim, nlist=1024)
    iv.train(x[: 256 * 1024])
    for a in range(0, args.rows, 65536):
        iv.add(x[a:a + 65536], ids[a:a + 65536])
    run("ivf_flat", iv, x, ids, rng, args.reps)
    del iv

    n = args.hnsw_rows
    hx, hids = x[:n], ids[:n]
    hn = b200vs.Index(b200vs.HNSW, b200vs.L2, args.dim, hnsw_m=16, hnsw_efc=64, max_elements=n)
    hn.add_batched(hx, hids)
    run("hnsw", hn, hx, hids, rng, args.reps)


if __name__ == "__main__":
    main()
