"""Split and merge rebuilds on the GPU (b200vs_rebuild_from_range) against the host rebuild a VectorIndexManager runs today
for each new region: b200vs_train, then b200vs_add_with_ids in 32768-row calls, over the region's rows in ascending id
order, already in host memory (the RocksDB scan in front of them is not included, as in bench_rebuild.py).

Workloads (regions auto-split at about 512 MB, so a 768-d region splits at about 170 k rows):
  split_170k  IVF-Flat L2, 170 k x 768, nlist 1024, split at its median id: both children are rebuilt from the parent's index.
  split_1m    the same at 1 M rows.
  merge_2x500k  two IVF-Flat L2 regions of 500 k x 768 (nlist 1024) merged into one: the target is rebuilt from both indexes.
  hnsw_split_1m HNSW L2, 1 M x 128, m 32, efconstruction 64, split at its median id.  The host rebuild is one
              b200vs_hnsw_add_batched call over the child's sorted host rows, which builds the same graph (the row-at-a-time
              host builder of b200vs_add_with_ids builds another graph and would not be comparable); rebuild_from_range adds no
              device gather here, since HNSW rows live in the host graph.

Every timed GPU result is checked equal to the host-built index (trained state, lists or graph, and search results) before
timing.  GPU and host runs alternate.  Prints one JSON line per workload with the GPU name and power limit (and appends it to
--out when given).
"""
import argparse
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "dingo-store_b200", "python"))
import b200vs  # noqa: E402
from bench_rebuild import check_equal, gpu_info, host_rebuild, live_sorted  # noqa: E402

I64_MAX = 2 ** 63 - 1


def region(kind, n, d, params, id0, rng):
    """An index holding n random rows under the ids [id0, id0 + n), added in a shuffled order."""
    x = rng.standard_normal((n, d)).astype(np.float32)
    ids = (rng.permutation(n) + id0).astype(np.int64)
    ix = b200vs.Index(kind, b200vs.L2, d, **params)
    if kind == b200vs.HNSW:
        ix.add_batched(x, ids)
    else:
        ix.train(x[:256 * params["nlist"]])
        for a in range(0, n, 262144):
            ix.add(x[a:a + 262144], ids[a:a + 262144])
    return ix


def nlist_of(ix):
    """The index's own list count: an IVF index trained on fewer rows than nlist has degenerated to one list."""
    if ix.type == b200vs.HNSW:
        return 1
    st = ix.get_trained_state()
    return int(st[:32].view(np.int64)[1])


def run(name, kind, d, params, srcs, targets, reps, out, rng):
    """targets: the (id_min, id_max) of each new region, each rebuilt from every index of srcs."""
    host_rows = []
    for lo, hi in targets:  # each new region's rows as the host would hold them: ascending id order
        parts = [live_sorted(s, kind, nlist_of(s)) for s in srcs]
        x = np.concatenate([p[0] for p in parts])
        ids = np.concatenate([p[1] for p in parts])
        keep = (ids >= lo) & (ids < hi)
        o = np.argsort(ids[keep], kind="stable")
        host_rows.append((x[keep][o], ids[keep][o]))
    chunked = kind != b200vs.HNSW
    q = rng.standard_normal((64, d)).astype(np.float32)

    def gpu_rebuild(lo, hi):
        dst = b200vs.Index(kind, b200vs.L2, d, **params)
        dst.rebuild_from_range(srcs, lo, hi)  # returns when the index is complete
        return dst

    for (lo, hi), (x, ids) in zip(targets, host_rows):  # equality of every timed result before any timing
        dev = gpu_rebuild(lo, hi)
        check_equal(dev, host_rebuild(kind, x, ids, params, b200vs.L2, chunked), kind, nlist_of(dev), q)

    t_dev, t_host = [], []
    for _ in range(reps):  # alternate them so drift on the shared machine hits each
        t0 = time.perf_counter()
        for lo, hi in targets:
            gpu_rebuild(lo, hi)  # each new index is freed before the next one is built
        t_dev.append(time.perf_counter() - t0)
        t0 = time.perf_counter()
        for x, ids in host_rows:
            h = host_rebuild(kind, x, ids, params, b200vs.L2, chunked)
            del h
        t_host.append(time.perf_counter() - t0)
    gpu, power = gpu_info()
    r = {"workload": name, "dim": d, "params": params, "source_rows": [int(s.get_count()) for s in srcs],
         "target_rows": [int(h[1].size) for h in host_rows], "timed_host_rebuild_equal": True,
         "rebuild_from_range_s": round(float(np.median(t_dev)), 3), "host_rebuild_s": round(float(np.median(t_host)), 3),
         "host_over_rebuild_from_range": round(float(np.median(t_host) / np.median(t_dev)), 2), "reps": reps,
         "rebuild_from_range_all_s": [round(t, 3) for t in t_dev], "host_rebuild_all_s": [round(t, 3) for t in t_host],
         "gpu": gpu, "power_limit": power}
    print(json.dumps(r), flush=True)
    if out:
        with open(out, "a") as f:
            f.write(json.dumps(r) + "\n")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", choices=["split_170k", "split_1m", "merge_2x500k", "hnsw_split_1m", "all"], default="all")
    ap.add_argument("--scale", type=float, default=1.0, help="multiply every row count (a quick run at a smaller size)")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None, help="append each result line to this file")
    a = ap.parse_args()
    rng = np.random.default_rng(0)
    ivf = {"nlist": 1024}
    n = lambda rows: max(1000, int(rows * a.scale))  # noqa: E731
    for rows, name in ((170_000, "split_170k"), (1_000_000, "split_1m")):
        if a.workload in (name, "all"):
            m = n(rows)
            src = region(b200vs.IVF_FLAT, m, 768, ivf, 0, rng)
            run(name, b200vs.IVF_FLAT, 768, ivf, [src], [(0, m // 2), (m // 2, I64_MAX)], a.reps, a.out, rng)
            del src
    if a.workload in ("merge_2x500k", "all"):
        m = n(500_000)
        own, sib = region(b200vs.IVF_FLAT, m, 768, ivf, 0, rng), region(b200vs.IVF_FLAT, m, 768, ivf, m, rng)
        run("merge_2x500k", b200vs.IVF_FLAT, 768, ivf, [own, sib], [(0, I64_MAX)], a.reps, a.out, rng)
        del own, sib
    if a.workload in ("hnsw_split_1m", "all"):
        m = n(1_000_000)
        hp = {"hnsw_m": 32, "hnsw_efc": 64, "max_elements": m}
        src = region(b200vs.HNSW, m, 128, hp, 0, rng)
        run("hnsw_split_1m", b200vs.HNSW, 128, hp, [src], [(0, m // 2), (m // 2, I64_MAX)], a.reps, a.out, rng)


if __name__ == "__main__":
    main()
