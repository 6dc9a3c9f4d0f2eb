"""Rebuild of an index from an old index's rows on the GPU (b200vs_rebuild_from) against the host rebuild a
VectorIndexManager runs today, whose rows come from the host.

Workloads:
  ivf   IVF-Flat L2, 1 M x 768, nlist 1024.  Host rebuild: b200vs_train, then b200vs_add_with_ids in 32768-row calls.
  hnsw  HNSW L2, 1 M x 128, m 32, efconstruction 64, with half the nodes tombstoned.  Host rebuild: one
        b200vs_hnsw_add_batched call over the sorted host rows, which builds the same graph as rebuild_from; rebuild_from
        adds no device work here (the live nodes are read from the host graph), so this measures what the host hand-over
        costs.  The plugin's bulk Add in 32768-row calls is timed beside it for reference; it builds another graph (each
        call batches on its own), so it is not checked for equality.

The timed host rebuild is checked equal to rebuild_from's index (trained state, lists or graph, and search results) before
timing.  Host times start from rows already in host memory: the RocksDB scan in front of them is not included.  Prints one
JSON line per workload with the GPU name and power limit (and appends it to --out when given).
"""
import argparse
import json
import subprocess
import sys
import time
import os

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "dingo-store_b200", "python"))
import b200vs  # noqa: E402


def gpu_info():
    try:
        out = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], text=True)
        name, power = [s.strip() for s in out.splitlines()[0].split(",")]
        return name, power
    except Exception as e:  # the numbers are still printed, marked with what is known
        return f"unknown ({e})", "unknown"


def host_rebuild(kind, x, ids, params, metric, chunked):
    ix = b200vs.Index(kind, metric, x.shape[1], **params)
    if kind != b200vs.HNSW:
        ix.train(x)
    step = 32768 if chunked else ids.size
    for a in range(0, ids.size, step):
        if kind == b200vs.HNSW:
            ix.add_batched(x[a:a + step], ids[a:a + step])
        else:
            ix.add(x[a:a + step], ids[a:a + step])
    return ix


def live_sorted(src, kind, nlist):
    if kind == b200vs.HNSW:
        _, _, _, ids = src.export_lists(1, with_vectors=False)
        ids = np.sort(ids)
        x, found = src.reconstruct(ids)
        assert found.all()
        return x, ids
    _, x, _, ids = src.export_lists(nlist)
    o = np.argsort(ids, kind="stable")
    return x[o], ids[o]


def check_equal(a, b, kind, nlist, q):
    assert np.array_equal(a.get_trained_state(), b.get_trained_state()), "trained state / graph differs"
    if kind != b200vs.HNSW:
        for u, v in zip(a.export_lists(nlist), b.export_lists(nlist)):
            assert (u is None and v is None) or np.array_equal(u, v), "lists differ"
    Da, Ia = a.search(q, 10, nprobe=16)
    Db, Ib = b.search(q, 10, nprobe=16)
    assert np.array_equal(Ia, Ib) and np.array_equal(Da.view(np.uint32), Db.view(np.uint32)), "search results differ"


def run(name, kind, n, d, params, tombstone_half, reps, out):
    rng = np.random.default_rng(0)
    x = rng.standard_normal((n, d)).astype(np.float32)
    ids = rng.permutation(n).astype(np.int64)  # ids given out of order
    src = b200vs.Index(kind, b200vs.L2, d, **params)
    if kind == b200vs.HNSW:
        src.add_batched(x, ids)
    else:
        src.train(x[:256 * params["nlist"]])
        for a in range(0, n, 262144):
            src.add(x[a:a + 262144], ids[a:a + 262144])
    if tombstone_half:
        src.delete(ids[::2])
    nlist = params.get("nlist", 1)
    xs, sids = live_sorted(src, kind, nlist)
    q = rng.standard_normal((64, d)).astype(np.float32)

    # equality: rebuild_from == the timed host rebuild (a train + add of the live rows in ascending id order)
    chunked = kind != b200vs.HNSW
    dst = b200vs.Index(kind, b200vs.L2, d, **params)
    dst.rebuild_from(src)
    check_equal(dst, host_rebuild(kind, xs, sids, params, b200vs.L2, chunked), kind, nlist, q)
    del dst

    t_dev, t_host, t_plugin = [], [], []
    for _ in range(reps):  # alternate them so drift on the shared machine hits each
        dst = b200vs.Index(kind, b200vs.L2, d, **params)
        t0 = time.perf_counter()
        dst.rebuild_from(src)  # returns when the index is complete
        t_dev.append(time.perf_counter() - t0)
        del dst
        t0 = time.perf_counter()
        h = host_rebuild(kind, xs, sids, params, b200vs.L2, chunked)
        t_host.append(time.perf_counter() - t0)
        del h
        if kind == b200vs.HNSW:
            t0 = time.perf_counter()
            h = host_rebuild(kind, xs, sids, params, b200vs.L2, True)
            t_plugin.append(time.perf_counter() - t0)
            del h
    gpu, power = gpu_info()
    r = {"workload": name, "rows_live": int(sids.size), "dim": d, "params": params, "timed_host_rebuild_equal": True,
         "rebuild_from_s": round(float(np.median(t_dev)), 3), "host_rebuild_s": round(float(np.median(t_host)), 3),
         "host_over_rebuild_from": round(float(np.median(t_host) / np.median(t_dev)), 2), "reps": reps,
         "rebuild_from_all_s": [round(t, 3) for t in t_dev], "host_rebuild_all_s": [round(t, 3) for t in t_host],
         "gpu": gpu, "power_limit": power}
    if t_plugin:
        r["plugin_bulk_add_32768_s"] = round(float(np.median(t_plugin)), 3)
    print(json.dumps(r), flush=True)
    if out:
        with open(out, "a") as f:
            f.write(json.dumps(r) + "\n")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", choices=["ivf", "hnsw", "all"], default="all")
    ap.add_argument("--ivf-rows", type=int, default=1_000_000)
    ap.add_argument("--hnsw-rows", type=int, default=1_000_000)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None, help="append each result line to this file")
    a = ap.parse_args()
    if a.workload in ("ivf", "all"):
        run("ivf_flat_l2_768_nlist1024", b200vs.IVF_FLAT, a.ivf_rows, 768, {"nlist": 1024}, False, a.reps, a.out)
    if a.workload in ("hnsw", "all"):
        run("hnsw_l2_128_m32_half_tombstoned", b200vs.HNSW, a.hnsw_rows, 128,
            {"hnsw_m": 32, "hnsw_efc": 64, "max_elements": a.hnsw_rows}, True, a.reps, a.out)


if __name__ == "__main__":
    main()
