"""Deep top-k (b200vs_search_deep) timing on a Flat 1M x 768 L2 index and on the headline IVF-Flat index (1M x 768 L2,
nlist 1024, nprobe 32), at nq in {1, 10, 100} and k in {4096, 40960}.

Each line reports the time per call of b200vs_search_deep, of b200vs_search at k = 4096 on the same index and queries, and
of the CPU oracle (--oracle-threads threads, default 16) at the same shape, and checks the deep call's ids and distance bits
against the oracle.  The card name and power limit are read in the same run.  Times are host clocks around synchronous
host-pointer calls (the results are on the host when a call returns), the median of --reps calls after one warm-up call.
The IVF-Flat centroids are rows drawn from the data (a fixed trained state, so the oracle searches the same lists).
Writes nothing to the tree; the JSON lines go to stdout."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(ROOT, "dingo-store_b200", "python"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import b200vs  # noqa: E402
import oracle_lib  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=60).stdout.strip().splitlines()
        name, power = [s.strip() for s in out[0].split(",")]
        return {"name": name, "power_limit": power}
    except Exception as e:  # noqa: BLE001 - reported, not hidden
        return {"error": str(e)}


def timed(fn, reps):
    fn()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        r = fn()
        ts.append(time.perf_counter() - t0)
    return float(np.median(ts)) * 1e3, r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--nb", type=int, default=1_000_000)
    ap.add_argument("--dim", type=int, default=768)
    ap.add_argument("--nlist", type=int, default=1024)
    ap.add_argument("--nprobe", type=int, default=32)
    ap.add_argument("--nq", type=int, nargs="+", default=[1, 10, 100])
    ap.add_argument("--k", type=int, nargs="+", default=[4096, 40960])
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--oracle-threads", type=int, default=16)
    ap.add_argument("--types", nargs="+", default=["FLAT", "IVF_FLAT"])
    a = ap.parse_args()

    import torch
    assert torch.cuda.is_available(), "bench_deep_topk.py measures the GPU path and needs cuda:0"
    print(json.dumps({"card": card()}), flush=True)
    o = oracle_lib.load()
    rng = np.random.default_rng(0)
    xb = rng.standard_normal((a.nb, a.dim), dtype=np.float32)
    ids = np.arange(a.nb, dtype=np.int64)
    xq_all = rng.standard_normal((max(a.nq), a.dim), dtype=np.float32)
    for t in a.types:
        if t == "FLAT":
            ix = b200vs.Index(b200vs.FLAT, b200vs.L2, a.dim)
            ix.add(xb, ids)
            kw = {}
            oracle = lambda xq, k: o.flat_search(oracle_lib.L2, xb, ids, xq, k, nthreads=a.oracle_threads)  # noqa: E731
        else:
            cent = xb[np.random.default_rng(1).choice(a.nb, a.nlist, replace=False)].copy()
            ix = b200vs.Index(b200vs.IVF_FLAT, b200vs.L2, a.dim, nlist=a.nlist)
            ix.set_trained_state(b200vs.ivf_state_blob(cent, b200vs.L2))
            ix.add(xb, ids)
            off, lx, _, lids = ix.export_lists(a.nlist)
            kw = {"nprobe": a.nprobe}
            oracle = lambda xq, k: o.ivfflat_search(oracle_lib.L2, cent, off, lx, lids, xq, k, a.nprobe,  # noqa: E731
                                                    nthreads=a.oracle_threads)
        for nq in a.nq:
            xq = xq_all[:nq]
            base_ms, _ = timed(lambda: ix.search(xq, 4096, **kw), a.reps)
            for k in a.k:
                deep_ms, (D, I) = timed(lambda: ix.search_deep(xq, k, **kw), a.reps)
                t0 = time.perf_counter()
                Do, Io = oracle(xq, k)
                cpu_ms = (time.perf_counter() - t0) * 1e3
                same = bool(np.array_equal(I, Io) and np.array_equal(D.view(np.uint32), Do.view(np.uint32)))
                print(json.dumps({"index": t, "nb": a.nb, "dim": a.dim, "nprobe": kw.get("nprobe"), "nq": nq, "k": k,
                                  "deep_ms_per_call": round(deep_ms, 3), "search_k4096_ms_per_call": round(base_ms, 3),
                                  "cpu_oracle_ms": round(cpu_ms, 1), "cpu_oracle_threads": a.oracle_threads,
                                  "equal_to_oracle": same}), flush=True)
                assert same, f"{t} nq={nq} k={k}: deep results differ from the oracle"
        del ix


if __name__ == "__main__":
    main()
