"""Sharded deep top-k (b200vs_shard_search_deep) on the headline IVF-Flat index (1M x 768 L2, nlist 1024, nprobe 32), at nq in
{1, 10, 100} and k in {4096, 40960}.

World 1: each line reports the time per call of b200vs_shard_search_deep on a world-one shard of the index and of
b200vs_search_deep on the plain index holding the same rows with the same trained state, and checks that the two agree bit
for bit (ids and distances).  Times are host clocks around synchronous host-pointer calls, the median of --reps calls after
one warm-up call.

--loopback W [W ...]: the same index split over W ranks that run as threads of this process on ONE GPU, their collectives
through the loopback NCCL stand-in of tests/nccl_loopback (built by build()).  Each line reports rank 0's profiled pack +
merge phase (b200vs_last_phase_times slot [11], device ms; the all-gather is slot [10]) and checks rank 0's results against
the plain index.  These are one-GPU loopback figures: the ranks share one GPU's SMs and HBM, so they say what the merge
costs, not what a multi-GPU search costs.

The card name and power limit are read in the same run.  Writes nothing to the tree; the JSON lines go to stdout."""
import argparse
import json
import os
import subprocess
import sys
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(ROOT, "dingo-store_b200", "python"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
LOOPBACK_LIB = os.path.join(ROOT, "tests", "nccl_loopback", "libnccl_loopback.so")

import b200vs  # noqa: E402


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


def same(a, b):
    return bool(np.array_equal(a[1], b[1]) and np.array_equal(a[0].view(np.uint32), b[0].view(np.uint32)))


def loopback(W, a, blob, xb, ids, xq_all, want):
    """The index split over W rank threads on one GPU: rank 0's profiled merge phase for every (nq, k)."""
    from shard_loopback import run_world
    cuts = np.linspace(0, a.nb, W + 1).astype(np.int64)

    def rank(r, world):
        ix = b200vs.Index(b200vs.IVF_FLAT, b200vs.L2, a.dim, nlist=a.nlist)
        ix.set_trained_state(blob)
        idb = world.gather(r, b200vs.Shard.unique_id() if r == 0 else None)[0]
        sh = b200vs.Shard(ix, r, W, idb)
        sh.add(xb[cuts[r]:cuts[r + 1]], ids[cuts[r]:cuts[r + 1]])
        ix.set_profiling(True)
        out = {}
        for nq in a.nq:
            for k in a.k:
                xq = xq_all[:nq]
                sh.search_deep(xq, k, nprobe=a.nprobe)  # warm-up
                merge, comm = [], []
                for _ in range(a.reps):
                    world.barrier.wait()
                    res = sh.search_deep(xq, k, nprobe=a.nprobe)
                    ph = ix.phase_times()
                    merge.append(ph["merge"])
                    comm.append(ph["comm"])
                out[(nq, k)] = (float(np.median(merge)), float(np.median(comm)), res)
        ix.set_profiling(False)
        sh.close()
        return out

    o = run_world(W, rank)[0]
    for (nq, k), (merge_ms, comm_ms, res) in o.items():
        eq = same(res, want[(nq, k)])
        print(json.dumps({"loopback_one_gpu_world": W, "nq": nq, "k": k, "merge_phase_ms_rank0": round(merge_ms, 3),
                          "allgather_phase_ms_rank0": round(comm_ms, 3), "equal_to_search_deep": eq}), flush=True)
        assert eq, f"loopback W={W} nq={nq} k={k}: results differ from the plain index"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--nb", type=int, default=1_000_000)
    ap.add_argument("--dim", type=int, default=768)
    ap.add_argument("--nlist", type=int, default=1024)
    ap.add_argument("--nprobe", type=int, default=32)
    ap.add_argument("--nq", type=int, nargs="+", default=[1, 10, 100])
    ap.add_argument("--k", type=int, nargs="+", default=[4096, 40960])
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--loopback", type=int, nargs="*", default=[])
    a = ap.parse_args()

    import torch
    assert torch.cuda.is_available(), "bench_shard_deep.py measures the GPU path and needs cuda:0"
    if a.loopback:
        assert os.path.exists(LOOPBACK_LIB), f"{LOOPBACK_LIB} not built (build() makes it)"
        os.environ["B200VS_NCCL_LIB"] = LOOPBACK_LIB  # read by the library's first NCCL call, which comes after this
    print(json.dumps({"card": card()}), flush=True)
    rng = np.random.default_rng(0)
    xb = rng.standard_normal((a.nb, a.dim), dtype=np.float32)
    ids = np.arange(a.nb, dtype=np.int64)
    xq_all = rng.standard_normal((max(a.nq), a.dim), dtype=np.float32)
    cent = xb[np.random.default_rng(1).choice(a.nb, a.nlist, replace=False)].copy()
    blob = b200vs.ivf_state_blob(cent, b200vs.L2)
    plain = b200vs.Index(b200vs.IVF_FLAT, b200vs.L2, a.dim, nlist=a.nlist)
    plain.set_trained_state(blob)
    plain.add(xb, ids)
    ix = b200vs.Index(b200vs.IVF_FLAT, b200vs.L2, a.dim, nlist=a.nlist)
    ix.set_trained_state(blob)
    sh = b200vs.Shard(ix, 0, 1, None)
    sh.add(xb, ids)
    want = {}
    for nq in a.nq:
        xq = xq_all[:nq]
        for k in a.k:
            plain_ms, want[(nq, k)] = timed(lambda: plain.search_deep(xq, k, nprobe=a.nprobe), a.reps)
            shard_ms, got = timed(lambda: sh.search_deep(xq, k, nprobe=a.nprobe), a.reps)
            eq = same(got, want[(nq, k)])
            print(json.dumps({"index": "IVF_FLAT", "nb": a.nb, "dim": a.dim, "nlist": a.nlist, "nprobe": a.nprobe, "world": 1, "nq": nq,
                              "k": k, "shard_search_deep_ms_per_call": round(shard_ms, 3),
                              "search_deep_ms_per_call": round(plain_ms, 3), "equal_to_search_deep": eq}), flush=True)
            assert eq, f"nq={nq} k={k}: shard_search_deep differs from search_deep"
    sh.close()
    del sh, ix
    for W in a.loopback:
        loopback(W, a, blob, xb, ids, xq_all, want)
    print(json.dumps({"multi_gpu": "not measured"}), flush=True)


if __name__ == "__main__":
    main()
