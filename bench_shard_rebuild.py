"""Rebuild of a sharded set on the GPU (b200vs_shard_rebuild_from) against the host-fed rebuild a front end runs without it:
export every rank's lists to the host, compute each rank's rows_r (the live rows whose row_owner is r, ascending id), then
shard_train + shard_add of rows_r on a fresh set.  Both are checked equal (trained state, lists, search results) before timing.

Workloads:
  ivf    IVF-Flat L2, 1 M x 768, nlist 1024, world 1 on one GPU.
  hnsw   HNSW L2, 200 k x 128, m 32, efconstruction 64, half the nodes tombstoned, world 1 (each rank rebuilds its own graph:
         the host-fed rebuild is the export + b200vs_hnsw_add_batched of the sorted live rows).
  loop   IVF-Flat L2, 200 k x 128, nlist 96, worlds 2 and 3 as threads of one process on ONE GPU over the loopback NCCL
         (tests/nccl_loopback, built by build()).  Every rank shares the one GPU and the loopback library copies through the
         host, so these are one-GPU figures of the flow, not multi-GPU timings; a multi-GPU run needs a multi-GPU machine.

Host times start from the indexes on the device and include the export.  Prints one JSON line per workload with the GPU
name and power limit (and appends it to --out when given).
"""
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
from b200vs.shard import row_owner  # noqa: E402

LOOPBACK_LIB = os.path.join(ROOT, "tests", "nccl_loopback", "libnccl_loopback.so")


def gpu_info():
    try:
        out = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], text=True)
        name, power = [s.strip() for s in out.splitlines()[0].split(",")]
        return name, power
    except Exception as e:  # the numbers are still printed, marked with what is known
        return f"unknown ({e})", "unknown"


def connect(world, ix, r):
    if world is None:
        return b200vs.Shard(ix, 0, 1, None)
    idb = world.gather(r, b200vs.Shard.unique_id() if r == 0 else None)[0]
    return b200vs.Shard(ix, r, world.W, idb)


def gather(world, r, v):
    return [v] if world is None else world.gather(r, v)


def rank_body(W, kind, n, d, params, reps):
    """fn(r, world) of one rank: builds src, checks the two rebuilds equal, then times them alternately."""
    nlist = params.get("nlist", 1)

    def body(r, world):
        rng = np.random.default_rng(0)
        x = rng.standard_normal((n, d)).astype(np.float32)
        ids = rng.permutation(n).astype(np.int64)
        part = slice(r * n // W, (r + 1) * n // W)
        src_ix = b200vs.Index(kind, b200vs.L2, d, **params)
        src = connect(world, src_ix, r)
        if kind == b200vs.HNSW:
            src.hnsw_add_batched(x[part], ids[part])
            src.delete(ids[::2])
        else:
            src.train(x[part][: 256 * nlist // W])
            for a in range(part.start, part.stop, 262144):
                src.add(x[a:min(a + 262144, part.stop)], ids[a:min(a + 262144, part.stop)])
        q = rng.standard_normal((64, d)).astype(np.float32)

        def device():
            ix = b200vs.Index(kind, b200vs.L2, d, **params)
            sh = connect(world, ix, r)
            sh.rebuild_from(src)
            return ix, sh

        def host():
            if kind == b200vs.HNSW:  # the rank's own live rows; nothing moves between ranks
                _, _, _, hid = src_ix.export_lists(1, with_vectors=False)
                hid = np.sort(hid)
                hx, found = src_ix.reconstruct(hid)
                ix = b200vs.Index(kind, b200vs.L2, d, **params)
                sh = connect(world, ix, r)
                ix.add_batched(hx, hid)
                return ix, sh
            _, ex, _, eid = src_ix.export_lists(nlist)
            parts = gather(world, r, (ex, eid))
            ai = np.concatenate([p[1] for p in parts])
            o = np.argsort(ai, kind="stable")
            o = o[row_owner(ai[o], W) == r]
            ax = np.concatenate([p[0] for p in parts])[o]
            ix = b200vs.Index(kind, b200vs.L2, d, **params)
            sh = connect(world, ix, r)
            sh.train(ax)
            sh.add(ax, ai[o])
            return ix, sh

        (a, sa), (b, sb) = device(), host()
        same = np.array_equal(a.get_trained_state(), b.get_trained_state())
        if kind != b200vs.HNSW:
            same = same and all(np.array_equal(u, v) for u, v in zip(a.export_lists(nlist), b.export_lists(nlist)))
            Da, Ia = sa.search(q, 10, nprobe=16)
            Db, Ib = sb.search(q, 10, nprobe=16)
        else:
            Da, Ia = a.search(q, 10)
            Db, Ib = b.search(q, 10)
        same = same and np.array_equal(Ia, Ib) and np.array_equal(Da.view(np.uint32), Db.view(np.uint32))
        assert all(gather(world, r, same)), "the device rebuild and the host-fed rebuild differ"
        rows = sum(gather(world, r, int(src_ix.get_count())))
        for s in (sa, sb):
            s.close()
        t_dev, t_host = [], []
        for _ in range(reps):  # alternated, so drift on the shared machine hits both
            gather(world, r, None)
            t0 = time.perf_counter()
            ix, sh = device()
            gather(world, r, None)
            t_dev.append(time.perf_counter() - t0)
            sh.close()
            del ix
            t0 = time.perf_counter()
            ix, sh = host()
            gather(world, r, None)
            t_host.append(time.perf_counter() - t0)
            sh.close()
            del ix
        src.close()
        return rows, t_dev, t_host

    return body


def report(name, W, rows, d, params, t_dev, t_host, out, note=None):
    gpu, power = gpu_info()
    r = {"workload": name, "world": W, "rows_live": rows, "dim": d, "params": params, "host_fed_rebuild_equal": True,
         "shard_rebuild_from_s": round(float(np.median(t_dev)), 3), "host_fed_s": round(float(np.median(t_host)), 3),
         "host_fed_over_rebuild_from": round(float(np.median(t_host) / np.median(t_dev)), 2), "reps": len(t_dev),
         "shard_rebuild_from_all_s": [round(t, 3) for t in t_dev], "host_fed_all_s": [round(t, 3) for t in t_host],
         "gpu": gpu, "power_limit": power}
    if note:
        r["note"] = note
    print(json.dumps(r), flush=True)
    if out:
        with open(out, "a") as f:
            f.write(json.dumps(r) + "\n")


def run_world1(name, kind, n, d, params, reps, out):
    rows, t_dev, t_host = rank_body(1, kind, n, d, params, reps)(0, None)
    report(name, 1, rows, d, params, t_dev, t_host, out)


def run_loopback(W, n, d, nlist, reps, out):
    """One world of the loopback run, in this process (started by main() with the loopback library selected)."""
    from shard_loopback import run_world
    res = run_world(W, rank_body(W, b200vs.IVF_FLAT, n, d, {"nlist": nlist}, reps))
    t_dev = np.max([r[1] for r in res], axis=0)  # a collective ends when its slowest rank does
    t_host = np.max([r[2] for r in res], axis=0)
    report(f"ivf_flat_l2_{d}_nlist{nlist}_loopback", W, res[0][0], d, {"nlist": nlist}, list(t_dev), list(t_host), out,
           note="ranks are threads on one GPU over the loopback NCCL: a one-GPU figure, not a multi-GPU timing")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", choices=["ivf", "hnsw", "loop", "all"], default="all")
    ap.add_argument("--ivf-rows", type=int, default=1_000_000)
    ap.add_argument("--hnsw-rows", type=int, default=200_000)
    ap.add_argument("--loop-rows", type=int, default=200_000)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None, help="append each result line to this file")
    ap.add_argument("--loopback-world", type=int, default=0, help=argparse.SUPPRESS)  # the child of the loopback run
    a = ap.parse_args()
    if a.loopback_world:
        run_loopback(a.loopback_world, a.loop_rows, 128, 96, a.reps, a.out)
        return
    if a.workload in ("ivf", "all"):
        run_world1("ivf_flat_l2_768_nlist1024", b200vs.IVF_FLAT, a.ivf_rows, 768, {"nlist": 1024}, a.reps, a.out)
    if a.workload in ("hnsw", "all"):
        run_world1("hnsw_l2_128_m32_half_tombstoned", b200vs.HNSW, a.hnsw_rows, 128,
                   {"hnsw_m": 32, "hnsw_efc": 64, "max_elements": a.hnsw_rows}, a.reps, a.out)
    if a.workload in ("loop", "all"):
        env = dict(os.environ, B200VS_NCCL_LIB=LOOPBACK_LIB)  # the library is chosen once per process
        for W in (2, 3):
            cmd = [sys.executable, os.path.abspath(__file__), "--loopback-world", str(W), "--loop-rows", str(a.loop_rows),
                   "--reps", str(a.reps)] + (["--out", a.out] if a.out else [])
            subprocess.check_call(cmd, env=env, cwd=ROOT)


if __name__ == "__main__":
    main()
