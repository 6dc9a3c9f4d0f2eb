"""Snapshot restore of a list-sharded IVF-Flat index against rebuilding it.

Builds a list-sharded IVF-Flat index (shard_train + shard_add, the rebuild a node without snapshots has to run), saves it with
b200vs_shard_save and restores it with b200vs_shard_load into fresh empty indexes, and prints one JSON line: save and load
GB/s over the snapshot's bytes, restore time against rebuild time, and optionally a restore onto another number of ranks.
Every time is a host clock around collective calls that end in a device synchronise; the median of --reps runs is kept.
The snapshot goes to a temporary directory (removed at the end); the loads read files that were just written, so they come
from the page cache and measure the restore path, not the disk.  Worlds above 1 run as threads of one process on one GPU
through the loopback NCCL of the test suite (tests/nccl_loopback), so their collectives are host rendezvous, not NVLink."""
import argparse
import json
import os
import shutil
import statistics
import subprocess
import sys
import tempfile
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
LOOPBACK = os.path.join(ROOT, "tests", "nccl_loopback", "libnccl_loopback.so")


class _Ids:
    """communicator ids: the c-th shard every rank creates shares one"""

    def __init__(self):
        self.lock, self.ids, self.calls = threading.Lock(), {}, {}

    def shard(self, ix, r, W):
        import b200vs
        with self.lock:
            c = self.calls.get(r, 0)
            self.calls[r] = c + 1
            if c not in self.ids:
                self.ids[c] = b200vs.Shard.unique_id()
            uid = self.ids[c]
        return b200vs.Shard(ix, r, W, uid)


def _world(W, fn):
    """fn(rank, barrier, ids) on W threads; returns every rank's result."""
    barrier = threading.Barrier(W)
    ids = _Ids()
    res, err = [None] * W, [None] * W

    def body(r):
        try:
            res[r] = fn(r, barrier, ids)
        except BaseException as e:  # noqa: B036 - re-raised below
            err[r] = e
            barrier.abort()

    ths = [threading.Thread(target=body, args=(r,), daemon=True) for r in range(W)]
    for t in ths:
        t.start()
    for t in ths:
        t.join()
    for e in err:
        if e is not None and not isinstance(e, threading.BrokenBarrierError):
            raise e
    return res


def run(args):
    import torch
    import b200vs
    from b200vs import IVF_FLAT, L2
    assert torch.cuda.is_available(), "bench_shard_restore needs a GPU"
    W, d, n, nlist = args.world, args.dim, args.rows, args.nlist
    rng = np.random.default_rng(0)
    per = n // W
    xs = [rng.standard_normal((per, d)).astype(np.float32) for _ in range(W)]
    ids = [np.arange(per, dtype=np.int64) + r * per for r in range(W)]
    xq = rng.standard_normal((64, d)).astype(np.float32)
    tmp = tempfile.mkdtemp(prefix="b2vs_restore_")
    prefix = os.path.join(tmp, "snap")
    out = {"world": W, "rows": per * W, "dim": d, "nlist": nlist, "device": torch.cuda.get_device_name(0)}

    def timed(barrier, f):
        barrier.wait()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        f()
        torch.cuda.synchronize()
        barrier.wait()
        return time.perf_counter() - t0

    def rank(r, barrier, conn):
        res = {"build": [], "save": [], "load": []}
        for rep in range(args.reps):
            ix = b200vs.Index(IVF_FLAT, L2, d, nlist=nlist)
            sh = conn.shard(ix, r, W)
            res["build"].append(timed(barrier, lambda: (sh.train(xs[r][: max(nlist // W * 64, nlist)]), sh.add(xs[r], ids[r]))))
            if rep == 0:
                res["want"] = sh.search(xq, 10, nprobe=16)
            res["save"].append(timed(barrier, lambda: sh.save(prefix)))
            sh.close(); ix.close()
            ix = b200vs.Index(IVF_FLAT, L2, d, nlist=nlist)
            sh = conn.shard(ix, r, W)
            res["load"].append(timed(barrier, lambda: sh.load(prefix)))
            if rep == 0:
                res["got"] = sh.search(xq, 10, nprobe=16)
            sh.close(); ix.close()
        return res

    try:
        res = _world(W, rank)
        snap = sum(os.path.getsize(os.path.join(tmp, f)) for f in os.listdir(tmp))
        med = {k: statistics.median(max(r[k][i] for r in res) for i in range(args.reps)) for k in ("build", "save", "load")}
        same = all(np.array_equal(r["got"][1], res[0]["want"][1]) for r in res)
        out.update(snapshot_bytes=snap, rebuild_s=med["build"], save_s=med["save"], load_s=med["load"],
                   save_GBps=snap / med["save"] / 1e9, load_GBps=snap / med["load"] / 1e9,
                   restore_speedup=med["build"] / med["load"], results_equal=bool(same))
        if args.world_to:
            W2 = args.world_to
            times = []
            for _ in range(args.reps):
                def rank2(r, barrier, conn):
                    ix = b200vs.Index(IVF_FLAT, L2, d, nlist=nlist)
                    sh = conn.shard(ix, r, W2)
                    t = timed(barrier, lambda: sh.load(prefix))
                    got = sh.search(xq, 10, nprobe=16)
                    sh.close(); ix.close()
                    return t, got
                rr = _world(W2, rank2)
                times.append(max(t for t, _ in rr))
            out.update(world_to=W2, load_to_s=statistics.median(times),
                       load_to_equal=bool(all(np.array_equal(g[1], res[0]["want"][1]) for _, g in rr)))
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    print(json.dumps(out))


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--world", type=int, default=1, help="ranks of the saved index (above 1: loopback threads on one GPU)")
    ap.add_argument("--world-to", type=int, default=0, help="also restore onto this many ranks")
    ap.add_argument("--rows", type=int, default=2_000_000)
    ap.add_argument("--dim", type=int, default=128)
    ap.add_argument("--nlist", type=int, default=1024)
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    if max(args.world, args.world_to) > 1 and os.environ.get("B200VS_NCCL_LIB") != LOOPBACK:
        # the loopback NCCL is chosen once per process: start again with it
        assert os.path.exists(LOOPBACK), f"{LOOPBACK} not built (build() runs make -C tests/nccl_loopback)"
        sys.exit(subprocess.call([sys.executable] + sys.argv, env=dict(os.environ, B200VS_NCCL_LIB=LOOPBACK)))
    sys.path.insert(0, os.path.join(ROOT, "dingo-store_b200", "python"))
    run(args)


if __name__ == "__main__":
    main()
