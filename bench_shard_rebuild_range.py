"""Split and merge rebuilds of a sharded set on the GPU (b200vs_shard_rebuild_from_range) against the host-fed rebuild a
front end runs without it: export every source rank's lists to the host, keep the rows in the id range, compute each rank's
rows_r (the rows whose row_owner is r, ascending id) in numpy, then shard_train + shard_add of rows_r on a fresh set.  Both
are checked equal (trained state, lists, search results) before anything is timed.

Workloads:
  ivf    IVF-Flat L2, 768-d, nlist 1024, world 1: the split child [mid, end) and the split parent [0, mid) of a 1 M-row set,
         and the merge of two 500 k-row sets.
  hnsw   HNSW L2, 200 k x 128, m 32, efconstruction 64, world 1: the split child of the set (the host-fed rebuild is the
         export, the range filter and b200vs_hnsw_add_batched of the sorted rows).
  loop   IVF-Flat L2, 200 k x 128, nlist 96, the split child at worlds 2 and 3 as threads of one process on ONE GPU over the
         loopback NCCL (tests/nccl_loopback, built by build()).  Every rank shares the one GPU and the loopback library copies
         through the host, so these are one-GPU figures of the flow, not multi-GPU timings.

Host times start from the indexes on the device and include the export.  Prints one JSON line per job with the GPU name and
power limit, the median and every run (and appends it to --out when given).
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
from bench_shard_rebuild import connect, gather, gpu_info  # noqa: E402

LOOPBACK_LIB = os.path.join(ROOT, "tests", "nccl_loopback", "libnccl_loopback.so")


def rank_body(W, kind, sets, d, params, jobs, reps):
    """fn(r, world) of one rank: builds the source sets (sets: row counts; ids are one permutation cut into disjoint ranges),
    then for each job (name, source set indexes, id_min, id_max) checks the two rebuilds equal and times them alternately."""
    nlist = params.get("nlist", 1)

    def body(r, world):
        rng = np.random.default_rng(0)
        n = sum(sets)
        x = rng.standard_normal((n, d)).astype(np.float32)
        ids = rng.permutation(n).astype(np.int64)
        srcs = []
        at = 0
        for m in sets:  # set k holds the ids [at, at + m): the disjoint ranges of a region split or merge
            sel = np.nonzero((ids >= at) & (ids < at + m))[0]
            part = sel[r * sel.size // W:(r + 1) * sel.size // W]
            ix = b200vs.Index(kind, b200vs.L2, d, **params)
            sh = connect(world, ix, r)
            if kind == b200vs.HNSW:
                sh.hnsw_add_batched(x[part], ids[part])
            else:
                sh.train(x[part][: 256 * nlist // W])
                for a in range(0, part.size, 262144):
                    sh.add(x[part[a:a + 262144]], ids[part[a:a + 262144]])
            srcs.append((ix, sh))
            at += m
        q = rng.standard_normal((64, d)).astype(np.float32)
        results = []
        for name, which, lo, hi in jobs:
            use = [srcs[k] for k in which]

            def device():
                ix = b200vs.Index(kind, b200vs.L2, d, **params)
                sh = connect(world, ix, r)
                sh.rebuild_from_range([s for _, s in use], lo, hi)
                return ix, sh

            def host():
                if kind == b200vs.HNSW:  # one source: the rank's own rows in the range; nothing moves between ranks
                    s_ix = use[0][0]
                    hid = s_ix.export_lists(1, with_vectors=False)[3]
                    hid = np.sort(hid[(hid >= lo) & (hid < hi)])
                    hx, _ = s_ix.reconstruct(hid)
                    ix = b200vs.Index(kind, b200vs.L2, d, **params)
                    sh = connect(world, ix, r)
                    ix.add_batched(hx, hid)
                    return ix, sh
                parts = []
                for s_ix, _ in use:
                    _, ex, _, eid = s_ix.export_lists(nlist)
                    keep = (eid >= lo) & (eid < hi)
                    parts.append((ex[keep], eid[keep]))
                parts = [p for rank_parts in gather(world, r, parts) for p in rank_parts]
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
            assert all(gather(world, r, same)), f"{name}: the device rebuild and the host-fed rebuild differ"
            rows = sum(gather(world, r, int(a.get_count())))
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
            results.append((name, rows, t_dev, t_host))
        for _, s in srcs:
            s.close()
        return results

    return body


def report(workload, W, d, params, res, out, note=None):
    gpu, power = gpu_info()
    for name, rows, t_dev, t_host in res:
        r = {"workload": workload, "job": name, "world": W, "rows_rebuilt": rows, "dim": d, "params": params,
             "host_fed_rebuild_equal": True, "shard_rebuild_from_range_s": round(float(np.median(t_dev)), 3),
             "host_fed_s": round(float(np.median(t_host)), 3),
             "host_fed_over_rebuild_from_range": round(float(np.median(t_host) / np.median(t_dev)), 2), "reps": len(t_dev),
             "shard_rebuild_from_range_all_s": [round(t, 3) for t in t_dev], "host_fed_all_s": [round(t, 3) for t in t_host],
             "gpu": gpu, "power_limit": power}
        if note:
            r["note"] = note
        print(json.dumps(r), flush=True)
        if out:
            with open(out, "a") as f:
                f.write(json.dumps(r) + "\n")


def run_loopback(W, n, d, nlist, reps, out):
    """One world of the loopback run, in this process (started by main() with the loopback library selected)."""
    from shard_loopback import run_world
    jobs = [("split_child", [0], n // 2, 2 ** 63 - 1)]
    res = run_world(W, rank_body(W, b200vs.IVF_FLAT, [n], d, {"nlist": nlist}, jobs, reps))
    merged = [(name, rows, list(np.max([r[i][2] for r in res], axis=0)), list(np.max([r[i][3] for r in res], axis=0)))
              for i, (name, rows, _, _) in enumerate(res[0])]  # a collective ends when its slowest rank does
    report(f"ivf_flat_l2_{d}_nlist{nlist}_loopback", W, d, {"nlist": nlist}, merged, out,
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
        n, p = a.ivf_rows, {"nlist": 1024}
        split = rank_body(1, b200vs.IVF_FLAT, [n], 768, p, [("split_child", [0], n // 2, 2 ** 63 - 1),
                                                           ("split_parent", [0], 0, n // 2)], a.reps)(0, None)
        merge = rank_body(1, b200vs.IVF_FLAT, [n // 2, n - n // 2], 768, p, [("merge", [0, 1], 0, 2 ** 63 - 1)], a.reps)(0, None)
        report("ivf_flat_l2_768_nlist1024", 1, 768, p, split + merge, a.out)
    if a.workload in ("hnsw", "all"):
        n, p = a.hnsw_rows, {"hnsw_m": 32, "hnsw_efc": 64, "max_elements": a.hnsw_rows}
        res = rank_body(1, b200vs.HNSW, [n], 128, p, [("split_child", [0], n // 2, 2 ** 63 - 1)], a.reps)(0, None)
        report("hnsw_l2_128_m32", 1, 128, p, res, a.out)
    if a.workload in ("loop", "all"):
        env = dict(os.environ, B200VS_NCCL_LIB=LOOPBACK_LIB)  # the library is chosen once per process
        for W in (2, 3):
            cmd = [sys.executable, os.path.abspath(__file__), "--loopback-world", str(W), "--loop-rows", str(a.loop_rows),
                   "--reps", str(a.reps)] + (["--out", a.out] if a.out else [])
            subprocess.check_call(cmd, env=env, cwd=ROOT)


if __name__ == "__main__":
    main()
