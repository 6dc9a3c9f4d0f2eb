"""torchrun worker of the sharded range-search test (tests/test_gpu_shard_range.py::test_two_ranks_match_oracle, also
runnable by hand: `python -m torch.distributed.run --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29523
tests/shard_worker_range.py`).  Skips (exit 0, "SHARD_WORKER_RANGE SKIP") when fewer than 2 GPUs are visible.

Every rank builds its part of ONE logical IVF-Flat index through b200vs_shard_* (rank 0's trained state broadcast, rows
routed to their list owner over NCCL); the same batches go through the sharded range search (host pointers, device
pointers on two streams, filters, interleaved with top-k batches) with every list probed, and rank 0 checks every answer
against the expectation restated on the gathered rows (test_gpu_exact_edges.range_expect, whose FP32 values the oracle's
top-k pins bit for bit): ids, distance bits and counts."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "dingo-store_b200", "python"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402

import b200vs  # noqa: E402
import oracle_lib  # noqa: E402
from test_gpu_exact_edges import prep, radius_for, range_expect, raw_fp32  # noqa: E402


def main():
    if torch.cuda.device_count() < 2:
        print("SHARD_WORKER_RANGE SKIP: needs 2 GPUs", flush=True)
        return
    import faulthandler
    faulthandler.dump_traceback_later(240, exit=True)  # a hung collective must not hold the GPUs
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    dist.init_process_group("nccl", device_id=dev)
    o = oracle_lib.load()
    failures = []
    for metric, d, n_per, nq, mr in ((b200vs.L2, 64, 20000, 120, 256), (b200vs.IP, 36, 8000, 40, 1024), (b200vs.COSINE, 32, 8000, 64, 64)):
        nlist = 8 * world
        rng = np.random.default_rng(3000 + rank)
        xb = rng.standard_normal((n_per, d)).astype(np.float32)
        ids = np.arange(1, n_per + 1, dtype=np.int64) + rank * n_per
        ix = b200vs.Index(b200vs.IVF_FLAT, metric, d, nlist=nlist, device=local)
        idb = torch.from_numpy(b200vs.Shard.unique_id() if rank == 0 else np.zeros(128, np.uint8)).to(dev)
        dist.broadcast(idb, 0)
        sh = b200vs.Shard(ix, rank, world, idb.cpu().numpy(), lanes=2)
        if rank == 0:
            ix.train(np.random.default_rng(7).standard_normal((nlist * 64, d)).astype(np.float32))
        sh.broadcast_state(0)
        sh.add(xb, ids)
        off, X, _, lids = ix.export_lists(nlist)
        parts = [None] * world
        dist.all_gather_object(parts, (X, lids))
        gX = np.concatenate([p[0] for p in parts], 0)
        gI = np.concatenate([p[1] for p in parts], 0)
        xq = np.random.default_rng(79).standard_normal((nq, d)).astype(np.float32)
        Q = prep(o, metric, xq)
        radius = radius_for(raw_fp32(gX, Q[0], metric), metric, 200)
        seq = iter(range(100))
        R1 = sh.range_search(xq, radius, mr, seq=next(seq), nprobe=nlist)
        sh.search(xq, 10, seq=next(seq), nprobe=nlist)
        qd = torch.from_numpy(xq).to(dev)
        outs = [(torch.empty((nq, mr), dtype=torch.float32, device=dev), torch.empty((nq, mr), dtype=torch.int64, device=dev),
                 torch.empty((nq,), dtype=torch.int32, device=dev)) for _ in range(2)]
        sts = [torch.cuda.Stream(device=dev) for _ in range(2)]
        sp, _keep = b200vs.make_search_params(nprobe=nlist)
        torch.cuda.synchronize()
        for i in range(2):
            sh.range_search_device(nq, qd.data_ptr(), radius, mr, outs[i][0].data_ptr(), outs[i][1].data_ptr(), outs[i][2].data_ptr(),
                                   stream=sts[i].cuda_stream, sp=sp, seq=next(seq))
        torch.cuda.synchronize()
        sel = np.arange(3, world * n_per, 4, dtype=np.int64)
        R2 = sh.range_search(xq, radius, mr, seq=next(seq), nprobe=nlist, sorted_ids=sel, negate=True)
        if rank == 0:
            def same(R, what, cand=None):
                D, I, C = R
                for qi in range(nq):
                    wi, wd, _ = range_expect(gX, gI, Q[qi], metric, radius, mr, cand)
                    if not (C[qi] == len(wi) and np.array_equal(I[qi, :C[qi]], wi) and np.array_equal(D[qi, :C[qi]].view(np.uint32), wd.view(np.uint32))):
                        failures.append(f"metric {metric} {what}: query {qi} differs from the expectation")
                        return
            same(R1, "host call")
            for i in range(2):
                same(tuple(t.cpu().numpy() for t in outs[i]), f"device call {i}")
            same(R2, "negated id-list call", cand=~np.isin(gI, sel))
        sh.close()
        ix.close()
        dist.barrier()
        faulthandler.cancel_dump_traceback_later()
        faulthandler.dump_traceback_later(240, exit=True)
    ok = torch.tensor([0 if failures else 1], device=dev)
    dist.broadcast(ok, 0)
    if rank == 0:
        print("SHARD_WORKER_RANGE", "OK" if not failures else "FAILED: " + "; ".join(failures), flush=True)
    dist.destroy_process_group()
    sys.exit(0 if int(ok.item()) == 1 else 1)


if __name__ == "__main__":
    main()
