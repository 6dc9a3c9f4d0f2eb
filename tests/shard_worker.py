"""torchrun worker of the list-sharded parity test (tests/test_gpu_shard.py::test_two_ranks_match_oracle, also runnable by
hand: `python -m torch.distributed.run --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29511 tests/shard_worker.py`).

Every rank builds its part of ONE logical IVF-Flat index through b200vs_shard_* (distributed training or a broadcast
trained state, rows routed to their list owner over NCCL), answers the same batches through the sharded search (device
pointers, host pointers, several batches in flight, explicit sequence numbers from concurrent threads) and rank 0 checks
every answer against the CPU oracle run on the gathered index: ids and distance bits must be identical.  Before building,
every rank checks that a train with too few rows on one rank and a broadcast from an untrained root are refused on every
rank with the same status."""
import os
import sys
import threading

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "dingo-store_b200", "python"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402

import b200vs  # noqa: E402
import oracle_lib  # noqa: E402


def note(rank, *a):
    if rank == 0:
        print("[shard_worker]", *a, file=sys.stderr, flush=True)


def main():
    import faulthandler
    faulthandler.dump_traceback_later(150, exit=True)  # a hung collective must not hold the GPUs
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    dist.init_process_group("nccl", device_id=dev)
    o = oracle_lib.load()
    failures = []
    for metric, om, d, nlist, n_per, nq, k, nprobe, mode in (
            (b200vs.L2, oracle_lib.L2, 128, 32 * world, 20000, 200, 10, 8, "broadcast"),
            (b200vs.COSINE, oracle_lib.COSINE, 64, 16 * world, 6000, 37, 5, 6, "broadcast"),
            (b200vs.IP, oracle_lib.IP, 96, 16 * world, 8000, 64, 10, 16, "train")):
        rng = np.random.default_rng(1000 + rank)
        xb = rng.random((n_per, d)).astype(np.float32)
        ids = np.arange(1, n_per + 1, dtype=np.int64) + rank * n_per
        ix = b200vs.Index(b200vs.IVF_FLAT, metric, d, nlist=nlist, device=local)
        idb = torch.from_numpy(b200vs.Shard.unique_id() if rank == 0 else np.zeros(128, np.uint8)).to(dev)
        dist.broadcast(idb, 0)
        sh = b200vs.Shard(ix, rank, world, idb.cpu().numpy(), lanes=2)
        # refusals every rank returns together, before any rank waits in a collective: the last rank trains on fewer than
        # nlist / world rows, and a broadcast from an untrained root
        for what, fn, want in (("short train", lambda: sh.train(xb[:nlist // world - 1] if rank == world - 1 else xb),
                                b200vs.EILLEGAL_PARAMETERS),
                               ("untrained root", lambda: sh.broadcast_state(0), b200vs.EVECTOR_NOT_TRAIN)):
            try:
                fn()
                got = b200vs.OK
            except b200vs.B200VSError as e:
                got = e.code
            if got != want or ix.is_trained():
                failures.append(f"metric {metric} {what}: rank {rank} returned {got}, want {want}")
        note(rank, "collective refusals done")
        if mode == "train":
            sh.train(xb)
        else:  # rank 0 holds an oracle-trained state, everybody receives it
            if rank == 0:
                xn = o.normalize_faiss(xb) if metric == b200vs.COSINE else xb
                cent = o.kmeans(om, xn, nlist, nthreads=8)
                ix.set_trained_state(b200vs.ivf_state_blob(cent, metric))
            sh.broadcast_state(0)
        # rows: half through host pointers, half through device pointers, uneven chunk sizes per rank
        h = n_per // 2 + 13 * rank
        sh.add(xb[:h], ids[:h])
        xd, idd = torch.from_numpy(xb[h:]).to(dev), torch.from_numpy(ids[h:]).to(dev)
        torch.cuda.synchronize()
        sh.add_device(n_per - h, xd.data_ptr(), idd.data_ptr())
        b, e = sh.list_range()
        off, lx, _, lids = ix.export_lists(nlist)
        lens = np.diff(off)
        assert lens[:b].sum() == 0 and lens[e:].sum() == 0, "a rank holds rows of lists it does not own"
        # gather the whole logical index on rank 0 for the oracle (list-major, rank order inside a list is irrelevant)
        parts = [None] * world
        dist.all_gather_object(parts, (off, lx, lids))
        cent = ix.get_trained_state()[32:].view(np.float32).reshape(nlist, d)
        xq = np.random.default_rng(77).random((nq, d)).astype(np.float32)
        note(rank, "built", metric, mode)
        # 1) host-pointer call
        D1, I1 = sh.search(xq, k, nprobe=nprobe)
        # 2) device-pointer calls, two batches in flight on two streams
        qd = torch.from_numpy(xq).to(dev)
        outs = [(torch.empty((nq, k), dtype=torch.float32, device=dev), torch.empty((nq, k), dtype=torch.int64, device=dev)) for _ in range(4)]
        sts = [torch.cuda.Stream(device=dev) for _ in range(2)]
        sp, _keep = b200vs.make_search_params(nprobe=nprobe)
        torch.cuda.synchronize()
        for i in range(4):
            sh.search_device(nq, qd.data_ptr(), k, outs[i][0].data_ptr(), outs[i][1].data_ptr(), stream=sts[i % 2].cuda_stream, sp=sp)
        torch.cuda.synchronize()
        note(rank, "device calls done")
        # 3) concurrent caller threads with explicit sequence numbers (1 + 4 searches so far -> next is 5)
        res = {}

        def call(sq):
            res[sq] = sh.search(xq, k, seq=sq, nprobe=nprobe)
        ths = [threading.Thread(target=call, args=(5 + t,)) for t in (1, 0, 3, 2)]
        for t in ths:
            t.start()
        for t in ths:
            t.join()
        note(rank, "threaded calls done")
        # 4) filters travel with the call
        D4, I4 = sh.search(xq, k, seq=9, nprobe=nprobe, id_range=(5, n_per + 7))
        # 5) collective delete: the same ids on every rank, rows dropped wherever they live; unknown ids -> EVECTOR_INVALID
        dead = np.concatenate([np.arange(1, 1 + n_per, 7, dtype=np.int64) + r * n_per for r in range(world)])
        removed = sh.delete(dead)
        D5, I5 = sh.search(xq, k, seq=10, nprobe=nprobe)
        try:
            sh.delete(np.array([-12345], dtype=np.int64))
            not_found_ok = False
        except b200vs.B200VSError as e:
            not_found_ok = e.code == b200vs.EVECTOR_INVALID
        if rank == 0:
            g_off = np.zeros(nlist + 1, np.int64)
            gx, gi = [], []
            for l in range(nlist):
                for (po, px, pi) in parts:
                    gx.append(px[po[l]:po[l + 1]])
                    gi.append(pi[po[l]:po[l + 1]])
                g_off[l + 1] = g_off[l] + sum(int(po[l + 1] - po[l]) for (po, _, _) in parts)
            gx, gi = np.concatenate(gx, 0), np.concatenate(gi, 0)
            assert gx.shape[0] == n_per * world
            qn = o.normalize_faiss(xq) if metric == b200vs.COSINE else xq
            Do, Io = o.ivfflat_search(om, cent, g_off, gx, gi, qn, k, nprobe, nthreads=16)
            Df, If = o.ivfflat_search(om, cent, g_off, gx, gi, qn, k, nprobe, nthreads=16, id_range=(5, n_per + 7))

            def same(D, I, Dw, Iw, what):
                if not (np.array_equal(I, Iw) and np.array_equal(D.view(np.uint32), Dw.view(np.uint32))):
                    failures.append(f"metric {metric} {what}: sharded result differs from the oracle")
            same(D1, I1, Do, Io, "host call")
            for i in range(4):
                same(outs[i][0].cpu().numpy(), outs[i][1].cpu().numpy(), Do, Io, f"device call {i}")
            for sq, (D, I) in res.items():
                same(D, I, Do, Io, f"threaded call seq {sq}")
            same(D4, I4, Df, If, "filtered call")
            if removed != dead.size or not not_found_ok:
                failures.append(f"metric {metric}: collective delete removed {removed} of {dead.size}, not-found status ok = {not_found_ok}")
            keep = ~np.isin(gi, dead)
            k_off = np.zeros(nlist + 1, np.int64)
            k_off[1:] = np.cumsum([int(keep[g_off[l]:g_off[l + 1]].sum()) for l in range(nlist)])
            Dd, Id = o.ivfflat_search(om, cent, k_off, gx[keep], gi[keep], qn, k, nprobe, nthreads=16)
            same(D5, I5, Dd, Id, "search after the collective delete")
        sh.close()
        ix.close()
        dist.barrier()
        faulthandler.cancel_dump_traceback_later()
        faulthandler.dump_traceback_later(150, exit=True)
    if rank != 0 and failures:
        print(f"[shard_worker] rank {rank} FAILED:", "; ".join(failures), file=sys.stderr, flush=True)
    ok = torch.tensor([0 if failures else 1], device=dev)
    dist.all_reduce(ok, op=dist.ReduceOp.MIN)  # a failure seen on any rank fails the worker
    if rank == 0:
        print("SHARD_WORKER", "OK" if int(ok.item()) == 1 else "FAILED: " + "; ".join(failures or ["on another rank"]), flush=True)
    dist.destroy_process_group()
    sys.exit(0 if int(ok.item()) == 1 else 1)


if __name__ == "__main__":
    main()
