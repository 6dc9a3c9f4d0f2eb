"""torchrun worker of the list-sharded IVF-PQ parity test (tests/test_gpu_shard_pq.py::test_two_ranks_match_oracle, also
runnable by hand: `python -m torch.distributed.run --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29513
tests/shard_worker_pq.py`).  Skips (exit 0, "SHARD_WORKER_PQ SKIP") when fewer than 2 GPUs are visible.

Every rank builds its part of ONE logical IVF-PQ index through b200vs_shard_* (distributed training, or rank 0's
b200vs_train state broadcast), rows routed to their list owner over NCCL; the same batches go through the sharded search
(host pointers, device pointers on two streams, concurrent threads with explicit sequence numbers, filters, a collective
delete) and rank 0 checks every answer against the CPU oracle run on the gathered exports: ids and distance bits."""
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
import pq_codes  # noqa: E402


def main():
    if torch.cuda.device_count() < 2:
        print("SHARD_WORKER_PQ SKIP: needs 2 GPUs", flush=True)
        return
    import faulthandler
    faulthandler.dump_traceback_later(240, exit=True)  # a hung collective must not hold the GPUs
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    dist.init_process_group("nccl", device_id=dev)
    o = oracle_lib.load()
    failures = []
    for metric, d, M, nbits, nlist, n_train, n_per, nq, k, nprobe, mode in (
            (b200vs.L2, 64, 16, 8, 16 * world, 70000, 20000, 120, 10, 8, "train"),
            (b200vs.COSINE, 48, 12, 4, 8 * world, 6000, 8000, 37, 5, 6, "train"),
            (b200vs.IP, 32, 8, 8, 8 * world, 70000, 6000, 64, 10, 5, "broadcast")):
        rng = np.random.default_rng(2000 + rank)
        xt = rng.standard_normal((n_train, d)).astype(np.float32)
        xb = rng.standard_normal((n_per, d)).astype(np.float32)
        ids = np.arange(1, n_per + 1, dtype=np.int64) + rank * n_per
        ix = b200vs.Index(b200vs.IVF_PQ, metric, d, nlist=nlist, pq_m=M, pq_nbits=nbits, device=local)
        idb = torch.from_numpy(b200vs.Shard.unique_id() if rank == 0 else np.zeros(128, np.uint8)).to(dev)
        dist.broadcast(idb, 0)
        sh = b200vs.Shard(ix, rank, world, idb.cpu().numpy(), lanes=2)
        if mode == "train":
            sh.train(xt)
        else:
            if rank == 0:
                ix.train(xt)
            sh.broadcast_state(0)
        h = n_per // 2 + 11 * rank
        sh.add(xb[:h], ids[:h])
        xd, idd = torch.from_numpy(xb[h:]).to(dev), torch.from_numpy(ids[h:]).to(dev)
        torch.cuda.synchronize()
        sh.add_device(n_per - h, xd.data_ptr(), idd.data_ptr())
        b, e = sh.list_range()
        cs = pq_codes.code_size(M, nbits)
        off, _, codes, lids = ix.export_lists(nlist, with_vectors=False, code_size=cs)
        lens = np.diff(off)
        assert lens[:b].sum() == 0 and lens[e:].sum() == 0, "a rank holds rows of lists it does not own"
        parts = [None] * world
        dist.all_gather_object(parts, (off, codes, lids))
        st = ix.get_trained_state()
        f = st[48:].view(np.float32)
        cent = f[:nlist * d].reshape(nlist, d)
        cb = f[nlist * d:].reshape(M, 1 << nbits, d // M)
        xq = np.random.default_rng(78).standard_normal((nq, d)).astype(np.float32)
        D1, I1 = sh.search(xq, k, nprobe=nprobe)
        qd = torch.from_numpy(xq).to(dev)
        outs = [(torch.empty((nq, k), dtype=torch.float32, device=dev), torch.empty((nq, k), dtype=torch.int64, device=dev)) for _ in range(4)]
        sts = [torch.cuda.Stream(device=dev) for _ in range(2)]
        sp, _keep = b200vs.make_search_params(nprobe=nprobe)
        torch.cuda.synchronize()
        for i in range(4):
            sh.search_device(nq, qd.data_ptr(), k, outs[i][0].data_ptr(), outs[i][1].data_ptr(), stream=sts[i % 2].cuda_stream, sp=sp)
        torch.cuda.synchronize()
        res = {}

        def call(sq):
            res[sq] = sh.search(xq, k, seq=sq, nprobe=nprobe)
        ths = [threading.Thread(target=call, args=(5 + t,)) for t in (1, 0, 3, 2)]
        for t in ths:
            t.start()
        for t in ths:
            t.join()
        D4, I4 = sh.search(xq, k, seq=9, nprobe=nprobe, id_range=(5, n_per + 7))
        sel = np.arange(3, world * n_per, 4, dtype=np.int64)
        D6, I6 = sh.search(xq, k, seq=10, nprobe=nprobe, sorted_ids=sel, negate=True)
        dead = np.concatenate([np.arange(1, 1 + n_per, 7, dtype=np.int64) + r * n_per for r in range(world)])
        removed = sh.delete(dead)
        D5, I5 = sh.search(xq, k, seq=11, nprobe=nprobe)
        if rank == 0:
            g_off = np.zeros(nlist + 1, np.int64)
            gc, gi = [], []
            for l in range(nlist):
                for (po, pc, pi) in parts:
                    gc.append(pc[po[l]:po[l + 1]])
                    gi.append(pi[po[l]:po[l + 1]])
                g_off[l + 1] = g_off[l] + sum(int(po[l + 1] - po[l]) for (po, _, _) in parts)
            gc, gi = np.concatenate(gc, 0), np.concatenate(gi, 0)
            assert gc.shape[0] == n_per * world

            def oracle(off_, codes_, ids_, **filt):
                return pq_codes.ivfpq_search(o, metric, cent, cb, off_, codes_, ids_, xq, k, nprobe, nthreads=16, **filt)

            def same(D, I, Dw, Iw, what):
                if not (np.array_equal(I, Iw) and np.array_equal(D.view(np.uint32), Dw.view(np.uint32))):
                    failures.append(f"metric {metric} nbits {nbits} {what}: sharded result differs from the oracle")
            Do, Io = oracle(g_off, gc, gi)
            same(D1, I1, Do, Io, "host call")
            for i in range(4):
                same(outs[i][0].cpu().numpy(), outs[i][1].cpu().numpy(), Do, Io, f"device call {i}")
            for sq, (Dt, It) in res.items():
                same(Dt, It, Do, Io, f"threaded call seq {sq}")
            same(D4, I4, *oracle(g_off, gc, gi, id_range=(5, n_per + 7)), "id-range call")
            same(D6, I6, *oracle(g_off, gc, gi, sorted_ids=sel, negate=True), "negated id-list call")
            if removed != dead.size:
                failures.append(f"metric {metric}: collective delete removed {removed} of {dead.size}")
            keep = ~np.isin(gi, dead)
            k_off = np.zeros(nlist + 1, np.int64)
            k_off[1:] = np.cumsum([int(keep[g_off[l]:g_off[l + 1]].sum()) for l in range(nlist)])
            same(D5, I5, *oracle(k_off, gc[keep], gi[keep]), "search after the collective delete")
        sh.close()
        ix.close()
        dist.barrier()
        faulthandler.cancel_dump_traceback_later()
        faulthandler.dump_traceback_later(240, exit=True)
    ok = torch.tensor([0 if failures else 1], device=dev)
    dist.broadcast(ok, 0)
    if rank == 0:
        print("SHARD_WORKER_PQ", "OK" if not failures else "FAILED: " + "; ".join(failures), flush=True)
    dist.destroy_process_group()
    sys.exit(0 if int(ok.item()) == 1 else 1)


if __name__ == "__main__":
    main()
