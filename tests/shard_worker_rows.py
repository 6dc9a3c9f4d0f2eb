"""torchrun worker of the row-sharded test (tests/test_gpu_shard_rows.py::test_two_ranks_match_a_plain_index, also runnable by
hand: `python -m torch.distributed.run --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29527
tests/shard_worker_rows.py`).  Skips (exit 0, "SHARD_WORKER_ROWS SKIP") when fewer than 2 GPUs are visible.

Every rank contributes different rows to ONE logical FLAT or HNSW index through b200vs_shard_add (rows routed to
row_owner(id) over NCCL).  Rank 0 checks:
  * FLAT (L2 / IP / cosine): the sharded search and range search equal, bit for bit, a plain index of all rows added in
    the same arrival order.  The IP case holds a pair of rows with distinct inner products and equal 1 - ip, whose ids are
    placed on different ranks: only a merge on the raw key keeps the single index's order.
  * HNSW (L2 / cosine): the sharded search equals the merge of b200vs_search on standalone graphs, each built by the same
    single-index call from the rows row_owner assigns to its rank, in arrival order."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "dingo-store_b200", "python"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402

import b200vs  # noqa: E402
from b200vs import shard as shard_py  # noqa: E402


def _same(a, b):
    return all(np.array_equal(x.view(np.uint32), y.view(np.uint32)) if x.dtype == np.float32 else np.array_equal(x, y)
               for x, y in zip(a, b))


def _pair_ids(world):
    """Two ids owned by different ranks."""
    cand = np.arange(1, 1000, dtype=np.int64) + 10 ** 7
    own = shard_py.row_owner(cand, world)
    return cand[own == 0][0], cand[own == 1][0]


def main():
    if torch.cuda.device_count() < 2:
        print("SHARD_WORKER_ROWS SKIP: needs 2 GPUs", flush=True)
        return
    import faulthandler
    faulthandler.dump_traceback_later(240, exit=True)  # a hung collective must not hold the GPUs
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    dist.init_process_group("nccl", device_id=dev)
    failures = []

    def connect(ix):
        idb = torch.from_numpy(b200vs.Shard.unique_id() if rank == 0 else np.zeros(128, np.uint8)).to(dev)
        dist.broadcast(idb, 0)
        return b200vs.Shard(ix, rank, world, idb.cpu().numpy(), lanes=2)

    def rank_rows(r, n_per, d, seed):
        x = np.random.default_rng(seed + r).standard_normal((n_per, d)).astype(np.float32)
        ids = np.random.default_rng(seed + 100 + r).choice(10 ** 6, n_per, replace=False).astype(np.int64) + r * 10 ** 6
        return x, ids

    for metric, d, n_per in ((b200vs.L2, 64, 12000), (b200vs.IP, 32, 6000), (b200vs.COSINE, 48, 6000)):
        rows = [rank_rows(r, n_per, d, 500) for r in range(world)]
        if metric == b200vs.IP:  # ip 2e-9 (id a, rank 0) and 1e-9 (id b, rank 1): both 1 - ip round to 1
            a, b = _pair_ids(world)
            for r, (rid, v) in enumerate(((a, 2e-9), (b, 1e-9))):
                x, ids = rows[r]
                x[0] = 0
                x[0, 0] = np.float32(v)
                ids[0] = rid
            for r in range(world):
                rows[r][0][1:, 0] = -1.0  # every other row scores ip < 0 against e0
        ix = b200vs.Index(b200vs.FLAT, metric, d, device=local)
        sh = connect(ix)
        sh.add(*rows[rank])
        # the plain index of all rows, in arrival order at each owner: rank 0's rows first, then rank 1's
        plain = b200vs.Index(b200vs.FLAT, metric, d, device=local)
        plain.add(np.concatenate([r[0] for r in rows]), np.concatenate([r[1] for r in rows]))
        xq = np.random.default_rng(77).standard_normal((100, d)).astype(np.float32)
        if metric == b200vs.IP:
            xq[:] = 0
            xq[:, 0] = 1
        for nq, k in ((100, 10), (100, 300), (4, 10)):
            if not _same(sh.search(xq[:nq], k), plain.search(xq[:nq], k)):
                failures.append(f"FLAT metric {metric} nq {nq} k {k}: search differs")
        if metric == b200vs.IP:
            D, I = sh.search(xq[:20], 2)
            if not (I[:, 0] == a).all() or not (I[:, 1] == b).all():
                failures.append("FLAT IP: the raw-key pair is not in the single index's order")
        else:
            Dp, _ = plain.search(xq[:1], 200)
            radius = float(Dp[0, -1])  # L2: the distance itself; cosine: 1 - ip, which the range rule compares alike
            if not _same(sh.range_search(xq, radius, 512), plain.range_search(xq, radius, 512)):
                failures.append(f"FLAT metric {metric}: range search differs")
        sh.delete(np.concatenate([r[1][::4] for r in rows]))
        plain.delete(np.concatenate([r[1][::4] for r in rows]))
        if not _same(sh.search(xq, 10), plain.search(xq, 10)):
            failures.append(f"FLAT metric {metric}: search after delete differs")
        sh.close()
        dist.barrier()

    for metric, d, n_per in ((b200vs.L2, 32, 3000), (b200vs.COSINE, 32, 3000)):
        rows = [rank_rows(r, n_per, d, 900) for r in range(world)]
        allx, alli = np.concatenate([r[0] for r in rows]), np.concatenate([r[1] for r in rows])
        own = b200vs.row_owner(alli, world)
        for batched in (False, True):
            g = b200vs.Index(b200vs.HNSW, metric, d, hnsw_m=16, hnsw_efc=100, max_elements=2 * n_per * world, device=local)
            sh = connect(g)
            if batched:
                sh.hnsw_add_batched(*rows[rank], 64)
            else:
                sh.add(*rows[rank])
            xq = np.random.default_rng(78).standard_normal((50, d)).astype(np.float32)
            got = sh.search(xq, 10, efsearch=64)
            parts = []
            for r in range(world):  # standalone graphs of every rank's rows, in arrival order
                p = b200vs.Index(b200vs.HNSW, metric, d, hnsw_m=16, hnsw_efc=100, max_elements=2 * n_per * world, device=local)
                if batched:
                    p.add_batched(allx[own == r], alli[own == r], 64)
                else:
                    p.add(allx[own == r], alli[own == r])
                if r == rank and not np.array_equal(p.get_trained_state(), g.get_trained_state()):
                    failures.append(f"HNSW metric {metric} batched {batched}: rank {rank}'s graph differs")
                parts.append(p.search(xq, 10, efsearch=64))
            want = shard_py.merge_topk(np.stack([p[0] for p in parts]), np.stack([p[1] for p in parts]), 10)
            if not _same(got, want):
                failures.append(f"HNSW metric {metric} batched {batched}: search differs from the merge of standalone graphs")
            sh.close()
            dist.barrier()
    allf = [None] * world
    dist.all_gather_object(allf, failures)
    failures = [f for fs in allf for f in fs]
    if rank == 0:
        print("SHARD_WORKER_ROWS", "OK" if not failures else "FAILED: " + "; ".join(failures), flush=True)
    faulthandler.cancel_dump_traceback_later()
    dist.destroy_process_group()
    sys.exit(0 if not failures else 1)


if __name__ == "__main__":
    main()
