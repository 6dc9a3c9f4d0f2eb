"""The cost of the sharded read flow on a Binary IVF-Flat index: b200vs_search_binary_device against
b200vs_shard_search_binary_device at world 1 on the same index.

Builds one Binary IVF-Flat index of --n packed rows (--dim bits) from a seeded clustered generator (each row is one of
--nlist random centres with about 1 / 8 of its bits flipped), installs the generator's centres as the trained state (the
benchmark measures the read, not k-means), and times batches of --batch queries, top --k at --nprobe, through the plain
device-pointer search and through a world-1 shard of the same index (the shard flow: query slice, coarse pass, pack of the
per-rank top-k and the merge kernel; no NCCL call at world 1).  The two are alternated in one process after warm-up, each
timed with CUDA events over --steps batches, --reps times; the medians are reported with the device name and power
limit, and the outputs of both must be bit-identical.  Under torchrun with several GPUs (WORLD_SIZE > 1) every rank holds
--n / W rows routed through b200vs_shard_add_binary and the W-GPU shard throughput is reported too.  Prints one JSON line."""
import argparse
import json
import os
import statistics
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(ROOT, "dingo-store_b200", "python"))


def clustered(rng, n, nb, centres):
    """n packed rows of nb bytes: a random centre each, every bit flipped with probability 1 / 8"""
    c = rng.integers(0, len(centres), n)
    noise = rng.integers(0, 256, (n, nb), dtype=np.uint8) & rng.integers(0, 256, (n, nb), dtype=np.uint8)
    noise &= rng.integers(0, 256, (n, nb), dtype=np.uint8)
    return centres[c] ^ noise


def device_info(dev):
    import torch
    name = torch.cuda.get_device_name(dev)
    try:
        out = subprocess.run(["nvidia-smi", "-i", str(dev), "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.TimeoutExpired):
        out = "unknown"
    return name, out


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--n", type=int, default=20_000_000, help="rows of the whole index")
    ap.add_argument("--dim", type=int, default=1024, help="bits per row")
    ap.add_argument("--nlist", type=int, default=4096)
    ap.add_argument("--nprobe", type=int, default=64)
    ap.add_argument("--batch", type=int, default=1024)
    ap.add_argument("--k", type=int, default=10)
    ap.add_argument("--steps", type=int, default=20, help="batches per timed window")
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--reps", type=int, default=5, help="alternated timed windows of each path")
    args = ap.parse_args()

    import torch
    import b200vs

    W = int(os.environ.get("WORLD_SIZE", "1"))
    r = int(os.environ.get("RANK", "0"))
    dev = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(dev)
    if W > 1:
        import torch.distributed as dist
        dist.init_process_group("gloo")
    nb = args.dim // 8
    rng = np.random.default_rng(1234)
    centres = rng.integers(0, 256, (args.nlist, nb), dtype=np.uint8)
    blob = b200vs.binary_ivf_state_blob(centres)
    qrng = np.random.default_rng(99)
    xq = clustered(qrng, args.batch, nb, centres)

    ix = b200vs.Index(b200vs.BINARY_IVF_FLAT, b200vs.HAMMING, args.dim, nlist=args.nlist, device=dev)
    ix.set_trained_state(blob)
    uid = None
    if W > 1:
        uid = torch.from_numpy(b200vs.Shard.unique_id() if r == 0 else np.zeros(128, np.uint8))
        dist.broadcast(uid, 0)
        uid = uid.numpy()
    sh = b200vs.BinaryShard(ix, r, W, uid)
    chunk = 1_000_000
    mine = args.n // W
    drng = np.random.default_rng(7 + r)
    for a in range(0, mine, chunk):  # each rank adds its own rows; W = 1: the plain index's rows
        m = min(chunk, mine - a)
        ids = np.arange(a, a + m, dtype=np.int64) * W + r
        if W == 1:
            ix.add(clustered(drng, m, nb, centres), ids)
        else:
            sh.add(clustered(drng, m, nb, centres), ids)
    if W > 1:  # every rank runs the same number of collective adds
        dist.barrier()

    qd = torch.from_numpy(xq).cuda(dev)
    out = {p: (torch.empty((args.batch, args.k), dtype=torch.float32, device=dev),
               torch.empty((args.batch, args.k), dtype=torch.int64, device=dev)) for p in ("plain", "shard")}
    sp, _keep = b200vs.make_search_params(nprobe=args.nprobe)
    stream = torch.cuda.Stream(device=dev)
    seq = [0]

    def run(path, steps):
        d, i = out[path]
        for _ in range(steps):
            if path == "plain":
                ix.search_device(args.batch, qd.data_ptr(), args.k, d.data_ptr(), i.data_ptr(), stream=stream.cuda_stream, sp=sp)
            else:
                sh.search_device(args.batch, qd.data_ptr(), args.k, d.data_ptr(), i.data_ptr(), stream=stream.cuda_stream, sp=sp, seq=seq[0])
                seq[0] += 1

    def timed(path):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize(dev)
        e0.record(stream)
        run(path, args.steps)
        e1.record(stream)
        e1.synchronize()
        return e0.elapsed_time(e1) / args.steps

    paths = ("plain", "shard") if W == 1 else ("shard",)
    for p in paths:
        run(p, args.warmup)
    ms = {p: [] for p in paths}
    for _ in range(args.reps):
        for p in paths:
            ms[p].append(timed(p))
    torch.cuda.synchronize(dev)
    name, power = device_info(dev)
    res = {"bench": "shard_binary", "device": name, "power_limit_and_max_sm_clock": power, "world": W, "n": args.n, "dim": args.dim,
           "nlist": args.nlist, "nprobe": args.nprobe, "batch": args.batch, "k": args.k}
    for p in paths:
        med = statistics.median(ms[p])
        res[f"{p}_ms_per_batch"] = round(med, 4)
        res[f"{p}_qps"] = round(args.batch * 1000.0 / med, 1)
    if W == 1:
        res["shard_overhead_ms"] = round(res["shard_ms_per_batch"] - res["plain_ms_per_batch"], 4)
        dp, ip_ = (t.cpu().numpy() for t in out["plain"])
        ds, is_ = (t.cpu().numpy() for t in out["shard"])
        res["bit_identical"] = bool(np.array_equal(ip_, is_) and np.array_equal(dp.view(np.uint32), ds.view(np.uint32)))
        if not res["bit_identical"]:
            print(json.dumps(res))
            raise SystemExit("the shard flow's results differ from the plain index's")
    sh.close()
    if r == 0:
        print(json.dumps(res))
    if W > 1:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
