#!/usr/bin/env python
"""bench_configs.py — the OTHER BASELINE.json configs (bench.py measures the headline one), one JSON line each.

  cfg1  Flat L2, 100K x 128, top-10, batch = 1            (the reference's own CPU-runnable case)
  cfg2  IVF-Flat L2, 1M x 768, nlist 1024, nprobe 32, batch 256, top-10
  cfg3  IVF-PQ IP, 10M x 768, M = 96, nbits 8, nlist 2048, nprobe 64, batch 1024, top-100   (--pq-n, --pq-nbits, --pq-m)
  cfg3s cfg3 through the list-sharded deployment b200vs_shard_* (world 1 on one GPU, beside the plain search at the same
        shape; under torchrun over the box's GPUs, n / world rows per GPU)                    (--pq-n, --pq-nbits, --pq-m)
  cfg4  HNSW cosine, 1M x 768, M = 16, efConstruction 200, efSearch 128, batch 512          (--hnsw-n; concurrent host build)
  1s    Flat L2, 2M x 768, batch 1024, top-10, through the row-sharded deployment b200vs_shard_* at world 1, beside the plain
        search on the same index (ids and distance bits compared)
  4s    cfg4's HNSW cosine (1M x 768, M = 16, efSearch 128, batch 512) through the row-sharded deployment at world 1, graph built
        by b200vs_shard_hnsw_add_batched, beside the plain search on the same index                           (--hnsw-n)
  cfg5  IVF-Flat L2, (rows-per-GPU x world) x 1536, nlist 2048 per GPU, nprobe 64, batch 4096, top-10, list-sharded over
        the GPUs of the box through b200vs_shard_* — run under torchrun (BASELINE: 100 M rows over 8 GPUs = 77 GB per GPU, more
        than an 80 GB H100 holds: default 6.25 M rows per GPU, 50 M over 8)
  cfg6  Binary Flat Hamming, 1M x 256 bits, batch 1024, top-10
  cfg6s Binary Flat Hamming, 16384 x 256 bits, batch 128, top-10 (below the tile scan's work threshold: exact scan)
  cfg7  Binary IVF-Flat Hamming, 10M x 512 bits, nlist 2048, nprobe 80, batch 1024, top-10   (--bin-n, --bin-dim)
  range IVF-Flat L2 range search at the headline shape (1M x 768, nlist 1024, nprobe 32, batch 1024, max_results 1024,
        radius keeping ~100 hits a query): the tile range scan against exact_only, alternating in one call; nq = 8 (the exact
        side of the dispatch); a radius every query's capture overflows; the same search through b200vs_shard_* at world 1
Each line: device-resident QPS (CUDA events), e2e QPS through the host-pointer C ABI, parity with the oracle on a
bounded sample, the dominant kernel's time from the library's profiling mode and the algorithmic figure of
SURVEY.md §8(d).  Scaled sizes are stated in the line ("scaled_from").
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(ROOT, "dingo-store_b200", "python"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import torch  # noqa: E402

import b200vs  # noqa: E402
import oracle_lib  # noqa: E402
import pq_codes  # noqa: E402
import binary_oracle  # noqa: E402
import b200vs.shard as shard_host  # noqa: E402


def peak():
    try:
        return float(json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))["hbm_gbs"])
    except Exception:
        return 3350.0  # H100 SXM data sheet


def time_search(ix, xq, k, steps=20, warmup=5, **kw):
    dev = torch.device("cuda", 0)
    nq = xq.shape[0]
    q = torch.from_numpy(xq).to(dev)
    od = torch.empty((nq, k), dtype=torch.float32, device=dev)
    oi = torch.empty((nq, k), dtype=torch.int64, device=dev)
    sp, keep = b200vs.make_search_params(**kw)
    st = torch.cuda.Stream(device=dev)
    for _ in range(warmup):
        ix.search_device(nq, q.data_ptr(), k, od.data_ptr(), oi.data_ptr(), stream=st.cuda_stream, sp=sp)
    st.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(st)
    for _ in range(steps):
        ix.search_device(nq, q.data_ptr(), k, od.data_ptr(), oi.data_ptr(), stream=st.cuda_stream, sp=sp)
    e1.record(st)
    st.synchronize()
    dev_ms = e0.elapsed_time(e1) / steps
    qh = torch.from_numpy(xq).pin_memory()
    hd = torch.empty((nq, k), dtype=torch.float32).pin_memory()
    hi = torch.empty((nq, k), dtype=torch.int64).pin_memory()
    for _ in range(warmup):
        ix.search_raw(nq, qh.data_ptr(), k, hd.data_ptr(), hi.data_ptr(), sp=sp)
    t = time.perf_counter()
    for _ in range(steps):
        ix.search_raw(nq, qh.data_ptr(), k, hd.data_ptr(), hi.data_ptr(), sp=sp)
    e2e_ms = (time.perf_counter() - t) / steps * 1e3
    ix.set_profiling(True)
    ix.search_device(nq, q.data_ptr(), k, od.data_ptr(), oi.data_ptr(), stream=st.cuda_stream, sp=sp)
    st.synchronize()
    stats = ix.stats()
    ix.set_profiling(False)
    return dev_ms, e2e_ms, stats, hd.numpy().copy(), hi.numpy().copy()


def rnd(n, d, seed, dist="uniform"):
    g = torch.Generator(device="cuda")
    g.manual_seed(seed)
    out = np.empty((n, d), np.float32)
    for a in range(0, n, 262144):
        m = min(262144, n - a)
        x = torch.rand((m, d), generator=g, device="cuda") if dist == "uniform" else torch.randn((m, d), generator=g, device="cuda")
        out[a:a + m] = x.cpu().numpy()
    return out


def cfg1(o, cores):
    n, d, k = 100_000, 128, 10
    xb = rnd(n, d, 1234)
    ids = np.arange(1, n + 1, dtype=np.int64)
    ix = b200vs.Index(b200vs.FLAT, b200vs.L2, d)
    for a in range(0, n, 32768):
        ix.add(xb[a:a + 32768], ids[a:a + 32768])
    xq = rnd(1, d, 4321)
    dev_ms, e2e_ms, st, D, I = time_search(ix, xq, k, steps=200, warmup=20)
    t = time.perf_counter()
    reps = 20
    for _ in range(reps):
        Do, Io = o.flat_search(oracle_lib.L2, xb, ids, xq, k, nthreads=1)
    cpu_ms = (time.perf_counter() - t) / reps * 1e3
    bytes_q = n * d * 4
    return {"config": "cfg1 Flat L2 100Kx128 top-10 batch=1", "qps_device": 1e3 / dev_ms, "latency_ms_device": dev_ms, "qps_e2e": 1e3 / e2e_ms,
            "ids_bit_exact": bool(np.array_equal(I, Io)), "dist_bit_exact": bool(np.array_equal(D.view(np.uint32), Do.view(np.uint32))),
            "algorithmic_bytes_per_query": bytes_q, "achieved_gbs_whole_call": bytes_q / (dev_ms * 1e-3) / 1e9, "hbm_peak_gbs": peak(),
            "cpu_baseline": {"qps": 1e3 / cpu_ms, "cores": 1, "kind": "port", "sample": "the same single query, one thread (the reference runs one query per task)"},
            "path": "exact FP32 scan (batch < 16)", "search_stats": st}


def cfg2(o, cores):
    n, d, nlist, nprobe, nq, k = 1_000_000, 768, 1024, 32, 256, 10
    xb = rnd(n, d, 1234)
    ids = np.arange(1, n + 1, dtype=np.int64)
    ix = b200vs.Index(b200vs.IVF_FLAT, b200vs.L2, d, nlist=nlist)
    ix.train(xb[:nlist * 256])
    for a in range(0, n, 32768):
        ix.add(xb[a:a + 32768], ids[a:a + 32768])
    xq = rnd(nq, d, 4321)
    dev_ms, e2e_ms, st, D, I = time_search(ix, xq, k, nprobe=nprobe)
    off, lx, _, lids = ix.export_lists(nlist)
    lx = o.numa_spread(lx, cores)
    cent = ix.get_trained_state()[32:].view(np.float32).reshape(nlist, d)
    t = time.perf_counter()
    Do, Io = o.ivfflat_search(oracle_lib.L2, cent, off, lx, lids, xq, k, nprobe, nthreads=cores)
    cpu_s = time.perf_counter() - t
    rows = st[4]
    return {"config": "cfg2 IVF-Flat L2 1Mx768 nlist=1024 nprobe=32 batch=256 top-10", "qps_device": nq / dev_ms * 1e3, "ms_per_batch_device": dev_ms,
            "qps_e2e": nq / e2e_ms * 1e3, "ids_bit_exact": bool(np.array_equal(I, Io)), "dist_bit_exact": bool(np.array_equal(D.view(np.uint32), Do.view(np.uint32))),
            "recall_at_10_vs_oracle": float(np.mean([len(set(a) & set(b)) / k for a, b in zip(I, Io)])),
            "roofline": {"bound": "hbm", "kernel": "tc_scan_kernel capture pass", "kernel_ms": st[3] / 1e6, "algorithmic_bytes": rows * (d * 4 + 8),
                         "achieved": rows * (d * 4 + 8) / max(st[3], 1) , "unit": "GB/s", "peak": peak(), "frac": rows * (d * 4 + 8) / max(st[3], 1) / peak()},
            "cpu_baseline": {"qps": nq / cpu_s, "cores": cores, "kind": "port", "sample": f"all {nq} queries, {cores} threads, one query per task"},
            "fallback_queries": st[2], "search_stats": st}


def cfg3(o, cores, n, nbits=8, M=96):
    d, nlist, nprobe, nq, k = 768, 2048, 64, 1024, 100
    ksub, code_size = 1 << nbits, pq_codes.code_size(M, nbits)
    ix = b200vs.Index(b200vs.IVF_PQ, b200vs.IP, d, nlist=nlist, pq_m=M, pq_nbits=nbits)
    g = torch.Generator(device="cuda")
    g.manual_seed(1234)
    t0 = time.time()
    ntrain = max(256 * nlist, 65536)
    train = torch.randn((ntrain, d), generator=g, device="cuda").cpu().numpy()
    ix.train(train)
    t_train = time.time() - t0
    keep = None
    t0 = time.time()
    nid = 1
    for a in range(0, n, 131072):
        m = min(131072, n - a)
        x = torch.randn((m, d), generator=g, device="cuda").cpu().numpy()
        if keep is None:
            keep = x[:20000].copy()
        for b in range(0, m, 32768):
            mm = min(32768, m - b)
            ix.add(x[b:b + mm], np.arange(nid, nid + mm, dtype=np.int64))
            nid += mm
    t_add = time.time() - t0
    xq = rnd(nq, d, 4321, "normal")
    dev_ms, e2e_ms, st, D, I = time_search(ix, xq, k, steps=5, warmup=2, nprobe=nprobe)
    # parity on a sample: oracle LUT scan over the exported codes with the GPU-trained state
    blob = ix.get_trained_state()
    cent = blob[48:48 + nlist * d * 4].view(np.float32).reshape(nlist, d)
    cb = blob[48 + nlist * d * 4:].view(np.float32).reshape(M, ksub, d // M)
    off, _, codes, lids = ix.export_lists(nlist, with_vectors=False, code_size=code_size)
    ns = 32
    t = time.perf_counter()
    if nbits == 8:
        Do, Io = o.ivfpq_search(oracle_lib.IP, cent, cb, off, codes, lids, xq[:ns], k, nprobe, nthreads=cores)
    else:
        Do, Io = pq_codes.ivfpq_search(o, oracle_lib.IP, cent, cb, off, codes, lids, xq[:ns], k, nprobe, nthreads=cores)
    cpu_s = time.perf_counter() - t
    lookups = float(st[4]) * M * 0 + 0  # per-batch lookups need the per-query probe sizes: use avg list len
    avg_len = n / nlist
    lookups = nq * nprobe * avg_len * M
    return {"config": f"cfg3 IVF-PQ IP {n}x768 M={M} nbits={nbits} nlist=2048 nprobe=64 batch=1024 top-100", "scaled_from": "10M x 768" if n < 10_000_000 else None,
            "qps_device": nq / dev_ms * 1e3, "ms_per_batch_device": dev_ms, "qps_e2e": nq / e2e_ms * 1e3,
            "ids_bit_exact_sample": bool(np.array_equal(I[:ns], Io)), "recall_at_100_vs_oracle": float(np.mean([len(set(a) & set(b)) / k for a, b in zip(I[:ns], Io)])),
            "max_rel_dist_err": float(np.max(np.abs(D[:ns] - Do) / np.maximum(np.abs(Do), 1e-6))),
            "roofline": {"bound": "shared-memory LUT", "kernel": "pq_scan_select_kernel" if nbits == 8 else f"pq_scan_packed_kernel<IP, {nbits}>",
                         "kernel_ms": st[3] / 1e6, "lookups_per_batch": lookups,
                         "achieved_lookups_per_s": lookups / max(st[3] * 1e-9, 1e-9), "bytes_scan_equiv_gbs": lookups / max(st[3], 1), "hbm_peak_gbs": peak(),
                         **({} if nbits == 8 else {"code_size": code_size, "code_bytes_per_batch": nq * nprobe * avg_len * code_size})},
            "cpu_baseline": {"qps": ns / cpu_s, "cores": cores, "kind": "port", "sample": f"first {ns} queries, {cores} threads"},
            "train_seconds": t_train, "add_seconds": t_add, "search_stats": st}


def cfg3s(o, cores, n, nbits=8, M=96, steps=5, warmup=2, oracle_q=32):
    """cfg3 through the list-sharded deployment (b200vs_shard_*): shard_train, shard_add_device (rows generated on the
    device, n / world per rank), the sharded search.  At world 1 the plain b200vs_search runs on the same index next to it;
    under torchrun rank 0 gathers the exported codes for the oracle.  Rank 0 returns the JSON line."""
    import torch.distributed as dist
    rank, world, local = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1)), int(os.environ.get("LOCAL_RANK", 0))
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    if world > 1 and not dist.is_initialized():
        dist.init_process_group("nccl", device_id=dev)
    d, nlist, nprobe, nq, k = 768, 2048, 64, 1024, 100
    ksub, code_size = 1 << nbits, pq_codes.code_size(M, nbits)
    ix = b200vs.Index(b200vs.IVF_PQ, b200vs.IP, d, nlist=nlist, pq_m=M, pq_nbits=nbits, device=local)
    idb = None
    if world > 1:
        t = torch.from_numpy(b200vs.Shard.unique_id() if rank == 0 else np.zeros(128, np.uint8)).to(dev)
        dist.broadcast(t, 0)
        idb = t.cpu().numpy()
    sh = b200vs.Shard(ix, rank, world, idb, lanes=2)
    g = torch.Generator(device=dev)
    g.manual_seed(1234 + rank)
    t0 = time.time()
    ntrain = max(256 * nlist // world, 65536)  # rank 0 needs 256 * 2^nbits rows for the codebooks
    sh.train(torch.randn((ntrain, d), generator=g, device=dev).cpu().numpy())
    t_train = time.time() - t0
    t0 = time.time()
    n_per = n // world
    for a in range(0, n_per, 131072):
        m = min(131072, n_per - a)
        x = torch.randn((m, d), generator=g, device=dev)
        ids = torch.arange(rank * n_per + a + 1, rank * n_per + a + 1 + m, dtype=torch.int64, device=dev)
        torch.cuda.synchronize()
        sh.add_device(m, x.data_ptr(), ids.data_ptr())
    t_add = time.time() - t0
    xq = rnd(nq, d, 4321, "normal")
    sp, _keep = b200vs.make_search_params(nprobe=nprobe)
    q = torch.from_numpy(xq).to(dev)
    od = torch.empty((nq, k), dtype=torch.float32, device=dev)
    oi = torch.empty((nq, k), dtype=torch.int64, device=dev)
    st = torch.cuda.Stream(device=dev)
    for _ in range(warmup):
        sh.search_device(nq, q.data_ptr(), k, od.data_ptr(), oi.data_ptr(), stream=st.cuda_stream, sp=sp)
    st.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(st)
    for _ in range(steps):
        sh.search_device(nq, q.data_ptr(), k, od.data_ptr(), oi.data_ptr(), stream=st.cuda_stream, sp=sp)
    e1.record(st)
    st.synchronize()
    dev_ms = e0.elapsed_time(e1) / steps
    t = time.perf_counter()
    for _ in range(steps):
        D, I = sh.search(xq, k, nprobe=nprobe)
    e2e_ms = (time.perf_counter() - t) / steps * 1e3
    plain = None
    if world == 1:  # the unsharded search on the same index, same shape
        p_dev, p_e2e, p_st, Dp, Ip = time_search(ix, xq, k, steps=steps, warmup=warmup, nprobe=nprobe)
        plain = {"qps_device": nq / p_dev * 1e3, "ms_per_batch_device": p_dev, "qps_e2e": nq / p_e2e * 1e3,
                 "ids_equal_sharded": bool(np.array_equal(I, Ip)), "dist_bits_equal_sharded": bool(np.array_equal(D.view(np.uint32), Dp.view(np.uint32)))}
    blob = ix.get_trained_state()
    cent = blob[48:48 + nlist * d * 4].view(np.float32).reshape(nlist, d)
    cb = blob[48 + nlist * d * 4:].view(np.float32).reshape(M, ksub, d // M)
    off, _, codes, lids = ix.export_lists(nlist, with_vectors=False, code_size=code_size)
    if world > 1:
        parts = [None] * world
        dist.all_gather_object(parts, (off, codes, lids))
        if rank != 0:
            sh.close()
            return None
        off = np.zeros(nlist + 1, np.int64)
        gc, gi = [], []
        for l in range(nlist):
            for (po, pc, pi) in parts:
                gc.append(pc[po[l]:po[l + 1]])
                gi.append(pi[po[l]:po[l + 1]])
            off[l + 1] = off[l] + sum(int(po[l + 1] - po[l]) for (po, _, _) in parts)
        codes, lids = np.concatenate(gc, 0), np.concatenate(gi, 0)
    sh.close()
    Do, Io = pq_codes.ivfpq_search(o, oracle_lib.IP, cent, cb, off, codes, lids, xq[:oracle_q], k, nprobe, nthreads=cores)
    return {"config": f"cfg3s IVF-PQ IP {n}x768 M={M} nbits={nbits} nlist=2048 nprobe=64 batch=1024 top-100, list-sharded over {world} GPU(s)",
            "scaled_from": "10M x 768" if n < 10_000_000 else None, "world": world,
            "qps_device": nq / dev_ms * 1e3, "ms_per_batch_device": dev_ms, "qps_e2e": nq / e2e_ms * 1e3,
            "ids_bit_exact_sample": bool(np.array_equal(I[:oracle_q], Io)),
            "dist_bit_exact_sample": bool(np.array_equal(D[:oracle_q].view(np.uint32), Do.view(np.uint32))),
            "plain_b200vs_search_same_shape": plain, "train_seconds": t_train, "add_seconds": t_add}


def cfg4(o, cores, n, build_threads=64, build="host", build_batch=0):
    """HNSW cosine.  build = "host": the graph is built by the engine with `build_threads` concurrent host writers — what the
    reference does with its thread pool (vector_index_hnsw.cc:229-243; such a graph is not reproducible run to run).
    build = "device": b200vs_hnsw_add_batched with `build_batch` rows per batch (0 = the library default).  Either way the
    oracle adopts that very graph (oracle_hnsw_import), so both sides search the SAME index, as for the IVF types."""
    d, M, efc, ef, nq, k = 768, 16, 200, 128, 512, 10
    xb = rnd(n, d, 1234)
    labels = np.arange(1, n + 1, dtype=np.int64)
    ix = b200vs.Index(b200vs.HNSW, b200vs.COSINE, d, hnsw_m=M, hnsw_efc=efc, max_elements=n * 2, hnsw_build_threads=build_threads)
    phases = {}
    if build == "device":
        ix.set_profiling(True)  # CUDA events between the phases of every batch; no synchronisation until the call ends
    t0 = time.time()
    for a in range(0, n, 65536):
        if build == "device":
            ix.add_batched(xb[a:a + 65536], labels[a:a + 65536], batch=build_batch)
            for p in ("build_search", "build_select", "build_link"):
                phases[p] = phases.get(p, 0.0) + ix.phase_times()[p] / 1e3
        else:
            ix.add(xb[a:a + 65536], labels[a:a + 65536])
    t_build = time.time() - t0
    ix.set_profiling(False)
    xq = rnd(nq, d, 4321)
    dev_ms, e2e_ms, st, D, I = time_search(ix, xq, k, steps=5, warmup=2, efsearch=ef)
    h = oracle_lib.OracleHnsw(o, oracle_lib.COSINE, d, n, M, efc)
    t0 = time.time()
    h.load(ix.get_trained_state())
    t_import = time.time() - t0
    t = time.perf_counter()
    Do, Io, nd, nh = h.search(xq, k, ef=ef, nthreads=cores)
    cpu_s = time.perf_counter() - t
    t = time.perf_counter()
    h.search(xq[:64], k, ef=ef, nthreads=min(16, cores))
    cpu16_s = time.perf_counter() - t
    # graph quality: recall of the search against the exact answer on a sample
    ns = 64
    xn = xb / (np.linalg.norm(xb, axis=1, keepdims=True) + 1e-30)
    qn = xq[:ns] / (np.linalg.norm(xq[:ns], axis=1, keepdims=True) + 1e-30)
    exact = np.argsort(-(qn @ xn.T), axis=1)[:, :k] + 1
    rec = float(np.mean([len(set(a) & set(b)) / k for a, b in zip(I[:ns], exact)]))
    bytes_batch = float(nd.sum()) * d * 4 + float(nh.sum()) * (4 + 2 * M * 4)
    return {"config": f"cfg4 HNSW cosine {n}x768 M=16 efC=200 efSearch=128 batch=512 top-10", "scaled_from": None if n >= 1_000_000 else "1M x 768",
            "qps_device": nq / dev_ms * 1e3, "ms_per_batch_device": dev_ms, "qps_e2e": nq / e2e_ms * 1e3,
            "graph": f"built by the engine with {build_threads} concurrent writers (reference: 16-thread pool); the oracle searches the same graph",
            "ids_bit_exact": bool(np.array_equal(I, Io)), "dist_bit_exact": bool(np.array_equal(D.view(np.uint32), Do.view(np.uint32))),
            "recall_at_10_vs_exact_cosine": rec,
            "roofline": {"bound": "hbm random gathers", "kernel": "hnsw_search_kernel", "kernel_ms": st[3] / 1e6, "algorithmic_bytes": bytes_batch,
                         "ndis_per_query": float(nd.mean()), "hops_per_query": float(nh.mean()), "achieved": bytes_batch / max(st[3], 1), "unit": "GB/s",
                         "peak": peak(), "frac": bytes_batch / max(st[3], 1) / peak()},
            "cpu_baseline": {"qps": nq / cpu_s, "cores": cores, "kind": "port", "sample": f"all {nq} queries, {cores} threads",
                             "reference_shape_16_threads_qps": 64 / cpu16_s},
            "build": build, "build_seconds_engine": t_build, "oracle_import_seconds": t_import, "search_stats": st,
            **({"graph": f"built on the device by b200vs_hnsw_add_batched, batch {build_batch or 'default'}; the oracle searches the same graph",
                "build_phase_seconds": phases} if build == "device" else {})}

def cfg5(o, cores, rows_per_gpu, steps=10, warmup=3, dim=1536, nlist_per_gpu=2048, nprobe=64, nq=4096, k=10, in_flight=2, verify=256, oracle_q=8):
    """BASELINE config 5: one logical IVF-Flat index list-sharded over the world's GPUs behind b200vs_shard_*.
    Build = distributed training, a planning pass that pre-sizes every owned list, then the add pass (rows generated on the
    device, routed to their list owner over NCCL).  Every rank prints nothing; rank 0 returns the JSON line."""
    import torch.distributed as dist
    rank, world, local = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1)), int(os.environ.get("LOCAL_RANK", 0))
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    if world > 1 and not dist.is_initialized():
        dist.init_process_group("nccl", device_id=dev)
    d, n = dim, rows_per_gpu
    nlist = nlist_per_gpu * world
    t0 = time.time()
    ix = b200vs.Index(b200vs.IVF_FLAT, b200vs.L2, d, nlist=nlist, device=local)
    idb = None
    if world > 1:
        t = torch.from_numpy(b200vs.Shard.unique_id() if rank == 0 else np.zeros(128, np.uint8)).to(dev)
        dist.broadcast(t, 0)
        idb = t.cpu().numpy()
    sh = b200vs.Shard(ix, rank, world, idb, lanes=in_flight)
    chunk = 65536

    def chunks():
        g = torch.Generator(device=dev)
        g.manual_seed(1234 + rank)
        for a in range(0, n, chunk):
            m = min(chunk, n - a)
            yield a, torch.rand((m, d), generator=g, device=dev, dtype=torch.float32)

    g0 = torch.Generator(device=dev)
    g0.manual_seed(99 + rank)
    ntrain = min(n, nlist_per_gpu * 64)
    sh.train(torch.rand((ntrain, d), generator=g0, device=dev, dtype=torch.float32).cpu().numpy())
    t_train = time.time() - t0
    t1 = time.time()
    for a, x in chunks():  # pass 1: assignment only -> per-list row counts
        torch.cuda.synchronize()
        sh.plan_add_device(x.shape[0], x.data_ptr())
    sh.plan_commit()       # all-reduce of the counts, ONE arena allocation per rank
    t_plan = time.time() - t1
    t2 = time.time()
    for a, x in chunks():  # pass 2: the same rows again, now stored on their list owner
        gid = torch.arange(a + 1, a + 1 + x.shape[0], dtype=torch.int64, device=dev) + rank * n
        torch.cuda.synchronize()
        sh.add_device(x.shape[0], x.data_ptr(), gid.data_ptr())
    t_add = time.time() - t2
    del x
    torch.cuda.empty_cache()
    mem = ix.get_memory_size()
    cnt = torch.tensor([ix.get_count()], dtype=torch.int64, device=dev)
    if world > 1:
        dist.all_reduce(cnt)
    # ---- timed search: device-resident queries, `in_flight` batches in flight ----
    gq = torch.Generator(device=dev)
    gq.manual_seed(4321)
    qs = [torch.rand((nq, d), generator=gq, device=dev, dtype=torch.float32) for _ in range(2)]
    L = in_flight
    od = [torch.empty((nq, k), dtype=torch.float32, device=dev) for _ in range(L)]
    oi = [torch.empty((nq, k), dtype=torch.int64, device=dev) for _ in range(L)]
    sp, _keep = b200vs.make_search_params(nprobe=nprobe)
    main = torch.cuda.Stream(device=dev)
    sts = [torch.cuda.Stream(device=dev) for _ in range(L)]
    torch.cuda.set_stream(main)
    seq = [0]

    host_ms = []

    def step(i, lanes):
        ln = i % lanes
        th = time.perf_counter()
        sh.search_device(nq, qs[i % 2].data_ptr(), k, od[ln].data_ptr(), oi[ln].data_ptr(), stream=sts[ln].cuda_stream, sp=sp, seq=seq[0])
        host_ms.append((time.perf_counter() - th) * 1e3)
        seq[0] += 1

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    def timed(nsteps, lanes):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(main)
        for st in sts[:lanes]:
            st.wait_event(e0)
        for i in range(nsteps):
            step(i, lanes)
        for st in sts[:lanes]:
            ev = torch.cuda.Event()
            ev.record(st)
            main.wait_event(ev)
        e1.record(main)
        barrier()
        return e0.elapsed_time(e1)

    for i in range(max(warmup, 2 * L)):
        step(i, L)
    barrier()
    ms = timed(steps, L)
    del host_ms[:]
    ms1 = timed(steps, 1)
    host_enqueue_ms = float(np.median(host_ms)) if host_ms else None
    # e2e through the host-pointer collective call
    qh = [q.cpu().pin_memory() for q in qs]
    hd = torch.empty((nq, k), dtype=torch.float32).pin_memory()
    hi = torch.empty((nq, k), dtype=torch.int64).pin_memory()
    for i in range(2):
        sh.search_raw(nq, qh[i % 2].data_ptr(), k, hd.data_ptr(), hi.data_ptr(), sp=sp, seq=seq[0]); seq[0] += 1
    barrier()
    tt = time.perf_counter()
    for i in range(steps):
        sh.search_raw(nq, qh[i % 2].data_ptr(), k, hd.data_ptr(), hi.data_ptr(), sp=sp, seq=seq[0]); seq[0] += 1
    barrier()
    e2e_ms = (time.perf_counter() - tt) * 1e3
    tm = torch.tensor([ms, ms1, e2e_ms], dtype=torch.float64, device=dev)
    if world > 1:
        dist.all_reduce(tm, op=dist.ReduceOp.MAX)
    ms, ms1, e2e_ms = tm.tolist()
    # roofline of the list scan on this rank (profiling pass, never part of the timed numbers)
    ix.set_profiling(True)
    sh.search_device(nq, qs[0].data_ptr(), k, od[0].data_ptr(), oi[0].data_ptr(), stream=sts[0].cuda_stream, sp=sp, seq=seq[0]); seq[0] += 1
    torch.cuda.synchronize()
    st = ix.stats()
    ph = ix.phase_times()
    ix.set_profiling(False)
    alg = st[4] * (d * 4 + 8)
    roof = torch.tensor([alg / max(st[3], 1), st[3] / 1e6, float(st[2])], dtype=torch.float64, device=dev)
    roofs = [torch.zeros_like(roof) for _ in range(world)]
    phs = [None] * world
    if world > 1:
        dist.all_gather(roofs, roof)
        dist.all_gather_object(phs, {a: round(v, 3) for a, v in ph.items()})
    else:
        roofs = [roof]
        phs = [ph]
    # ---- verification 1: tile path vs the exact FP32 scan path (different kernels) on `verify` queries, full scale ----
    xq = qh[0].numpy()[:verify].copy()
    Dt, It = sh.search(xq, k, seq=seq[0], nprobe=nprobe); seq[0] += 1
    De, Ie = sh.search(xq, k, seq=seq[0], nprobe=nprobe, exact_only=True); seq[0] += 1
    # ---- verification 2: the CPU oracle on the lists the first `oracle_q` queries probe (exported list by list) ----
    cent = ix.get_trained_state()[32:].view(np.float32).reshape(nlist, d)
    xo = xq[:oracle_q]
    # lists worth exporting: the exact top-(nprobe + 8) centroids of each query (a few extra: rounding at the boundary is harmless)
    dd = ((xo[:, None, :].astype(np.float64) - cent[None, :, :].astype(np.float64)) ** 2).sum(-1)
    pls = set(np.unique(np.argsort(dd, axis=1, kind="stable")[:, :nprobe + 8]).tolist())
    b, e = sh.list_range()
    off = np.zeros(nlist + 1, np.int64)
    vs, idl = [], []
    for l in range(nlist):
        if b <= l < e and l in pls:
            v, i_ = ix.export_list(l)
            vs.append(v); idl.append(i_)
            off[l + 1] = off[l] + v.shape[0]
        else:
            off[l + 1] = off[l]
    lx = np.concatenate(vs, 0) if vs else np.zeros((0, d), np.float32)
    lids = np.concatenate(idl, 0) if idl else np.zeros(0, np.int64)
    threads = max(1, cores // world)
    tt = time.time()
    Do, Io = o.ivfflat_search(oracle_lib.L2, cent, off, lx, lids, xo, k, nprobe, nthreads=min(threads, oracle_q))
    cpu_s = time.time() - tt
    if world > 1:
        gd = [torch.empty((oracle_q, k), dtype=torch.float32, device=dev) for _ in range(world)]
        gi = [torch.empty((oracle_q, k), dtype=torch.int64, device=dev) for _ in range(world)]
        dist.all_gather(gd, torch.from_numpy(Do).to(dev))
        dist.all_gather(gi, torch.from_numpy(Io).to(dev))
        Dm, Im = shard_host.merge_topk(torch.stack(gd).cpu().numpy(), torch.stack(gi).cpu().numpy(), k)
        cs = torch.tensor([cpu_s], dtype=torch.float64, device=dev)
        dist.all_reduce(cs, op=dist.ReduceOp.MAX)
        cpu_s = float(cs.item())
    else:
        Dm, Im = Do, Io
    line = None
    if rank == 0:
        fr = [float(r[0]) / peak() for r in roofs]
        line = {"config": f"cfg5 IVF-Flat L2 {n * world}x{d} ({n} rows per GPU x {world} GPUs), nlist={nlist} ({nlist_per_gpu} per GPU), nprobe={nprobe}, batch={nq}, top-{k}, list-sharded (b200vs_shard_*)",
                "scaled_from": None if n * world >= 100_000_000 else "100M x 1536 over 8 GPUs (12.5 M rows = 77 GB per GPU, more than an 80 GB H100 holds beside its workspace)",
                "assumptions": "nlist / nprobe are not given in BASELINE.json: 16384 / 64 at 8 GPUs (SURVEY 8d); synthetic U[0,1) rows generated on the device",
                "n_gpus": world, "rows_total": int(cnt.item()), "index_bytes_per_gpu": mem,
                "qps_device": nq * steps / (ms / 1e3), "ms_per_batch_device": ms / steps, "batches_in_flight": L,
                "qps_single_stream": nq * steps / (ms1 / 1e3), "qps_e2e": nq * steps / (e2e_ms / 1e3), "ms_per_batch_e2e": e2e_ms / steps,
                "roofline_per_rank": {"bound": "hbm", "kernel": "tc_scan_kernel capture pass", "achieved_gbs": [float(r[0]) for r in roofs], "kernel_ms": [float(r[1]) for r in roofs],
                                      "peak": peak(), "frac": fr, "frac_min": min(fr), "frac_max": max(fr), "fallback_queries": [int(r[2]) for r in roofs],
                                      "algorithmic_bytes_rank0": alg},
                "phase_ms_rank0": {a: round(v, 4) for a, v in ph.items()}, "phase_ms_all_ranks": phs, "host_enqueue_ms_per_batch_median": host_enqueue_ms,
                "verify_tile_vs_exact_scan": {"queries": int(verify), "ids_bit_exact": bool(np.array_equal(It, Ie)),
                                              "dist_bit_exact": bool(np.array_equal(Dt.view(np.uint32), De.view(np.uint32)))},
                "verify_vs_oracle": {"queries": int(oracle_q), "ids_bit_exact": bool(np.array_equal(It[:oracle_q], Im)),
                                     "dist_bit_exact": bool(np.array_equal(Dt[:oracle_q].view(np.uint32), Dm.view(np.uint32))),
                                     "recall_at_10": float(np.mean([len(set(a_) & set(b_)) / k for a_, b_ in zip(It[:oracle_q], Im)])),
                                     "how": "CPU oracle on every rank's probed lists (exported list by list), per-rank top-k merged with the MergeSearchResults rule"},
                "cpu_baseline": {"qps": oracle_q / cpu_s, "cores": threads * world, "kind": "port",
                                 "sample": f"{oracle_q} queries; each rank's oracle scans only the probed lists that rank owns ({threads} threads per rank, max over ranks)"},
                "build_seconds": {"train": t_train, "plan_pass": t_plan, "add_pass": t_add}, "search_stats": st}
    sh.close()
    return line


def cfg_calc(o, cores):
    """SURVEY 8f-4: the UtilService distance matrix (VectorCalcDistance), 1024 x 1024 x 768, host pointers in and out."""
    nl = nr = 1024
    d = 768
    left, right = rnd(nl, d, 11), rnd(nr, d, 12)
    out = {}
    for name, metric in (("l2", b200vs.L2), ("cosine", b200vs.COSINE)):
        b200vs.calc_distance(b200vs.ALGORITHM_FAISS, metric, left, right)  # warm-up (context, allocations)
        t = time.time()
        reps = 5
        for _ in range(reps):
            got = b200vs.calc_distance(b200vs.ALGORITHM_FAISS, metric, left, right)
        gpu_s = (time.time() - t) / reps
        ns = 64  # bounded CPU sample: 64 left rows against all right rows
        t = time.time()
        want, _, _ = o.calc_distance(1, oracle_lib.L2 if metric == b200vs.L2 else oracle_lib.COSINE, left[:ns], right)
        cpu_s = (time.time() - t) * nl / ns
        out[name] = {"pairs_per_s_e2e": nl * nr / gpu_s, "ms_e2e": gpu_s * 1e3, "bit_exact_vs_oracle": bool(np.array_equal(got[:ns].view(np.uint32), want.view(np.uint32))),
                     "cpu_pairs_per_s_1thread": nl * nr / cpu_s}
    return {"config": "calc_distance", "workload": f"VectorCalcDistance {nl} x {nr} x {d} f32, ALGORITHM_FAISS, host buffers (H2D + D2H inside)", **out}


def cfg_brute(o, cores):
    """SURVEY 8f-3: BruteForceSearch over 200K x 768 rows streamed in 2048-row tiles (FLAGS_vector_index_bruteforce_batch_count)."""
    n, d, nq, k, tile = 200_000, 768, 256, 10, 2048
    xb, xq = rnd(n, d, 21), rnd(nq, d, 22)
    ids = np.arange(1, n + 1, dtype=np.int64)

    def run(t):
        sc = b200vs.BruteForceScan(b200vs.L2, d, xq, k)
        for a in range(0, n, t):
            sc.push(xb[a:a + t], ids[a:a + t])
        return sc.finish()

    run(tile)
    res = {}
    for t in (tile, 32768):
        t0 = time.time()
        gd, gi = run(t)
        res[f"tile_{t}"] = {"seconds": time.time() - t0, "rows_per_s": n / (time.time() - t0), "queries_x_rows_per_s": nq * n / (time.time() - t0)}
    ns = 16
    t0 = time.time()
    wd, wi = o.flat_search(oracle_lib.L2, xb, ids, xq[:ns], k, nthreads=cores)
    cpu_s = (time.time() - t0) * nq / ns
    return {"config": "bruteforce_scan", "workload": f"BruteForceSearch L2 {n} x {d} streamed from host, batch {nq}, top-{k}", **res,
            "ids_bit_exact_vs_oracle": bool(np.array_equal(gi[:ns], wi)), "dist_bit_exact_vs_oracle": bool(np.array_equal(gd[:ns].view(np.uint32), wd.view(np.uint32))),
            "cpu_baseline_seconds_scaled": cpu_s, "cpu_cores": cores}


# __popc issues 16 per clock per SM on sm_90 (CUDA programming guide throughput table; not measured): 132 SMs at ~1.7 GHz
POPC_BOUND_WORDS_PER_S = 16 * 132 * 1.7e9


def rnd_bits(n, nb, seed):
    g = torch.Generator(device="cuda")
    g.manual_seed(seed)
    out = np.empty((n, nb), np.uint8)
    for a in range(0, n, 1 << 20):
        m = min(1 << 20, n - a)
        out[a:a + m] = torch.randint(0, 256, (m, nb), generator=g, device="cuda", dtype=torch.uint8).cpu().numpy()
    return out


EXACT_ONLY = False


def binary_line(name, ix, xq, k, word_popcounts, Do, Io, oracle_q, **kw):
    """Device / e2e QPS, list-scan kernel time, word popcounts per second against the popcount bound, parity on the first
    oracle_q queries."""
    nq = xq.shape[0]
    dev_ms, e2e_ms, st, D, I = time_search(ix, xq, k, exact_only=EXACT_ONLY, **kw)
    kernel_s = st[3] / 1e9
    tile = st[1] > 0
    return {"config": name, "qps_device": nq / dev_ms * 1e3, "ms_per_batch_device": dev_ms, "qps_e2e": nq / e2e_ms * 1e3,
            "ids_bit_exact": bool(np.array_equal(I[:oracle_q], Io)), "dist_bit_exact": bool(np.array_equal(D[:oracle_q].view(np.uint32), Do.view(np.uint32))),
            "parity_sample": f"first {oracle_q} of {nq} queries against tests/binary_oracle.py",
            "roofline": {"bound": "popcount issue rate", "kernel": "bt_scan_kernel<1> (capture)" if tile else "scan_select_kernel<HammingDist>", "kernel_ms": kernel_s * 1e3,
                         "word_popcounts": word_popcounts, "achieved": word_popcounts / max(kernel_s, 1e-12), "unit": "word popcounts/s",
                         "peak": POPC_BOUND_WORDS_PER_S, "frac": word_popcounts / max(kernel_s, 1e-12) / POPC_BOUND_WORDS_PER_S,
                         "peak_source": "16 __popc / clock / SM (CUDA programming guide) x 132 SMs x 1.7 GHz, not measured"},
            "bit_pairs_per_s": word_popcounts * 32 / max(kernel_s, 1e-12),
            "path": "BMMA tile scan (list-major)" if tile else "exact Hamming scan (query-major)", "search_stats": st}


def cfg6(o, cores, oracle_q=64):
    n, dim, nq, k = 1_000_000, 256, 1024, 10
    nb, w = dim // 8, (dim // 8 + 3) // 4
    xb = rnd_bits(n, nb, 1234)
    ids = np.arange(1, n + 1, dtype=np.int64)
    ix = b200vs.Index(b200vs.BINARY_FLAT, b200vs.HAMMING, dim)
    for a in range(0, n, 1 << 18):
        ix.add(xb[a:a + (1 << 18)], ids[a:a + (1 << 18)])
    xq = rnd_bits(nq, nb, 4321)
    Do, Io = binary_oracle.flat_search(xb, ids, xq[:oracle_q], k)
    return binary_line(f"cfg6 Binary Flat Hamming {n}x{dim} bits batch={nq} top-{k}", ix, xq, k, nq * n * w, Do, Io, oracle_q)


def cfg6s(o, cores, oracle_q=64):
    """Below the tile scan's work threshold (nq x rows < 2^23): the exact scan is the faster path and serves it."""
    n, dim, nq, k = 16384, 256, 128, 10
    nb, w = dim // 8, (dim // 8 + 3) // 4
    xb = rnd_bits(n, nb, 1234)
    ids = np.arange(1, n + 1, dtype=np.int64)
    ix = b200vs.Index(b200vs.BINARY_FLAT, b200vs.HAMMING, dim)
    ix.add(xb, ids)
    xq = rnd_bits(nq, nb, 4321)
    Do, Io = binary_oracle.flat_search(xb, ids, xq[:oracle_q], k)
    return binary_line(f"cfg6s Binary Flat Hamming {n}x{dim} bits batch={nq} top-{k}", ix, xq, k, nq * n * w, Do, Io, oracle_q)


def cfg7(o, cores, n, dim, oracle_q=16):
    nlist, nprobe, nq, k = 2048, 80, 1024, 10
    nb, w = dim // 8, (dim // 8 + 3) // 4
    xb = rnd_bits(n, nb, 1234)
    ids = np.arange(1, n + 1, dtype=np.int64)
    ix = b200vs.Index(b200vs.BINARY_IVF_FLAT, b200vs.HAMMING, dim, nlist=nlist)
    t = time.perf_counter()
    ix.train(xb)
    train_s = time.perf_counter() - t
    for a in range(0, n, 1 << 20):
        ix.add(xb[a:a + (1 << 20)], ids[a:a + (1 << 20)])
    xq = rnd_bits(nq, nb, 4321)
    cent = ix.get_trained_state()[32:].reshape(-1, nb)
    off, _, codes, lids = ix.export_lists(cent.shape[0])
    P = binary_oracle.probes(cent, xq, min(nprobe, cent.shape[0]))
    rows = int(np.diff(off)[P].sum())  # candidate rows over the batch: each is one row of w word popcounts
    Do, Io = binary_oracle.ivf_search(cent, off, codes, lids, xq[:oracle_q], k, nprobe)
    line = binary_line(f"cfg7 Binary IVF-Flat Hamming {n}x{dim} bits nlist={nlist} nprobe={nprobe} batch={nq} top-{k}", ix, xq, k, rows * w,
                       Do, Io, oracle_q, nprobe=nprobe)
    line["scaled_from"] = None if (n, dim) == (10_000_000, 512) else "10M x 512 bits"
    line["train_seconds"] = train_s
    return line


def card():
    """The card the numbers were measured on: name and power limit (nvidia-smi), stated beside every number."""
    import subprocess
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return out.stdout.strip().splitlines()[0]
    except Exception as e:
        return f"unknown ({e!r})"


def _shard_vs_plain(ix, sh, xq, k, steps, **kw):
    """Device-resident ms per batch (CUDA events) of the sharded and the plain search on the same index, alternating
    (three rounds each, the best kept), and whether the two return the same ids and distance bits."""
    dev = torch.device("cuda", 0)
    nq = xq.shape[0]
    q = torch.from_numpy(xq).to(dev)
    sp, _keep = b200vs.make_search_params(**kw)
    bufs = {w: (torch.empty((nq, k), dtype=torch.float32, device=dev), torch.empty((nq, k), dtype=torch.int64, device=dev)) for w in ("shard", "plain")}
    st = torch.cuda.Stream(device=dev)
    run = {"shard": lambda od, oi: sh.search_device(nq, q.data_ptr(), k, od.data_ptr(), oi.data_ptr(), stream=st.cuda_stream, sp=sp),
           "plain": lambda od, oi: ix.search_device(nq, q.data_ptr(), k, od.data_ptr(), oi.data_ptr(), stream=st.cuda_stream, sp=sp)}
    ms = {"shard": [], "plain": []}
    for w in run:
        for _ in range(2):
            run[w](*bufs[w])
    st.synchronize()
    for _ in range(3):
        for w in run:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(st)
            for _ in range(steps):
                run[w](*bufs[w])
            e1.record(st)
            st.synchronize()
            ms[w].append(e0.elapsed_time(e1) / steps)
    Ds, Is = (t.cpu().numpy() for t in bufs["shard"])
    Dp, Ip = (t.cpu().numpy() for t in bufs["plain"])
    return {"ms_per_batch_device_sharded": ms["shard"], "ms_per_batch_device_plain": ms["plain"],
            "qps_device_sharded": nq / min(ms["shard"]) * 1e3, "qps_device_plain": nq / min(ms["plain"]) * 1e3,
            "ids_equal": bool(np.array_equal(Is, Ip)), "dist_bits_equal": bool(np.array_equal(Ds.view(np.uint32), Dp.view(np.uint32)))}


def cfg1s(o, cores, n=2_000_000, steps=10):
    """Flat L2 through the row-sharded deployment at world 1: rows generated on the device and added with
    b200vs_shard_add_device, then the sharded and the plain search of the same index."""
    d, nq, k = 768, 1024, 10
    dev = torch.device("cuda", 0)
    ix = b200vs.Index(b200vs.FLAT, b200vs.L2, d)
    sh = b200vs.Shard(ix, 0, 1, None, lanes=2)
    g = torch.Generator(device=dev)
    g.manual_seed(1234)
    t0 = time.time()
    for a in range(0, n, 262144):
        m = min(262144, n - a)
        x = torch.rand((m, d), generator=g, device=dev)
        ids = torch.arange(a + 1, a + 1 + m, dtype=torch.int64, device=dev)
        torch.cuda.synchronize()
        sh.add_device(m, x.data_ptr(), ids.data_ptr())
    t_add = time.time() - t0
    xq = rnd(nq, d, 4321)
    line = _shard_vs_plain(ix, sh, xq, k, steps)
    sh.close()
    return {"config": f"1s Flat L2 {n}x{d} batch={nq} top-{k}, row-sharded at world 1 (one GPU)", "card": card(), **line,
            "add_seconds": t_add, "multi_gpu": "not measured (one GPU)"}


def cfg4s(o, cores, n, steps=10):
    """cfg4's HNSW cosine shape through the row-sharded deployment at world 1: the graph is built with
    b200vs_shard_hnsw_add_batched, then the sharded and the plain search of the same index."""
    d, nq, k, ef = 768, 512, 10, 128
    ix = b200vs.Index(b200vs.HNSW, b200vs.COSINE, d, hnsw_m=16, hnsw_efc=200, max_elements=n)
    sh = b200vs.Shard(ix, 0, 1, None, lanes=2)
    t0 = time.time()
    for a in range(0, n, 262144):
        m = min(262144, n - a)
        sh.hnsw_add_batched(rnd(m, d, 1234 + a), np.arange(a + 1, a + 1 + m, dtype=np.int64))
    t_build = time.time() - t0
    xq = rnd(nq, d, 4321)
    line = _shard_vs_plain(ix, sh, xq, k, steps, efsearch=ef)
    sh.close()
    return {"config": f"4s HNSW cosine {n}x{d} M=16 efSearch={ef} batch={nq} top-{k}, row-sharded at world 1 (one GPU)",
            "scaled_from": "1M x 768" if n < 1_000_000 else None, "card": card(), **line, "build_seconds": t_build,
            "multi_gpu": "not measured (one GPU)"}


def cfg_range(o, cores, steps=5):
    """Range search at the headline IVF-Flat shape.  The plain call has no device-pointer entry point, so its times are host
    calls (query upload, [nq, max_results] results back); the sharded call is timed device-resident with CUDA events."""
    n, d, nlist, nprobe, nq, mr = 1_000_000, 768, 1024, 32, 1024, 1024
    xb = rnd(n, d, 1234)
    ix = b200vs.Index(b200vs.IVF_FLAT, b200vs.L2, d, nlist=nlist)
    ix.train(xb[:nlist * 256])
    for a in range(0, n, 32768):
        ix.add(xb[a:a + 32768], np.arange(a + 1, a + 1 + min(32768, n - a), dtype=np.int64))
    del xb
    xq = rnd(nq, d, 4321)
    Dk, _ = ix.search(xq[:64], 100, nprobe=nprobe)
    radius = float(np.median(Dk[:, 99]))  # ~100 hits a query

    def same(a, b):
        return bool(np.array_equal(a[2], b[2]) and np.array_equal(a[1], b[1]) and np.array_equal(a[0].view(np.uint32), b[0].view(np.uint32)))

    def timed(q, r, exact):
        ix.range_search(q, r, mr, nprobe=nprobe, exact_only=exact)
        t = time.perf_counter()
        for _ in range(steps):
            res = ix.range_search(q, r, mr, nprobe=nprobe, exact_only=exact)
        return (time.perf_counter() - t) / steps * 1e3, res

    def profiled(q, r):
        ix.set_profiling(True)
        ix.range_search(q, r, mr, nprobe=nprobe)
        st, ph = ix.stats(), ix.phase_times()
        ix.set_profiling(False)
        return st, ph

    def pair(q, r, reps=3):
        tile, exact, eq = [], [], True
        for _ in range(reps):  # alternating, so both see the same machine state
            tm, a = timed(q, r, False)
            em, b = timed(q, r, True)
            tile.append(tm); exact.append(em); eq = eq and same(a, b)
        st, ph = profiled(q, r)
        return {"nq": len(q), "ms_per_batch_e2e_tile": tile, "ms_per_batch_e2e_exact_only": exact,
                "qps_e2e_tile": len(q) / min(tile) * 1e3, "qps_e2e_exact_only": len(q) / min(exact) * 1e3,
                "ids_dist_counts_equal_all_queries": eq, "mean_hits_kept": float(np.mean(a[2])),
                "tile_queries": st[1], "rerun_queries": st[2], "capture_kernel_ms": st[3] / 1e6, "phase_ms": ph}

    lines = {"headline": pair(xq, radius), "nq8": pair(xq[:8], radius), "overflow": pair(xq, radius * 4)}
    sh = b200vs.Shard(ix, 0, 1, None, lanes=2)
    sp, _keep = b200vs.make_search_params(nprobe=nprobe)
    dev = torch.device("cuda", 0)
    q = torch.from_numpy(xq).to(dev)
    od = torch.empty((nq, mr), dtype=torch.float32, device=dev)
    oi = torch.empty((nq, mr), dtype=torch.int64, device=dev)
    oc = torch.empty((nq,), dtype=torch.int32, device=dev)
    st = torch.cuda.Stream(device=dev)
    for _ in range(2):
        sh.range_search_device(nq, q.data_ptr(), radius, mr, od.data_ptr(), oi.data_ptr(), oc.data_ptr(), stream=st.cuda_stream, sp=sp)
    st.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(st)
    for _ in range(steps):
        sh.range_search_device(nq, q.data_ptr(), radius, mr, od.data_ptr(), oi.data_ptr(), oc.data_ptr(), stream=st.cuda_stream, sp=sp)
    e1.record(st)
    st.synchronize()
    dev_ms = e0.elapsed_time(e1) / steps
    t = time.perf_counter()
    for _ in range(steps):
        hs = sh.range_search(xq, radius, mr, nprobe=nprobe)
    e2e_ms = (time.perf_counter() - t) / steps * 1e3
    plain = ix.range_search(xq, radius, mr, nprobe=nprobe)
    dev_res = (od.cpu().numpy(), oi.cpu().numpy(), oc.cpu().numpy())
    lines["shard_world1"] = {"ms_per_batch_device": dev_ms, "qps_device": nq / dev_ms * 1e3, "ms_per_batch_e2e": e2e_ms,
                             "qps_e2e": nq / e2e_ms * 1e3, "equal_plain_host": same(hs, plain), "equal_plain_device": same(dev_res, plain)}
    sh.close()
    return {"config": "range IVF-Flat L2 1Mx768 nlist=1024 nprobe=32 batch=1024 max_results=1024", "card": card(),
            "radius": radius, **lines}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", default="1,2,3,4")
    ap.add_argument("--pq-n", type=int, default=10_000_000)
    ap.add_argument("--pq-nbits", type=int, default=8, help="cfg3: bits per PQ code, 1-8")
    ap.add_argument("--pq-m", type=int, default=96, help="cfg3: sub-quantisers (768 must divide by it)")
    ap.add_argument("--hnsw-n", type=int, default=1_000_000)
    ap.add_argument("--hnsw-build-threads", type=int, default=64)
    ap.add_argument("--hnsw-build", choices=("host", "device"), default="host", help="cfg4: graph built by host writers or on the device")
    ap.add_argument("--hnsw-build-batch", type=int, default=0, help="cfg4 --hnsw-build device: rows per batch (0 = library default)")
    ap.add_argument("--cfg5-rows", type=int, default=6_250_000, help="cfg5: database rows per GPU (6.25 M x 1536 f32 = 38 GB of an 80 GB H100)")
    ap.add_argument("--cfg5-batch", type=int, default=4096)
    ap.add_argument("--cfg5-steps", type=int, default=10)
    ap.add_argument("--bin-n", type=int, default=10_000_000, help="cfg7: database rows")
    ap.add_argument("--bin-dim", type=int, default=512, help="cfg7: bits per row (multiple of 8)")
    ap.add_argument("--exact-only", action="store_true", help="cfg6 / cfg7: search with exact_only (the query-major exact scan)")
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    global EXACT_ONLY
    EXACT_ONLY = a.exact_only
    o = oracle_lib.load()
    cores = os.cpu_count() or 1
    fns = {"1": lambda: cfg1(o, cores), "2": lambda: cfg2(o, cores), "3": lambda: cfg3(o, cores, a.pq_n, a.pq_nbits, a.pq_m), "4": lambda: cfg4(o, cores, a.hnsw_n, a.hnsw_build_threads, a.hnsw_build, a.hnsw_build_batch),
           "calc": lambda: cfg_calc(o, cores), "brute": lambda: cfg_brute(o, cores),
           "3s": lambda: cfg3s(o, cores, a.pq_n, a.pq_nbits, a.pq_m),
           "1s": lambda: cfg1s(o, cores), "4s": lambda: cfg4s(o, cores, a.hnsw_n),
           "5": lambda: cfg5(o, cores, a.cfg5_rows, steps=a.cfg5_steps, nq=a.cfg5_batch),
           "6": lambda: cfg6(o, cores), "6s": lambda: cfg6s(o, cores), "7": lambda: cfg7(o, cores, a.bin_n, a.bin_dim),
           "range": lambda: cfg_range(o, cores)}
    rank = int(os.environ.get("RANK", 0))
    for c in a.configs.split(","):
        t0 = time.time()
        try:
            line = fns[c]()
        except Exception as e:  # keep going: one line per config
            import traceback
            line = {"config": f"cfg{c}", "error": repr(e), "traceback": traceback.format_exc()[-1500:]}
        if line is None or rank != 0:  # multi-rank configs: rank 0 prints
            continue
        line["wall_seconds"] = time.time() - t0
        s = json.dumps(line)
        print(s, flush=True)
        if a.out:
            with open(a.out, "a") as f:
                f.write(s + "\n")


if __name__ == "__main__":
    main()
