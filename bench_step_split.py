#!/usr/bin/env python
"""bench_step_split.py — what one IVF-Flat search step is made of, at bench.py's headline shape.

Builds the same index and query batches as bench.py (same seeds), then measures on one GPU:
  * the step: K batches with `in_flight` batches in flight on as many streams, and the same K batches back to back on one
    stream (CUDA events, as bench.py times `value` and `single_stream`), repeated `--reps` times;
  * each tile pass on its own: the coarse scan, sample and capture launches of the tile kernel (in that order in every
    search), timed by torch.profiler's CUDA activity trace over `--profiled` searches run one at a time on an idle GPU,
    beside the library's own phase profile (`phase_ms`, CUDA events at phase boundaries);
  * the additive model step ~ capture + sample + coarse scan: these three passes each take every SM's shared memory, so
    no other lane's pass can run beside them.
It also derives, from the shapes, each short pass's MMA floor and the bytes it moves (HBM / L2) against the H100 SXM data
sheet.  Prints one JSON line; `--out DIR` also writes it to DIR/step_split.json.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(ROOT, "dingo-store_b200", "python"))

# H100 SXM data sheet, dense: FP16 989 TFLOP/s, TF32 495 TFLOP/s, HBM3 3.35 TB/s
PEAK_FP16, PEAK_TF32, PEAK_HBM = 989e12, 495e12, 3.35e12

# tile geometry (csrc/tc_scan.cuh, TcCfg and tc_dense_scan in csrc/tc_scan.cu)
TC_NQT, TC_CHUNK, TC_SPAN, TC_SAMPLE = 128, 512, 2048, 32
DENSE_BM, DENSE_NQT, DENSE_CTAS = 64, 64, 3


def cdiv(a, b):
    return -(-a // b)


def ncols(nq):  # the wgmma N a group of nq queries is padded to
    return 16 if nq <= 16 else 32 if nq <= 32 else 64 if nq <= 64 else 128


def coarse_model(nrows, nq, d, sms, tile=DENSE_BM, max_w=DENSE_NQT, slots_per_sm=DENSE_CTAS):
    """The coarse split pass (hi*hi + lo*hi + hi*lo, TF32): items by tc_dense_scan's width rule, the MMA floor, and the
    hi / lo tile bytes every item reads from L2 (the table and the queries each fit in L2)."""
    chunk = tile if nrows <= 16384 else TC_CHUNK
    best, w_best, w = None, max_w, max_w
    while w >= 16:
        cost = cdiv(cdiv(nrows, chunk) * cdiv(nq, w), sms * slots_per_sm) * (tile + w)
        if best is None or cost < best:
            best, w_best = cost, w
        w //= 2
    items = cdiv(nrows, chunk) * cdiv(nq, w_best)
    kblocks = cdiv(d, 32)
    tiles = cdiv(nrows, tile) * cdiv(nq, w_best)
    l2 = tiles * kblocks * 2 * (tile * 128 + w_best * 128)  # hi and lo stages: A tile + B tile of 128 B rows each
    flops = 3 * 2 * cdiv(nrows, tile) * tile * cdiv(nq, w_best) * w_best * d
    return {"tile_rows": tile, "group": w_best, "items": items, "l2_bytes": l2, "mma_flops": flops,
            "mma_floor_us": flops / PEAK_TF32 * 1e6, "hbm_bytes": 2 * nrows * d * 4 + 2 * nq * d * 4}


def sample_model(probes, list_len, d):
    """The sample pass at this probe table: one sampled item per (query group, 2048-row span) of every probed list; each
    scores its first 32 rows (A: FP16 rows, first read from HBM) against its group's padded B tile (FP16 queries, L2)."""
    cnt = np.bincount(probes[probes >= 0].ravel(), minlength=len(list_len))
    items = a_bytes = b_bytes = flops = 0
    for c, ln in zip(cnt, list_len):
        if c <= 0 or ln <= 0:
            continue
        spans = cdiv(int(ln), TC_SPAN)
        for g in range(cdiv(int(c), TC_NQT)):
            n = ncols(min(TC_NQT, int(c) - g * TC_NQT))
            items += spans
            a_bytes += spans * TC_SAMPLE * d * 2
            b_bytes += spans * n * d * 2
            flops += spans * 2 * 64 * n * d  # the M = 64 wgmma also multiplies the 32 rows after the box
    return {"items": int(items), "hbm_bytes": int(a_bytes), "l2_bytes": int(b_bytes), "mma_flops": int(flops),
            "mma_floor_us": flops / PEAK_FP16 * 1e6, "hbm_floor_us": a_bytes / PEAK_HBM * 1e6}


def stats(xs):
    xs = sorted(xs)
    return {"min": xs[0], "median": float(np.median(xs)), "max": xs[-1], "n": len(xs)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--nb", type=int, default=1_000_000)
    ap.add_argument("--dim", type=int, default=768)
    ap.add_argument("--nlist", type=int, default=1024)
    ap.add_argument("--nprobe", type=int, default=32)
    ap.add_argument("--batch", type=int, default=1024)
    ap.add_argument("--k", type=int, default=10)
    ap.add_argument("--in-flight", type=int, default=8)
    ap.add_argument("--steps", type=int, default=20, help="batches per timed step window")
    ap.add_argument("--reps", type=int, default=5, help="timed windows per measurement")
    ap.add_argument("--profiled", type=int, default=20, help="searches traced for the per-pass kernel times")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    import torch
    import b200vs
    from bench import gen_chunks

    assert torch.cuda.is_available(), "bench_step_split.py needs a CUDA device"
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    card = {"name": torch.cuda.get_device_name(dev)}
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        card["power_limit, clocks.max.sm"] = q
    except Exception as e:  # read-only query; the numbers stay valid without it
        card["power_limit, clocks.max.sm"] = f"unavailable ({e})"

    n, d, nlist, k, L = args.nb, args.dim, args.nlist, args.k, max(1, args.in_flight)
    ix = b200vs.Index(b200vs.IVF_FLAT, b200vs.L2, d, nlist=nlist, device=0)
    chunks = [(a, x.cpu().numpy()) for a, x in gen_chunks(torch, n, d, 1234, dev)]
    ix.train(np.concatenate([c for _, c in chunks], 0)[:min(n, nlist * 256)])
    for a, x in chunks:
        for b in range(0, x.shape[0], 32768):
            ix.add(x[b:b + 32768], np.arange(a + b + 1, a + b + 1 + min(32768, x.shape[0] - b), dtype=np.int64))
    del chunks

    gq = torch.Generator(device=dev)
    gq.manual_seed(4321)
    nq = args.batch
    q_dev = [torch.rand((nq, d), generator=gq, device=dev, dtype=torch.float32) for _ in range(4)]
    out_d = [torch.empty((nq, k), dtype=torch.float32, device=dev) for _ in range(L)]
    out_i = [torch.empty((nq, k), dtype=torch.int64, device=dev) for _ in range(L)]
    sp, _keep = b200vs.make_search_params(nprobe=args.nprobe)
    main_stream = torch.cuda.Stream(device=dev)
    streams = [torch.cuda.Stream(device=dev) for _ in range(L)]
    torch.cuda.set_stream(main_stream)

    def step(i, lanes):
        ln = i % lanes
        ix.search_device(nq, q_dev[i % 4].data_ptr(), k, out_d[ln].data_ptr(), out_i[ln].data_ptr(),
                         stream=streams[ln].cuda_stream, sp=sp)

    def timed(steps, lanes):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(main_stream)
        for st in streams[:lanes]:
            st.wait_event(e0)
        for i in range(steps):
            step(i, lanes)
        for st in streams[:lanes]:
            ev = torch.cuda.Event()
            ev.record(st)
            main_stream.wait_event(ev)
        e1.record(main_stream)
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / steps * 1e3  # us per batch

    for i in range(max(5, 2 * L)):  # every lane twice: a lane's first search sizes its scratch arena
        step(i, L)
    torch.cuda.synchronize()
    inflight, single = [], []
    for _ in range(args.reps):  # alternate, so drifting clocks touch both alike
        inflight.append(timed(args.steps, L))
        single.append(timed(args.steps, 1))

    # per-pass kernel times, one search at a time
    from torch.profiler import profile, ProfilerActivity
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for i in range(args.profiled):
            step(i, 1)
            torch.cuda.synchronize()
    evs = sorted((e for e in prof.events() if e.device_type.name == "CUDA"), key=lambda e: e.time_range.start)
    tile = [e for e in evs if "tc_scan_kernel" in e.name]
    passes = {"coarse_scan": [], "sample": [], "capture": []}
    per_search = len(tile) // max(1, args.profiled)
    if per_search == 3 and len(tile) == 3 * args.profiled:
        for j, e in enumerate(tile):
            passes[("coarse_scan", "sample", "capture")[j % 3]].append(e.time_range.elapsed_us())
    kernels = {}
    for e in evs:
        kernels.setdefault(e.name.split("(")[0][:90], []).append(e.time_range.elapsed_us())
    kernels = {name: round(sum(v) / args.profiled, 2) for name, v in kernels.items()}
    busy_us = sum(kernels.values())

    ix.set_profiling(True)
    phases = []
    for i in range(args.profiled):
        step(i, 1)
        torch.cuda.synchronize()
        phases.append({a: v * 1e3 for a, v in ix.phase_times().items() if v > 0})
    ix.set_profiling(False)
    phase_us = {a: stats([p.get(a, 0.0) for p in phases]) for a in phases[0]}

    # shapes: the probe table of batch 0 and the list lengths
    probes = torch.empty((nq, args.nprobe), dtype=torch.int64, device=dev)
    score = torch.empty((nq, args.nprobe), dtype=torch.float32, device=dev)
    ix.coarse_device(nq, q_dev[0].data_ptr(), args.nprobe, 0, nlist, score.data_ptr(), probes.data_ptr(),
                     stream=main_stream.cuda_stream)
    torch.cuda.synchronize()
    off = ix.export_lists(nlist, with_vectors=False)[0]
    list_len = np.diff(off)
    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    coarse = coarse_model(nlist, nq, d, sms)
    sample = sample_model(probes.cpu().numpy(), list_len, d)
    probed = np.unique(probes.cpu().numpy())
    capture_hbm = int(list_len[probed].sum()) * (2 * d + 16)  # FP16 row + scale + norm + id

    med = {a: float(np.median(v)) if v else None for a, v in passes.items()}
    model = None
    if all(med.values()):
        model = {"capture+sample+coarse_us": med["capture"] + med["sample"] + med["coarse_scan"],
                 "in_flight_step_us": float(np.median(inflight)),
                 "ratio": float(np.median(inflight)) / (med["capture"] + med["sample"] + med["coarse_scan"])}
    if med["coarse_scan"]:
        coarse["achieved_l2_tbs"] = coarse["l2_bytes"] / med["coarse_scan"] / 1e6
        coarse["mma_floor_frac"] = coarse["mma_floor_us"] / med["coarse_scan"]
    if med["sample"]:
        sample["mma_floor_frac"] = sample["mma_floor_us"] / med["sample"]
        sample["hbm_floor_frac"] = sample["hbm_floor_us"] / med["sample"]
        sample["achieved_l2_tbs"] = sample["l2_bytes"] / med["sample"] / 1e6
    if med["capture"]:
        capture = {"hbm_bytes": capture_hbm, "achieved_hbm_tbs": capture_hbm / med["capture"] / 1e6,
                   "hbm_floor_frac": capture_hbm / PEAK_HBM * 1e6 / med["capture"]}
    else:
        capture = {"hbm_bytes": capture_hbm}

    line = {"card": card, "shape": {"nb": n, "dim": d, "nlist": nlist, "nprobe": args.nprobe, "batch": nq, "k": k, "in_flight": L},
            "step_us": {"in_flight": stats(inflight), "single_stream": stats(single)},
            "pass_us": {a: stats(v) if v else None for a, v in passes.items()},
            "model": model, "kernel_us_per_search": kernels, "kernel_busy_us_per_search": round(busy_us, 1),
            "phase_us": phase_us, "coarse": coarse, "sample": sample, "capture": capture}
    s = json.dumps(line)
    print(s, flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "step_split.json"), "w") as f:
            f.write(s + "\n")


if __name__ == "__main__":
    main()
