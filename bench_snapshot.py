"""Fork-based snapshots: how long the snapshot path holds the write lock (b200vs_save_stage) against the export b200vs_save
runs today (b200vs_export_lists: one synchronous copy per inverted list), and how fast the forked child writes the file
(b200vs_save_staged).  The staged image is checked byte-equal to b200vs_save's file before anything is timed.

Workloads:
  ivf_1m      IVF-Flat L2, 1 M x 768, nlist 1024 (the headline index of bench.py).
  ivf_region  IVF-Flat L2, 170 k x 768, nlist 1024: a region at the 512 MB auto-split size (SURVEY §5).
  ivf_pq      IVF-PQ L2, 500 k x 128, nlist 1024, 16 sub-vectors of 8 bits.
  hnsw        HNSW L2, 100 k x 128, m 16 (built with b200vs_hnsw_add_batched): its graph is host-side, so the stage is host
              copies only.
One tenth of each index's rows is tombstoned.

Per workload and repetition:
  stage_host_s   host clock around b200vs_save_stage (it ends in a stream synchronise): the write-lock window.
  stage_dev_ms   device time of the stage's pack kernels and device-to-host copies, from torch.profiler (one profiled run).
  export_s       host clock around b200vs_export_lists into preallocated host arrays (b200vs_save's export step).
  save_s         host clock around a whole b200vs_save to a file, for context.
  write_GBps     the staged image's bytes over the host clock of b200vs_save_staged in a forked child, fork to reap.
Files go to a temporary directory (--dir) and are deleted after each write.  Prints one JSON line per workload with the GPU
name and power limit.
"""
import argparse
import json
import os
import shutil
import signal
import subprocess
import sys
import tempfile
import time
import warnings

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(ROOT, "dingo-store_b200", "python"))
import b200vs  # noqa: E402

WORKLOADS = {
    "ivf_1m": dict(kind=b200vs.IVF_FLAT, n=1_000_000, d=768, kw=dict(nlist=1024)),
    "ivf_region": dict(kind=b200vs.IVF_FLAT, n=170_000, d=768, kw=dict(nlist=1024)),
    "ivf_pq": dict(kind=b200vs.IVF_PQ, n=500_000, d=128, kw=dict(nlist=1024, pq_m=16, pq_nbits=8)),
    "hnsw": dict(kind=b200vs.HNSW, n=100_000, d=128, kw=dict(hnsw_m=16, hnsw_efc=64, max_elements=200_000)),
}


def gpu_info():
    try:
        out = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], text=True)
        name, power = [s.strip() for s in out.splitlines()[0].split(",")]
        return name, power
    except Exception as e:  # the numbers are still printed, marked with what is known
        return f"unknown ({e})", "unknown"


def build(w):
    rng = np.random.default_rng(0)
    x = rng.standard_normal((w["n"], w["d"]), dtype=np.float32)
    ids = np.arange(w["n"], dtype=np.int64)
    ix = b200vs.Index(w["kind"], b200vs.L2, w["d"], **w["kw"])
    if w["kind"] == b200vs.HNSW:
        ix.add_batched(x, ids)
    else:
        ix.train(x)
        ix.add(x, ids)
    ix.delete(ids[::10])
    return ix


def same_file(a, b):
    with open(a, "rb") as fa, open(b, "rb") as fb:
        while True:
            ba, bb = fa.read(1 << 24), fb.read(1 << 24)
            if ba != bb:
                return False
            if not ba:
                return True


def forked_write_s(ix, path, timeout_s=600):
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", DeprecationWarning)
        t0 = time.perf_counter()
        pid = os.fork()
    if pid == 0:
        code = 1
        try:
            ix.save_staged(path)
            code = 0
        finally:
            os._exit(code)
    deadline = time.monotonic() + timeout_s
    while time.monotonic() < deadline:
        got, status = os.waitpid(pid, os.WNOHANG)
        if got == pid:
            dt = time.perf_counter() - t0
            if os.waitstatus_to_exitcode(status) != 0:
                raise RuntimeError("the child's staged write failed")
            return dt
        time.sleep(0.001)
    os.kill(pid, signal.SIGKILL)
    os.waitpid(pid, 0)
    raise RuntimeError("the child's staged write timed out")


def stage_device_ms(ix):
    """Device time of one stage's kernels and copies (torch.profiler, CUDA activities)."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        ix.save_stage()
        torch.cuda.synchronize()
    ix.save_unstage()
    total = 0.0
    for e in prof.events():
        if e.device_type.name == "CUDA" and ("pack_rows_kernel" in e.name or "Memcpy" in e.name):
            total += e.device_time_total if hasattr(e, "device_time_total") else e.cuda_time_total
    return total / 1e3


def run(name, w, reps, tmp):
    ix = build(w)
    nlist = w["kw"].get("nlist", 1)
    ref, staged = os.path.join(tmp, "ref"), os.path.join(tmp, "staged")
    ix.save(ref)
    ix.save_stage()
    ix.save_staged(staged)
    ix.save_unstage()
    if not same_file(ref, staged):
        raise RuntimeError(f"{name}: the staged image differs from b200vs_save's file")
    nbytes = os.path.getsize(ref)
    os.remove(ref), os.remove(staged)
    code_size = (w["kw"]["pq_m"] * w["kw"]["pq_nbits"] + 7) // 8 if w["kind"] == b200vs.IVF_PQ else 0
    out = dict(workload=name, rows=w["n"], dim=w["d"], live=ix.get_count(), file_bytes=nbytes, reps=reps,
               stage_host_s=[], export_s=[], save_s=[], write_GBps=[])
    for _ in range(reps):
        t0 = time.perf_counter()
        ix.save_stage()
        out["stage_host_s"].append(round(time.perf_counter() - t0, 4))
        out["write_GBps"].append(round(nbytes / forked_write_s(ix, staged) / 1e9, 3))
        ix.save_unstage()
        os.remove(staged)
        if w["kind"] != b200vs.HNSW:
            t0 = time.perf_counter()
            ix.export_lists(nlist, with_vectors=w["kind"] != b200vs.IVF_PQ, code_size=code_size)
            out["export_s"].append(round(time.perf_counter() - t0, 4))
        t0 = time.perf_counter()
        ix.save(ref)
        out["save_s"].append(round(time.perf_counter() - t0, 4))
        os.remove(ref)
    out["stage_dev_ms"] = round(stage_device_ms(ix), 3)
    ix.close()
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--workloads", default=",".join(WORKLOADS), help="comma-separated subset of " + ", ".join(WORKLOADS))
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--dir", default=None, help="directory for the snapshot files (default: a new temporary directory)")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("bench_snapshot.py needs a CUDA device")
    name, power = gpu_info()
    tmp = tempfile.mkdtemp(prefix="b2vs_snap_", dir=args.dir)
    try:
        for wl in args.workloads.split(","):
            res = run(wl, WORKLOADS[wl], args.reps, tmp)
            res.update(gpu=name, power_limit=power)
            print(json.dumps(res), flush=True)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


if __name__ == "__main__":
    main()
