"""Thread harness of the loopback shard tests (tests/test_gpu_shard_loopback.py).

A sharded index of W ranks runs as W Python threads of one process on one GPU: each thread builds its own b200vs.Index on
device 0 and its b200vs.Shard, and the ranks' collectives go through tests/nccl_loopback/libnccl_loopback.so, an NCCL
stand-in whose ranks are threads (real NCCL refuses two ranks on one device).  ctypes releases the GIL for every call, so a
rank blocked in a rendezvous does not hold up the others.  Test-side exchange is plain shared state and a Barrier.

The library is chosen once per process (B200VS_NCCL_LIB is read by the first NCCL call), so every case runs in a subprocess
of its own: run_case(case, *args) starts `python tests/shard_loopback.py <case> <json args>`, which imports
test_gpu_shard_loopback, calls its function `case` and exits.  The subprocess has a timeout and a faulthandler dump before
it, and it exits with os._exit, so no thread or process is left behind."""
import faulthandler
import json
import os
import subprocess
import sys
import threading

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
LIB = os.path.join(HERE, "nccl_loopback", "libnccl_loopback.so")
CASE_TIMEOUT = 300  # seconds of one subprocess; every rendezvous of the library times out after 60 s


class World:
    """What the W rank threads of one run share: communicator ids, a barrier, and all-gather of Python values."""

    def __init__(self, W):
        self.W = W
        self.barrier = threading.Barrier(W, timeout=150)
        self._lock = threading.Lock()
        self._ids = {}
        self._slots = {}
        self._calls = [0] * W
        self._gathers = [0] * W

    def connect(self, ix, rank, lanes=2):
        """b200vs.Shard of rank `rank` over a fresh communicator: the c-th connect of every rank shares one id."""
        import b200vs
        c = self._calls[rank]
        self._calls[rank] += 1
        with self._lock:
            if c not in self._ids:
                self._ids[c] = b200vs.Shard.unique_id()
            idb = self._ids[c]
        return b200vs.Shard(ix, rank, self.W, idb, lanes=lanes)

    def gather(self, rank, value):
        """Every rank's `value`, in rank order (collective over the rank threads)."""
        c = self._gathers[rank]
        self._gathers[rank] += 1
        with self._lock:
            self._slots.setdefault(c, [None] * self.W)[rank] = value
        self.barrier.wait()
        out = list(self._slots[c])
        self.barrier.wait()
        return out


def run_world(W, fn):
    """fn(rank, world) on W threads; returns every rank's result, or re-raises the first exception (rank order)."""
    world = World(W)
    res, err = [None] * W, [None] * W

    def body(r):
        try:
            res[r] = fn(r, world)
        except BaseException as e:  # noqa: B036 - re-raised below
            err[r] = e
            world.barrier.abort()  # peers waiting in the barrier fail at once instead of timing out

    ths = [threading.Thread(target=body, args=(r,), daemon=True, name=f"rank{r}") for r in range(W)]
    for t in ths:
        t.start()
    for t in ths:
        t.join()
    first = next((e for e in err if e is not None and not isinstance(e, threading.BrokenBarrierError)), None)
    first = first or next((e for e in err if e is not None), None)
    if first is not None:
        raise first
    return res


def run_case(case, *args, timeout=CASE_TIMEOUT):
    """Runs test_gpu_shard_loopback.<case>(*args) in a subprocess on the loopback library; returns its output, and fails
    the calling test with that output if the case failed."""
    assert os.path.exists(LIB), f"{LIB} not built (build() runs make -C tests/nccl_loopback)"
    env = dict(os.environ, B200VS_NCCL_LIB=LIB)
    cmd = [sys.executable, os.path.abspath(__file__), case, json.dumps(list(args)), str(timeout - 20)]
    try:
        p = subprocess.run(cmd, env=env, cwd=ROOT, capture_output=True, text=True, timeout=timeout)
    except subprocess.TimeoutExpired as e:  # run() has killed the child
        raise AssertionError(f"{case}{args}: no result within {timeout} s\n{e.stdout or ''}\n{e.stderr or ''}")
    out = p.stdout + p.stderr
    if p.returncode != 0 or "LOOPBACK CASE OK" not in p.stdout:
        raise AssertionError(f"{case}{args} failed (exit {p.returncode}):\n{out[-6000:]}")
    return out


def _main():
    case, args, dump_after = sys.argv[1], json.loads(sys.argv[2]), int(sys.argv[3])
    faulthandler.dump_traceback_later(dump_after, exit=True)
    sys.path.insert(0, os.path.join(ROOT, "dingo-store_b200", "python"))
    sys.path.insert(0, HERE)
    rc = 1
    try:
        import test_gpu_shard_loopback as cases
        getattr(cases, case)(*args)
        print("LOOPBACK CASE OK", flush=True)
        rc = 0
    except BaseException:
        import traceback
        traceback.print_exc()
    finally:
        faulthandler.cancel_dump_traceback_later()
        sys.stdout.flush()
        sys.stderr.flush()
        os._exit(rc)  # daemon rank threads never outlive the case


if __name__ == "__main__":
    _main()
