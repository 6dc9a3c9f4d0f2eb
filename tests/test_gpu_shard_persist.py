"""Snapshots of sharded indexes: b200vs_shard_save and b200vs_shard_load at world > 1 on one GPU.

The ranks run as threads of one process over the loopback NCCL (tests/shard_loopback.py: World, run_world).  Each case runs
in a subprocess of its own, started by run() below through this file's own __main__ (the library is chosen once per
process).  Three groups:
  1. same-world round trips, W in {1, 2, 3, 5, 8}, for every shard kind: every read after the reload is bit-identical to the
     same read before the save, every rank's exports and trained state are byte-equal to the saved rank's, and a delete and
     an upsert after the reload keep the index equal to a twin that was never saved;
  2. restores onto another number of ranks (FLAT, IVF_FLAT, IVF_PQ): results bit-identical to one unsharded index of the
     same rows and trained state, row counts by the owner rule, IVF-PQ codes unchanged per id;
  3. refusals: every rank returns the same status, every index is left empty and a later correct load succeeds."""
import faulthandler
import json
import os
import shutil
import subprocess
import sys
import tempfile

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
if __name__ == "__main__":
    sys.path.insert(0, os.path.join(os.path.dirname(HERE), "dingo-store_b200", "python"))
    sys.path.insert(0, HERE)

import b200vs  # noqa: E402
from b200vs import COSINE, FLAT, HNSW, IP, IVF_FLAT, IVF_PQ, L2  # noqa: E402
from b200vs import shard as shard_py  # noqa: E402
from gpu_util import require_gpu  # noqa: E402
from shard_loopback import CASE_TIMEOUT, LIB, ROOT, run_world  # noqa: E402

pytestmark = pytest.mark.gpu
WORLDS = (1, 2, 3, 5, 8)
D = 16


@pytest.fixture(autouse=True)
def _gpu():
    require_gpu()


def run(case, *args, timeout=CASE_TIMEOUT):
    """this_module.<case>(*args) in a subprocess on the loopback library (as shard_loopback.run_case)."""
    assert os.path.exists(LIB), f"{LIB} not built (build() runs make -C tests/nccl_loopback)"
    env = dict(os.environ, B200VS_NCCL_LIB=LIB)
    cmd = [sys.executable, os.path.abspath(__file__), case, json.dumps(list(args)), str(timeout - 20)]
    try:
        p = subprocess.run(cmd, env=env, cwd=ROOT, capture_output=True, text=True, timeout=timeout)
    except subprocess.TimeoutExpired as e:
        raise AssertionError(f"{case}{args}: no result within {timeout} s\n{e.stdout or ''}\n{e.stderr or ''}")
    out = p.stdout + p.stderr
    if p.returncode != 0 or "PERSIST CASE OK" not in p.stdout:
        raise AssertionError(f"{case}{args} failed (exit {p.returncode}):\n{out[-6000:]}")


def _same(got, want, what):
    for x, y in zip(got, want):
        x, y = np.asarray(x), np.asarray(y)
        assert x.shape == y.shape, f"{what}: shape {x.shape} != {y.shape}"
        if x.dtype == np.float32:
            x, y = x.view(np.uint32), y.view(np.uint32)
        bad = np.argwhere(x != y)
        assert bad.size == 0, f"{what}: differs at {bad[:4].tolist()}"


def _status(fn):
    try:
        fn()
        return b200vs.OK
    except b200vs.B200VSError as e:
        return e.code


# ---------------------------------------------------------------------------------------------
# index kinds: (type, metric, creation parameters, trained state)
# ---------------------------------------------------------------------------------------------
KINDS = {
    "flat_l2": (FLAT, L2, {}), "flat_ip": (FLAT, IP, {}), "flat_cos": (FLAT, COSINE, {}),
    "ivf_l2": (IVF_FLAT, L2, {"nlist": "uneven"}), "ivf_cos": (IVF_FLAT, COSINE, {"nlist": "few"}),
    "pq8_l2": (IVF_PQ, L2, {"nlist": "uneven", "pq_m": 4, "pq_nbits": 8}),
    "pq4_ip": (IVF_PQ, IP, {"nlist": "uneven", "pq_m": 4, "pq_nbits": 4}),
    "hnsw_l2": (HNSW, L2, {"hnsw_m": 8, "hnsw_efc": 40, "max_elements": 4000}),
    "hnsw_cos": (HNSW, COSINE, {"hnsw_m": 8, "hnsw_efc": 40, "max_elements": 4000}),
}


class Kind:
    def __init__(self, name, W, seed=0, nlist=None):
        t, m, kw = KINDS[name]
        self.name, self.type, self.metric = name, t, m
        kw = dict(kw)
        if "nlist" in kw:
            kw["nlist"] = nlist or (2 * W + 1 if kw["nlist"] == "uneven" else 3)
        self.kw = kw
        self.nlist = kw.get("nlist", 1)
        rng = np.random.default_rng(1000 * W + 17 * seed + len(name))
        self.rng = rng
        self.blob = None
        if t in (IVF_FLAT, IVF_PQ):
            cent = rng.standard_normal((self.nlist, D)).astype(np.float32)
            if t == IVF_PQ:
                nb = kw["pq_nbits"]
                self.blob = b200vs.ivfpq_state_blob(cent, rng.standard_normal((4, 1 << nb, D // 4)).astype(np.float32), m)
            else:
                self.blob = b200vs.ivf_state_blob(cent, m)
        self.code_size = (kw["pq_m"] * kw["pq_nbits"] + 7) // 8 if t == IVF_PQ else 0

    def index(self, trained=True):
        ix = b200vs.Index(self.type, self.metric, D, **self.kw)
        if trained and self.blob is not None:
            ix.set_trained_state(self.blob)
        return ix

    def exports(self, ix):
        off, vec, codes, ids = ix.export_lists(max(self.nlist, 1), with_vectors=self.type != IVF_PQ, code_size=self.code_size)
        return [off, ids] + [a for a in (vec, codes) if a is not None] + [np.frombuffer(bytes(ix.get_trained_state()), np.uint8)]


def _rows(W, n_per, seed):
    rng = np.random.default_rng(seed)
    xs = [rng.standard_normal((n_per + 37 * r, D)).astype(np.float32) for r in range(W)]
    ids = [np.arange(len(x), dtype=np.int64) * W + r + 1 for r, x in enumerate(xs)]
    return xs, ids, rng.standard_normal((24, D)).astype(np.float32)


def _reads(kind, sh, xq, seq):
    """every read of a sharded index that applies to its kind: host and device top-k, filtered top-k, range"""
    import torch
    nprobe = min(kind.nlist, 5)
    kw = dict(nprobe=nprobe) if kind.type in (IVF_FLAT, IVF_PQ) else {}
    out = {}
    for k in (1, 10):
        out[("topk", k)] = sh.search(xq, k, seq=seq, **kw); seq += 1
    out["filter"] = sh.search(xq, 10, seq=seq, id_range=(3, 300), **kw); seq += 1
    out["ids"] = sh.search(xq, 10, seq=seq, sorted_ids=np.arange(1, 900, 3), **kw); seq += 1
    qd = torch.from_numpy(xq).cuda()
    od = torch.empty((len(xq), 10), dtype=torch.float32, device="cuda:0")
    oi = torch.empty((len(xq), 10), dtype=torch.int64, device="cuda:0")
    sp, _keep = b200vs.make_search_params(**kw)
    torch.cuda.synchronize()
    sh.search_device(len(xq), qd.data_ptr(), 10, od.data_ptr(), oi.data_ptr(), sp=sp, seq=seq); seq += 1
    torch.cuda.synchronize()
    out["device"] = (od.cpu().numpy(), oi.cpu().numpy())
    if kind.type != HNSW:
        out["range"] = sh.range_search(xq, 30.0 if kind.metric == L2 else 0.5, 64, seq=seq, **kw); seq += 1
    return out, seq


# ---------------------------------------------------------------------------------------------
# 1. same-world round trips
# ---------------------------------------------------------------------------------------------
def case_round_trip(name):
    for W in WORLDS:
        try:
            _round_trip(name, W)
        except AssertionError as e:
            raise AssertionError(f"world {W}: {e}") from e


def _round_trip(name, W):
    kind = Kind(name, W)
    xs, ids, xq = _rows(W, 150, W)
    tmp = tempfile.mkdtemp(prefix="b2vs_persist_")
    prefix = os.path.join(tmp, "snap")
    up_id = ids[0][0] if len(ids[0]) else 1
    up_x = np.full((1, D), 0.25, np.float32)

    def rank(r, world):
        def build():
            ix = kind.index()
            sh = world.connect(ix, r)
            sh.add(xs[r], ids[r])
            return ix, sh
        ix, sh = build()
        before, _ = _reads(kind, sh, xq, 0)
        saved = kind.exports(ix)
        sh.save(prefix)
        sh.close(); ix.close()
        ix2 = kind.index(trained=False)
        sh2 = world.connect(ix2, r)
        sh2.load(prefix)
        after, seq2 = _reads(kind, sh2, xq, 0)
        restored = kind.exports(ix2)
        file_ok = os.path.exists(f"{prefix}.{r}-of-{W}")
        # delete, then upsert (delete + add), on the restored index and on a twin that was never saved
        twin, sht = build()
        edits = {}
        for tag, s_, x_, seq in (("restored", sh2, ix2, seq2), ("twin", sht, twin, 0)):
            s_.delete(np.array([ids[0][1] if len(ids[0]) > 1 else 2, 10 ** 9], np.int64))
            s_.delete(np.array([up_id], np.int64))
            s_.add(up_x if r == 0 else np.zeros((0, D), np.float32), np.array([up_id] if r == 0 else [], np.int64))
            res, _ = _reads(kind, s_, xq, seq)
            edits[tag] = (res, kind.exports(x_)[:-1] if kind.type != HNSW else [x_.get_count()])
        sh2.close(); sht.close(); ix2.close(); twin.close()
        return before, after, saved, restored, file_ok, edits

    try:
        res = run_world(W, rank)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    for r, (before, after, saved, restored, file_ok, edits) in enumerate(res):
        assert file_ok, f"rank {r}: no rank file"
        for key, want in before.items():
            _same(after[key], want, f"rank {r} {key} after reload")
        _same(restored, saved, f"rank {r} exports / trained state after reload")
        for key, want in edits["twin"][0].items():
            _same(edits["restored"][0][key], want, f"rank {r} {key} after delete + upsert")
        _same(edits["restored"][1], edits["twin"][1], f"rank {r} exports after delete + upsert")


@pytest.mark.parametrize("name", sorted(KINDS))
def test_round_trip(name):
    run("case_round_trip", name)


# ---------------------------------------------------------------------------------------------
# 2. another number of ranks
# ---------------------------------------------------------------------------------------------
PAIRS = ((2, 3), (3, 2), (5, 8), (8, 1), (1, 5))


def case_world_change(name):
    for W, W2 in PAIRS:
        try:
            _world_change(name, W, W2)
        except AssertionError as e:
            raise AssertionError(f"{W} -> {W2}: {e}") from e


def _world_change(name, W, W2):
    kind = Kind(name, W, nlist=7)
    xs, ids, xq = _rows(W, 120, 7 * W + W2)
    plain = kind.index()
    plain.add(np.concatenate(xs), np.concatenate(ids))
    want, _ = _reads(kind, _Plain(plain, kind), xq, 0)
    if kind.type == IVF_PQ:
        _, _, p_codes, p_ids = plain.export_lists(kind.nlist, with_vectors=False, code_size=kind.code_size)
        p_code = {int(i): bytes(c) for i, c in zip(p_ids, p_codes)}
    tmp = tempfile.mkdtemp(prefix="b2vs_persist_")
    prefix = os.path.join(tmp, "snap")

    def save_rank(r, world):
        ix = kind.index()
        sh = world.connect(ix, r)
        sh.add(xs[r], ids[r])
        sh.save(prefix)
        sh.close(); ix.close()

    def load_rank(r, world):
        ix = kind.index(trained=False)
        sh = world.connect(ix, r)
        sh.load(prefix)
        out, _ = _reads(kind, sh, xq, 0)
        _, _, codes, got_ids = ix.export_lists(kind.nlist, with_vectors=False, code_size=kind.code_size)
        rng = sh.list_range() if kind.type != FLAT else None
        sh.close()
        return out, got_ids, codes, rng

    try:
        run_world(W, save_rank)
        res = run_world(W2, load_rank)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    all_ids = np.concatenate(ids)
    seen = []
    for r, (out, got_ids, codes, rng) in enumerate(res):
        for key, w in want.items():
            _same(out[key], w, f"rank {r} {key}")
        if kind.type == FLAT:
            mine = all_ids[shard_py.row_owner(all_ids, W2) == r]
        else:
            p_off = plain.export_lists(kind.nlist, with_vectors=False, code_size=kind.code_size)
            mine = p_off[3][p_off[0][rng[0]]:p_off[0][rng[1]]]
        assert np.array_equal(np.sort(got_ids), np.sort(mine)), f"rank {r}: holds {len(got_ids)} rows, the owner rule gives {len(mine)}"
        if kind.type == IVF_PQ:
            for i, c in zip(got_ids, codes):
                assert bytes(c) == p_code[int(i)], f"rank {r}: id {i} changed its code"
        seen.append(got_ids)
    assert np.array_equal(np.sort(np.concatenate(seen)), np.sort(all_ids))


class _Plain:
    """the unsharded reference, read through the shard read signature"""

    def __init__(self, ix, kind):
        self.ix, self.kind = ix, kind

    def search(self, xq, k, seq=-1, **kw):
        return self.ix.search(xq, k, **kw)

    def range_search(self, xq, radius, max_results, seq=-1, **kw):
        return self.ix.range_search(xq, radius, max_results, **kw)

    def search_device(self, nq, xq_ptr, k, od, oi, sp=None, seq=-1):
        self.ix.search_device(nq, xq_ptr, k, od, oi, sp=sp)


@pytest.mark.parametrize("name", ("flat_cos", "ivf_cos", "pq8_l2"))
def test_world_change(name):
    run("case_world_change", name)


# ---------------------------------------------------------------------------------------------
# 3. refusals
# ---------------------------------------------------------------------------------------------
def _empty(ix, trained):
    return ix.get_count() == 0 and ix.get_deleted_count() == 0 and bool(ix.is_trained()) == trained


def case_refusals():
    W = 3
    tmp = tempfile.mkdtemp(prefix="b2vs_persist_")
    try:
        _refusals(W, tmp)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


def _refusals(W, tmp):
    kind = Kind("pq8_l2", W)
    other = Kind("pq8_l2", W, seed=5)  # another trained state
    xs, ids, xq = _rows(W, 300, 11)
    A, B = os.path.join(tmp, "a"), os.path.join(tmp, "b")
    files = [f"{A}.{r}-of-{W}" for r in range(W)] + [A + ".manifest"]

    def save(k, prefix):
        def rank(r, world):
            ix = k.index()
            sh = world.connect(ix, r)
            sh.add(xs[r], ids[r])
            sh.save(prefix)
            out, _ = _reads(k, sh, xq, 0)
            sh.close(); ix.close()
            return out
        return run_world(W, rank)[0]

    want = save(kind, A)
    save(other, B)
    good = {p: open(p, "rb").read() for p in files}

    def attempt(make, prefix=A, world=W, trained=False):
        """every rank's status of one load, each index checked empty afterwards"""
        def rank(r, wd):
            ix = make(r)
            sh = wd.connect(ix, r)
            st = _status(lambda: sh.load(prefix))
            ok = _empty(ix, trained) if st != b200vs.OK else True
            sh.close(); ix.close()
            return st, ok
        return run_world(world, rank)

    def expect(res, code, what):
        assert all(s == code for s, _ in res), f"{what}: statuses {[s for s, _ in res]}, want {code} on every rank"
        assert all(ok for _, ok in res), f"{what}: an index is not left empty"

    def restore():
        for p, b in good.items():
            with open(p, "wb") as f:
                f.write(b)

    fresh = lambda r: kind.index(trained=False)  # noqa: E731
    expect(attempt(fresh, prefix=os.path.join(tmp, "none")), b200vs.EINTERNAL, "missing manifest")
    os.remove(files[1])
    expect(attempt(fresh), b200vs.EINTERNAL, "missing rank file")
    restore()
    os.replace(files[0], files[2] + ".x"); os.replace(files[2], files[0]); os.replace(files[2] + ".x", files[2])
    expect(attempt(fresh), b200vs.EINTERNAL, "swapped rank files")
    restore()
    with open(files[2], "r+b") as f:
        f.truncate(len(good[files[2]]) - 9)
    expect(attempt(fresh), b200vs.EINTERNAL, "truncated rank file")
    restore()
    shutil.copyfile(f"{B}.1-of-{W}", files[1])
    expect(attempt(fresh), b200vs.EINTERNAL, "rank file of another trained state")
    restore()
    for what, mk in (("type", lambda r: b200vs.Index(IVF_FLAT, L2, D, nlist=kind.nlist)),
                     ("metric", lambda r: b200vs.Index(IVF_PQ, IP, D, nlist=kind.nlist, pq_m=4, pq_nbits=8)),
                     ("dim", lambda r: b200vs.Index(IVF_PQ, L2, 2 * D, nlist=kind.nlist, pq_m=4, pq_nbits=8)),
                     ("nlist", lambda r: b200vs.Index(IVF_PQ, L2, D, nlist=kind.nlist + 1, pq_m=4, pq_nbits=8)),
                     ("pq_m", lambda r: b200vs.Index(IVF_PQ, L2, D, nlist=kind.nlist, pq_m=8, pq_nbits=8)),
                     ("nbits", lambda r: b200vs.Index(IVF_PQ, L2, D, nlist=kind.nlist, pq_m=4, pq_nbits=4))):
        expect(attempt(mk), b200vs.EINTERNAL, f"wrapped index with another {what}")
    # a wrapped index trained with another state
    expect(attempt(lambda r: other.index(), trained=True), b200vs.EINTERNAL, "wrapped index with another trained state")

    def nonempty(r):
        ix = kind.index()
        if r == W - 1:
            ix.add(xs[0][:1], np.array([10 ** 8], np.int64))
        return ix
    res = attempt(nonempty)
    assert all(s == b200vs.EILLEGAL_PARAMETERS for s, _ in res), f"non-empty wrapped index: {res}"
    # HNSW onto another world
    hk = Kind("hnsw_l2", 2)
    H = os.path.join(tmp, "h")

    def hsave(r, world):
        ix = hk.index()
        sh = world.connect(ix, r)
        sh.add(xs[r], ids[r])
        sh.save(H)
        sh.close(); ix.close()
    run_world(2, hsave)
    expect(attempt(lambda r: hk.index(), prefix=H, trained=True), b200vs.EVECTOR_NOT_SUPPORT, "HNSW onto another world")
    # a save that rank 1 cannot write leaves the earlier snapshot intact, byte for byte
    os.mkdir(files[1] + ".tmp")

    def failing_save(r, world):
        ix = other.index()
        sh = world.connect(ix, r)
        sh.add(xs[r], ids[r])
        st = _status(lambda: sh.save(A))
        sh.close(); ix.close()
        return st
    sts = run_world(W, failing_save)
    assert all(s == b200vs.EINTERNAL for s in sts), f"unwritable save: {sts}"
    os.rmdir(files[1] + ".tmp")
    for p, b in good.items():
        assert open(p, "rb").read() == b, f"{p} changed by a failed save"
    left = [n for n in os.listdir(tmp) if n.endswith(".tmp")]
    assert not left, f"temporary files left: {left}"
    # after every refusal: a correct load into empty indexes (untrained and already trained) gives the saved results
    for trained in (False, True):
        def rank(r, world):
            ix = kind.index(trained=trained)
            sh = world.connect(ix, r)
            sh.load(A)
            out, _ = _reads(kind, sh, xq, 0)
            sh.close(); ix.close()
            return out
        for r, out in enumerate(run_world(W, rank)):
            for key, w in want.items():
                _same(out[key], w, f"rank {r} {key} after the refusals (trained {trained})")
    # an untrained list-sharded snapshot restores untrained
    U = os.path.join(tmp, "u")

    def usave(r, world):
        ix = kind.index(trained=False)
        sh = world.connect(ix, r)
        sh.save(U)
        sh.close(); ix.close()
    run_world(W, usave)

    def uload(r, world):
        ix = kind.index(trained=False)
        sh = world.connect(ix, r)
        sh.load(U)
        ok = _empty(ix, False)
        sh.close(); ix.close()
        return ok
    assert all(run_world(W, uload)), "an untrained snapshot did not restore untrained"


def test_refusals():
    run("case_refusals")


def _main():
    case, args, dump_after = sys.argv[1], json.loads(sys.argv[2]), int(sys.argv[3])
    faulthandler.dump_traceback_later(dump_after, exit=True)
    rc = 1
    try:
        globals()[case](*args)
        print("PERSIST CASE OK", flush=True)
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
