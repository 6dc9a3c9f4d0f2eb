"""Sharded binary indexes: BINARY_IVF_FLAT by inverted list and BINARY_FLAT by row through b200vs_shard_*_binary.

World 1 runs in this process (no NCCL).  Worlds 2, 3, 5 and 8 run as threads of one process on one GPU over the loopback
NCCL (tests/shard_loopback.py's World and run_world), each case in a subprocess of its own started through this file's
__main__.  The reference is always a plain single binary index holding every row: distances, ids and counts must be equal
bit for bit."""
import faulthandler
import json
import os
import subprocess
import sys
import threading

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, os.path.join(ROOT, "dingo-store_b200", "python"))
sys.path.insert(0, HERE)

import b200vs  # noqa: E402
from b200vs import BINARY_FLAT, BINARY_IVF_FLAT, HAMMING  # noqa: E402
from gpu_util import require_gpu  # noqa: E402
from shard_loopback import LIB, run_world  # noqa: E402

pytestmark = pytest.mark.gpu
WORLDS = (2, 3, 5, 8)
CASE_TIMEOUT = 600  # seconds of one subprocess; every rendezvous of the loopback library times out after 60 s


@pytest.fixture(autouse=True)
def _gpu():
    require_gpu()


def _assert_same(got, want, what):
    for x, y in zip(got, want):
        bad = np.argwhere((x.view(np.uint32) if x.dtype == np.float32 else x) != (y.view(np.uint32) if y.dtype == np.float32 else y))
        assert bad.size == 0, f"{what}: differs at {bad[:4].tolist()}: got {x[tuple(bad[0])]}, want {y[tuple(bad[0])]}"


def _status(fn):
    try:
        fn()
        return b200vs.OK
    except b200vs.B200VSError as e:
        return e.code


def _bits(rng, n, dim, ties=False):
    """n packed rows of dim bits; ties: only the first byte varies, so many rows share a Hamming distance to any query."""
    x = rng.integers(0, 256, (n, dim // 8), dtype=np.uint8)
    if ties:
        x[:, 1:] = 0
        x[:, 0] &= 0x0F
    return x


def _index(kind, dim, nlist):
    return b200vs.Index(kind, HAMMING, dim, nlist=nlist) if kind == BINARY_IVF_FLAT else b200vs.Index(kind, HAMMING, dim)


FILTERS = [dict(), dict(id_range=(3, 400)), dict(sorted_ids=np.arange(1, 900, 3)), dict(sorted_ids=np.arange(1, 900, 3), negate=True),
           dict(exact_only=True)]


# ---------------------------------------------------------------------------------------------
# world 1: the shard flow on one rank against a plain index
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dim", (64, 200, 1024))
@pytest.mark.parametrize("kind", (BINARY_FLAT, BINARY_IVF_FLAT))
def test_world1_matches_plain_index(kind, dim):
    import torch
    rng = np.random.default_rng(dim + kind)
    n, nlist, nprobe = 5000, 16, 5
    x = _bits(rng, n, dim)
    ids = rng.permutation(10 ** 6)[:n].astype(np.int64) + 10 ** 6
    ids[:999] = np.arange(1, 1000)  # the filters select some of these
    xq = _bits(rng, 33, dim)
    plain = _index(kind, dim, nlist)
    ix = _index(kind, dim, nlist)
    sh = b200vs.BinaryShard(ix, 0, 1, None)
    if kind == BINARY_IVF_FLAT:
        plain.train(x)
        sh.train(x)
        assert np.array_equal(ix.get_trained_state(), plain.get_trained_state()), "world-1 train differs from b200vs_train_binary"
    plain.add(x, ids)
    sh.add(x[:n // 2], ids[:n // 2])
    xd, idd = torch.from_numpy(x[n // 2:].copy()).cuda(), torch.from_numpy(ids[n // 2:].copy()).cuda()
    torch.cuda.synchronize()
    sh.add_device(n - n // 2, xd.data_ptr(), idd.data_ptr())
    if kind == BINARY_IVF_FLAT:
        p_off, _, p_rows, p_ids = plain.export_lists(nlist)
        off, _, rows, lid = ix.export_lists(nlist)
        assert np.array_equal(off, p_off) and np.array_equal(lid, p_ids) and np.array_equal(rows, p_rows), "lists differ"
    kw0 = dict(nprobe=nprobe) if kind == BINARY_IVF_FLAT else {}
    for k in (1, 10, 4096):
        _assert_same(sh.search(xq, k, **kw0), plain.search(xq, k, **kw0), f"k {k}")
    for j, kw in enumerate(FILTERS):
        _assert_same(sh.search(xq, 10, **kw0, **kw), plain.search(xq, 10, **kw0, **kw), f"filter {j}")
    for radius in (0, 1, 7.9, dim / 4, dim + 5, float("inf")):
        _assert_same(sh.range_search(xq, radius, 16, **kw0), plain.range_search(xq, radius, 16, **kw0), f"range {radius}")
    # device pointers
    qd = torch.from_numpy(xq).cuda()
    od = torch.empty((33, 10), dtype=torch.float32, device="cuda:0")
    oi = torch.empty((33, 10), dtype=torch.int64, device="cuda:0")
    sp, _keep = b200vs.make_search_params(**kw0)
    torch.cuda.synchronize()
    sh.search_device(33, qd.data_ptr(), 10, od.data_ptr(), oi.data_ptr(), sp=sp)
    torch.cuda.synchronize()
    _assert_same((od.cpu().numpy(), oi.cpu().numpy()), plain.search(xq, 10, **kw0), "device search")
    rd = torch.empty((33, 16), dtype=torch.float32, device="cuda:0")
    ri = torch.empty((33, 16), dtype=torch.int64, device="cuda:0")
    rc = torch.empty(33, dtype=torch.int32, device="cuda:0")
    sh.range_search_device(33, qd.data_ptr(), dim / 4, 16, rd.data_ptr(), ri.data_ptr(), rc.data_ptr(), sp=sp)
    torch.cuda.synchronize()
    _assert_same((rd.cpu().numpy(), ri.cpu().numpy(), rc.cpu().numpy()), plain.range_search(xq, dim / 4, 16, **kw0), "device range")
    sh.close()


def test_world1_bmma_tile_scan_serves_the_batch():
    rng = np.random.default_rng(5)
    n, dim, nlist, nq = 65536, 256, 8, 256
    x = _bits(rng, n, dim)
    ids = np.arange(n, dtype=np.int64)
    xq = _bits(rng, nq, dim)
    plain = _index(BINARY_IVF_FLAT, dim, nlist)
    plain.train(x)
    plain.add(x, ids)
    ix = _index(BINARY_IVF_FLAT, dim, nlist)
    ix.set_trained_state(plain.get_trained_state())
    sh = b200vs.BinaryShard(ix, 0, 1, None)
    sh.add(x, ids)
    ix.set_profiling(True)
    got = sh.search(xq, 10, nprobe=nlist)
    tile = ix.stats()[1]
    exact = sh.search(xq, 10, nprobe=nlist, exact_only=True)
    exact_tile = ix.stats()[1]
    ix.set_profiling(False)
    assert tile > 0, "the BMMA tile scan served no query"
    assert exact_tile == 0, "exact_only still reached the tile scan"
    want = plain.search(xq, 10, nprobe=nlist)
    _assert_same(got, want, "tile scan")
    _assert_same(exact, want, "exact scan")
    sh.close()


def test_world1_refusals():
    ill, nots = b200vs.EILLEGAL_PARAMETERS, b200vs.EVECTOR_NOT_SUPPORT
    L = b200vs.lib()
    dim = 64
    u = np.zeros((2, dim // 8), np.uint8)
    f = np.zeros((2, dim), np.float32)
    ids = np.arange(2, dtype=np.int64)
    D, I, C = np.zeros((2, 1), np.float32), np.zeros((2, 1), np.int64), np.zeros(2, np.int32)
    bi = _index(BINARY_IVF_FLAT, dim, 2)
    fx = b200vs.Index(b200vs.FLAT, b200vs.L2, dim)
    # creation: b200vs_shard_create keeps refusing binary indexes; the binary create refuses float ones
    with pytest.raises(b200vs.B200VSError) as e:
        b200vs.Shard(bi, 0, 1, None)
    assert e.value.code == nots
    with pytest.raises(b200vs.B200VSError) as e:
        b200vs.BinaryShard(fx, 0, 1, None)
    assert e.value.code == ill
    with pytest.raises(b200vs.B200VSError) as e:  # a row-sharded binary index must be empty
        bf = _index(BINARY_FLAT, dim, 0)
        bf.add(u, ids)
        b200vs.BinaryShard(bf, 0, 1, None)
    assert e.value.code == nots
    fsh = b200vs.Shard(fx, 0, 1, None)
    for kind in (BINARY_IVF_FLAT, BINARY_FLAT):
        ix = _index(kind, dim, 2)
        sh = b200vs.BinaryShard(ix, 0, 1, None)
        h = sh.h
        if kind == BINARY_IVF_FLAT:
            assert sh.delete(ids) == 0  # untrained: OK
            sh.train(np.random.default_rng(0).integers(0, 256, (40, dim // 8), dtype=np.uint8))
        # float data calls on a binary shard
        assert L.b200vs_shard_train(h, 2, f.ctypes.data) == ill
        assert L.b200vs_shard_add(h, 2, f.ctypes.data, ids.ctypes.data) == ill
        assert L.b200vs_shard_add_device(h, 0, None, None) == ill
        assert L.b200vs_shard_search(h, 0, 2, f.ctypes.data, 1, None, D.ctypes.data, I.ctypes.data) == ill
        assert L.b200vs_shard_search_device(h, 1, 2, f.ctypes.data, 1, None, D.ctypes.data, I.ctypes.data, None) == ill
        assert L.b200vs_shard_range_search(h, 2, 2, f.ctypes.data, 1.0, 1, None, D.ctypes.data, I.ctypes.data, C.ctypes.data) == ill
        assert L.b200vs_shard_range_search_device(h, 3, 2, f.ctypes.data, 1.0, 1, None, D.ctypes.data, I.ctypes.data, C.ctypes.data, None) == ill
        # the refused reads used up their sequence numbers 0..3: the next read is number 4
        assert L.b200vs_shard_search_binary(h, 3, 2, u.ctypes.data, 1, None, D.ctypes.data, I.ctypes.data) == ill
        assert _status(lambda: sh.search(u, 1, seq=4)) == b200vs.OK
        # a NaN radius, and max_results outside [1, 4096]: refused, the sequence number used up
        assert _status(lambda: sh.range_search(u, float("nan"), 4, seq=5)) == ill
        assert _status(lambda: sh.range_search(u, 1.0, 0, seq=6)) == ill
        assert _status(lambda: sh.range_search(u, 1.0, 4097, seq=7)) == ill
        assert _status(lambda: sh.range_search(u, 1.0, 4, seq=8)) == b200vs.OK
        # pre-sizing and the batched HNSW build
        assert L.b200vs_shard_plan_add_device(h, 2, f.ctypes.data) == nots
        assert L.b200vs_shard_plan_commit(h) == nots
        assert L.b200vs_shard_hnsw_add_batched(h, 2, f.ctypes.data, ids.ctypes.data, 0) == ill
        if kind == BINARY_IVF_FLAT:
            assert sh.list_range() == (0, 2)
            assert _status(lambda: sh.delete(np.array([77], np.int64))) == b200vs.EVECTOR_INVALID
            assert _status(lambda: sh.broadcast_state(0)) == b200vs.OK
        else:
            assert _status(lambda: sh.list_range()) == nots
            assert _status(lambda: sh.broadcast_state(0)) == nots
            assert sh.delete(np.array([77], np.int64)) == 0
            assert _status(lambda: sh.train(u)) == b200vs.OK
        sh.close()
    # the binary data calls on a float shard
    h = fsh.h
    assert L.b200vs_shard_train_binary(h, 2, u.ctypes.data) == ill
    assert L.b200vs_shard_add_binary(h, 2, u.ctypes.data, ids.ctypes.data) == ill
    assert L.b200vs_shard_add_binary_device(h, 0, None, None) == ill
    assert L.b200vs_shard_search_binary(h, 0, 2, u.ctypes.data, 1, None, D.ctypes.data, I.ctypes.data) == ill
    assert L.b200vs_shard_search_binary_device(h, 1, 2, u.ctypes.data, 1, None, D.ctypes.data, I.ctypes.data, None) == ill
    assert L.b200vs_shard_range_search_binary(h, 2, 2, u.ctypes.data, 1.0, 1, None, D.ctypes.data, I.ctypes.data, C.ctypes.data) == ill
    assert L.b200vs_shard_range_search_binary_device(h, 3, 2, u.ctypes.data, 1.0, 1, None, D.ctypes.data, I.ctypes.data,
                                                     C.ctypes.data, None) == ill
    fsh.close()
    # the single-index device building blocks keep refusing binary indexes
    bi.train(np.random.default_rng(1).integers(0, 256, (40, dim // 8), dtype=np.uint8))
    assert L.b200vs_add_with_ids_device(bi.h, 2, u.ctypes.data, ids.ctypes.data, None, 0) == nots
    assert L.b200vs_assign_device(bi.h, 2, u.ctypes.data, I.ctypes.data) == nots
    assert L.b200vs_coarse_device(bi.h, 2, u.ctypes.data, 1, 0, 2, D.ctypes.data, I.ctypes.data, None) == nots
    assert L.b200vs_search_probes_device(bi.h, 2, u.ctypes.data, 1, I.ctypes.data, 1, None, D.ctypes.data, I.ctypes.data, None) == nots


# ---------------------------------------------------------------------------------------------
# worlds 2, 3, 5, 8 over the loopback NCCL
# ---------------------------------------------------------------------------------------------
def _connect(world, ix, rank, lanes=2):
    """The shard of rank `rank` over a fresh communicator whose id rank 0 makes: BinaryShard for a binary index."""
    idb = world.gather(rank, b200vs.Shard.unique_id() if rank == 0 else None)[0]
    return (b200vs.BinaryShard if ix.binary else b200vs.Shard)(ix, rank, world.W, idb, lanes=lanes)


def _row_counts(W, big):
    """Rows each rank sends: none on rank 0, less than one 256-row tile on rank 1, `big` on the last rank."""
    n = [0] + [97 + 31 * r for r in range(1, W)]
    n[-1] = big
    return n


def _cent(rng, allx, nlist):
    return allx[rng.choice(len(allx), nlist, replace=False)].copy()


def case_ivf(W, lists):
    """lists "uneven" (nlist = 2W + 1) or "few" (nlist = 3 < W: the state comes from the last rank's broadcast_state);
    data with many exact Hamming ties, ids interleaved across ranks."""
    import torch
    nlist = 2 * W + 1 if lists == "uneven" else 3
    dim = 200
    rng = np.random.default_rng(1000 * W + nlist)
    n = _row_counts(W, 700)
    xs = [_bits(rng, m, dim, ties=True) for m in n]
    ids = [np.arange(m, dtype=np.int64) * W + r + 1 for r, m in enumerate(n)]
    allx = np.concatenate(xs)
    blob = b200vs.binary_ivf_state_blob(_cent(rng, allx, nlist))
    h = [m // 2 for m in n]  # host pointers for the first half, device pointers for the rest
    plain = _index(BINARY_IVF_FLAT, dim, nlist)
    plain.set_trained_state(blob)
    plain.add(np.concatenate([x[:hh] for x, hh in zip(xs, h)]), np.concatenate([i[:hh] for i, hh in zip(ids, h)]))
    plain.add(np.concatenate([x[hh:] for x, hh in zip(xs, h)]), np.concatenate([i[hh:] for i, hh in zip(ids, h)]))
    p_off, _, p_rows, p_ids = plain.export_lists(nlist)
    xq = _bits(rng, 64, dim, ties=True)
    nprobe = min(nlist, 5)
    shapes = [(nq, k) for nq in (1, W - 1, W + 1, 64) if nq > 0 for k in (1, 10)] + [(W + 1, 256 // W), (W + 1, 256 // W + 1)]
    want = {s: plain.search(xq[:s[0]], s[1], nprobe=nprobe) for s in shapes}
    for j, kw in enumerate(FILTERS):
        want[("filter", j)] = plain.search(xq, 10, nprobe=nprobe, **kw)
    broadcast = nlist < W

    def rank(r, world):
        ix = _index(BINARY_IVF_FLAT, dim, nlist)
        if not broadcast or r == W - 1:
            ix.set_trained_state(blob)
        sh = _connect(world, ix, r)
        if broadcast:
            sh.broadcast_state(W - 1)
        sh.add(xs[r][:h[r]], ids[r][:h[r]])
        rest = xs[r][h[r]:]
        xd, idd = torch.from_numpy(rest.copy()).cuda(), torch.from_numpy(ids[r][h[r]:].copy()).cuda()
        torch.cuda.synchronize()
        sh.add_device(len(rest), xd.data_ptr() if len(rest) else None, idd.data_ptr() if len(rest) else None)
        out = {"range": sh.list_range(), "lists": ix.export_lists(nlist), "state": ix.get_trained_state()}
        seq = 0
        for s in shapes:
            out[s] = sh.search(xq[:s[0]], s[1], seq=seq, nprobe=nprobe)
            seq += 1
        for j, kw in enumerate(FILTERS):
            out[("filter", j)] = sh.search(xq, 10, seq=seq, nprobe=nprobe, **kw)
            seq += 1
        # device pointers: four batches in flight on two streams over two lanes
        qd = torch.from_numpy(xq).cuda()
        sts = [torch.cuda.Stream(device="cuda:0") for _ in range(2)]
        dev_out = [(torch.empty((64, 10), dtype=torch.float32, device="cuda:0"), torch.empty((64, 10), dtype=torch.int64, device="cuda:0"))
                   for _ in range(4)]
        sp, _keep = b200vs.make_search_params(nprobe=nprobe)
        torch.cuda.synchronize()
        for i in range(4):
            sh.search_device(64, qd.data_ptr(), 10, dev_out[i][0].data_ptr(), dev_out[i][1].data_ptr(), stream=sts[i % 2].cuda_stream, sp=sp, seq=seq)
            seq += 1
        torch.cuda.synchronize()
        out["device"] = [(a.cpu().numpy(), b.cpu().numpy()) for a, b in dev_out]
        got = {}

        def call(q):
            got[q] = sh.search(xq, 10, seq=q, nprobe=nprobe)
        ths = [threading.Thread(target=call, args=(seq + t,)) for t in (2, 0, 3, 1)]
        for t in ths:
            t.start()
        for t in ths:
            t.join()
        out["threads"] = [got[seq + t] for t in range(4)]
        sh.close()
        return out

    res = run_world(W, rank)
    per = -(-nlist // W)
    for r, o in enumerate(res):
        assert np.array_equal(o["state"], plain.get_trained_state()), f"rank {r}: trained state"
        b, e = o["range"]
        assert (b, e) == (min(nlist, per * r), min(nlist, per * (r + 1))), f"rank {r}: list range {(b, e)}"
        off, _, rows, lid = o["lists"]
        lens = np.diff(off)
        assert lens[:b].sum() == 0 and lens[e:].sum() == 0, f"rank {r} holds rows of lists it does not own"
        for l in range(b, e):
            assert np.array_equal(lid[off[l]:off[l + 1]], p_ids[p_off[l]:p_off[l + 1]]), f"rank {r} list {l}: ids or arrival order"
            assert np.array_equal(rows[off[l]:off[l + 1]], p_rows[p_off[l]:p_off[l + 1]]), f"rank {r} list {l}: packed rows"
        for key, w in want.items():
            _assert_same(o[key], w, f"rank {r} search {key}")
        for i, got in enumerate(o["device"] + o["threads"]):
            _assert_same(got, want[(64, 10)], f"rank {r} device / threaded batch {i}")


def case_flat(W):
    rng = np.random.default_rng(77 + W)
    dim = 64
    n = _row_counts(W, 900)
    xs = [_bits(rng, m, dim, ties=True) for m in n]
    ids = [rng.choice(10 ** 6, m, replace=False).astype(np.int64) + r * 10 ** 6 for r, m in enumerate(n)]
    allx, alli = np.concatenate(xs), np.concatenate(ids)
    own = b200vs.row_owner(alli, W)
    xq = _bits(rng, 40, dim, ties=True)
    plain = _index(BINARY_FLAT, dim, 0)
    plain.add(allx, alli)
    shapes = [(nq, k) for nq in (1, W - 1, W + 1, 40) if nq > 0 for k in (1, 10)] + [(W + 1, 256 // W + 1), (7, 300)]
    want = {s: plain.search(xq[:s[0]], s[1]) for s in shapes}
    for j, kw in enumerate(FILTERS):
        want[("filter", j)] = plain.search(xq, 10, **kw)
    # re-adding an existing id replaces its row (as b200vs_add_with_ids_binary), wherever the caller sends it from
    re_id, re_x, dup_x = alli[len(alli) // 2], _bits(rng, 1, dim), _bits(rng, 1, dim)
    plain.add(re_x, np.array([re_id], np.int64))
    want["readd"] = plain.search(xq, 10)

    def rank(r, world):
        ix = _index(BINARY_FLAT, dim, 0)
        sh = _connect(world, ix, r)
        sh.add(xs[r], ids[r])
        out = {"held": np.sort(ix.export_lists(1)[3])}
        out.update({s: sh.search(xq[:s[0]], s[1]) for s in shapes})
        for j, kw in enumerate(FILTERS):
            out[("filter", j)] = sh.search(xq, 10, **kw)
        before = (ix.get_count(), ix.get_memory_size())
        # ranks 0 and 1 each send a row with one new id: its owner receives the id twice
        out["dup"] = _status(lambda: sh.add(dup_x if r < 2 else dup_x[:0], np.array([10 ** 9] if r < 2 else [], np.int64)))
        out["dup_state"] = before == (ix.get_count(), ix.get_memory_size())
        last = r == W - 1
        sh.add(re_x if last else re_x[:0], np.array([re_id] if last else [], np.int64))
        out["readd"] = sh.search(xq, 10)
        out["count"] = ix.get_count()
        sh.close()
        return out

    res = run_world(W, rank)
    for r, o in enumerate(res):
        assert np.array_equal(o["held"], np.sort(alli[own == r])), f"rank {r} holds rows it does not own"
        assert o["dup"] == b200vs.EVECTOR_ID_DUPLICATED and o["dup_state"], f"rank {r}: repeated id returned {o['dup']}"
        for key, w in want.items():
            _assert_same(o[key], w, f"rank {r} {key}")
    assert sum(o["count"] for o in res) == len(alli)


def case_range(W, kind):
    import torch
    dim = 64
    rng = np.random.default_rng(31 + W)
    n = _row_counts(W, 600)
    xs = [_bits(rng, m, dim, ties=True) for m in n]
    ids = [np.arange(m, dtype=np.int64) * W + r + 1 for r, m in enumerate(n)]
    allx, alli = np.concatenate(xs), np.concatenate(ids)
    xq = _bits(rng, W + 1, dim, ties=True)
    nlist = 2 * W + 1
    blob = b200vs.binary_ivf_state_blob(_cent(rng, allx, nlist))
    plain = _index(kind, dim, nlist)
    if kind == BINARY_IVF_FLAT:
        plain.set_trained_state(blob)
    plain.add(allx, alli)
    kw = {"nprobe": nlist} if kind == BINARY_IVF_FLAT else {}
    radii = (0, 1, 7.9, dim / 4, dim + 5, float("inf"))
    want = [plain.range_search(xq, rad, 24, **kw) for rad in radii]
    assert (want[-1][2] == 24).all(), "max_results must be below the hit count"

    def rank(r, world):
        ix = _index(kind, dim, nlist)
        if kind == BINARY_IVF_FLAT:
            ix.set_trained_state(blob)
        sh = _connect(world, ix, r)
        sh.add(xs[r], ids[r])
        out = [sh.range_search(xq, rad, 24, seq=i, **kw) for i, rad in enumerate(radii)]
        nan = _status(lambda: sh.range_search(xq, float("nan"), 24, seq=len(radii), **kw))
        qd = torch.from_numpy(xq).cuda()
        d = torch.empty((W + 1, 24), dtype=torch.float32, device="cuda:0")
        i = torch.empty((W + 1, 24), dtype=torch.int64, device="cuda:0")
        c = torch.empty(W + 1, dtype=torch.int32, device="cuda:0")
        sp, _keep = b200vs.make_search_params(**kw)
        torch.cuda.synchronize()
        sh.range_search_device(W + 1, qd.data_ptr(), dim / 4, 24, d.data_ptr(), i.data_ptr(), c.data_ptr(), sp=sp, seq=len(radii) + 1)
        torch.cuda.synchronize()
        out.append((d.cpu().numpy(), i.cpu().numpy(), c.cpu().numpy()))
        sh.close()
        return out, nan

    for r, (o, nan) in enumerate(run_world(W, rank)):
        assert nan == b200vs.EILLEGAL_PARAMETERS, f"rank {r}: a NaN radius returned {nan}"
        for got, w, rad in zip(o, want + [want[3]], radii + (dim / 4,)):
            _assert_same(got, w, f"rank {r} radius {rad}")


def case_delete(W):
    dim = 64
    nlist = 2 * W + 1
    rng = np.random.default_rng(9 + W)
    n = _row_counts(W, 500)
    xs = [_bits(rng, m, dim) for m in n]
    ids = [np.arange(m, dtype=np.int64) * W + r + 1 for r, m in enumerate(n)]
    allx, alli = np.concatenate(xs), np.concatenate(ids)
    blob = b200vs.binary_ivf_state_blob(_cent(rng, allx, nlist))
    gone = alli[::7]

    def rank(r, world):
        out = {}
        for kind in (BINARY_IVF_FLAT, BINARY_FLAT):
            ix = _index(kind, dim, nlist)
            sh = _connect(world, ix, r)
            if kind == BINARY_IVF_FLAT:
                out["untrained"] = _status(lambda: sh.delete(gone))
                ix.set_trained_state(blob)
            sh.add(xs[r], ids[r])
            out[(kind, "some")] = sh.delete(gone)
            out[(kind, "none")] = _status(lambda: sh.delete(np.array([-5, -6], np.int64)))
            out[(kind, "count")] = ix.get_count()
            sh.close()
        return out

    res = run_world(W, rank)
    for r, o in enumerate(res):
        assert o["untrained"] == b200vs.OK
        for kind in (BINARY_IVF_FLAT, BINARY_FLAT):
            assert o[(kind, "some")] == len(gone), f"rank {r} kind {kind}: removed {o[(kind, 'some')]}"
        assert o[(BINARY_IVF_FLAT, "none")] == b200vs.EVECTOR_INVALID and o[(BINARY_FLAT, "none")] == b200vs.OK
    for kind in (BINARY_IVF_FLAT, BINARY_FLAT):
        assert sum(o[(kind, "count")] for o in res) == len(alli) - len(gone)


def case_train(W):
    dim = 200
    nlist = 2 * W
    rng = np.random.default_rng(3 + W)
    xs = [_bits(rng, 300 + 50 * r, dim) for r in range(W)]
    parts = []
    for r in range(W):  # standalone trains of nlist / W lists on each rank's rows
        p = _index(BINARY_IVF_FLAT, dim, nlist // W)
        p.train(xs[r])
        parts.append(p.get_trained_state()[32:])
    want = np.concatenate(parts)

    def rank(r, world):
        ix = _index(BINARY_IVF_FLAT, dim, nlist)
        sh = _connect(world, ix, r)
        out = {"short": _status(lambda: sh.train(xs[r][:nlist // W - 1] if r == W - 1 else xs[r])), "trained": ix.is_trained()}
        odd = _index(BINARY_IVF_FLAT, dim, nlist + 1)
        sh2 = _connect(world, odd, r)
        out["odd"] = _status(lambda: sh2.train(xs[r]))
        out["odd trained"] = odd.is_trained()
        sh2.close()
        sh.train(xs[r])
        out["state"] = ix.get_trained_state()
        sh.close()
        return out

    for r, o in enumerate(run_world(W, rank)):
        assert o["short"] == b200vs.EILLEGAL_PARAMETERS and not o["trained"], f"rank {r}: short-row refusal {o['short']}"
        assert o["odd"] == b200vs.EILLEGAL_PARAMETERS and not o["odd trained"], f"rank {r}: nlist % W refusal {o['odd']}"
        assert np.array_equal(o["state"][32:], want), f"rank {r}: centroids differ from the standalone trains"
        assert o["state"][8:16].view(np.int64)[0] == nlist


def _snap_data(kind, W0, seed):
    dim, nlist = 200, 6
    rng = np.random.default_rng(seed)
    n = [150 + 40 * r for r in range(W0)]
    xs = [_bits(rng, m, dim, ties=True) for m in n]
    ids = [np.arange(m, dtype=np.int64) * W0 + r + 1 for r, m in enumerate(n)]
    allx, alli = np.concatenate(xs), np.concatenate(ids)
    blob = b200vs.binary_ivf_state_blob(_cent(rng, allx, nlist))
    xq = _bits(rng, 9, dim, ties=True)
    return dim, nlist, xs, ids, allx, alli, blob, xq


def case_snapshot(W, W2, kind, prefix):
    """Save at W, load at W2 (the same world: byte-equal lists); results equal a plain index of every row."""
    dim, nlist, xs, ids, allx, alli, blob, xq = _snap_data(kind, W, 11 * W + W2)
    plain = _index(kind, dim, nlist)
    if kind == BINARY_IVF_FLAT:
        plain.set_trained_state(blob)
    plain.add(allx, alli)
    kw = {"nprobe": nlist} if kind == BINARY_IVF_FLAT else {}
    want = plain.search(xq, 10, **kw), plain.range_search(xq, dim / 4, 32, **kw)

    def save(r, world):
        ix = _index(kind, dim, nlist)
        if kind == BINARY_IVF_FLAT:
            ix.set_trained_state(blob)
        sh = _connect(world, ix, r)
        sh.add(xs[r], ids[r])
        sh.save(prefix)
        lists = ix.export_lists(nlist if kind == BINARY_IVF_FLAT else 1)
        sh.close()
        return lists

    saved = run_world(W, save)

    def load(r, world):
        ix = _index(kind, dim, nlist)
        sh = _connect(world, ix, r)
        sh.load(prefix)
        out = {"lists": ix.export_lists(nlist if kind == BINARY_IVF_FLAT else 1), "search": sh.search(xq, 10, **kw),
               "range": sh.range_search(xq, dim / 4, 32, **kw)}
        sh.close()
        return out

    for r, o in enumerate(run_world(W2, load)):
        _assert_same(o["search"], want[0], f"rank {r}: search after load {W} -> {W2}")
        _assert_same(o["range"], want[1], f"rank {r}: range search after load {W} -> {W2}")
        if W2 == W:
            for a, b in zip(o["lists"], saved[r]):
                assert (a is None and b is None) or np.array_equal(a, b), f"rank {r}: restored lists differ from the saved ones"


def case_snapshot_refusals(W, prefix):
    """A float snapshot into a binary shard and a snapshot of another nlist: EINTERNAL, the index left empty and loadable."""
    dim, nlist, xs, ids, allx, alli, blob, xq = _snap_data(BINARY_IVF_FLAT, W, 5 * W)
    rng = np.random.default_rng(W)
    fcent = rng.standard_normal((nlist, dim)).astype(np.float32)
    fx = [rng.standard_normal((20, dim)).astype(np.float32) for _ in range(W)]

    def rank(r, world):
        f = b200vs.Index(b200vs.IVF_FLAT, b200vs.L2, dim, nlist=nlist)
        f.set_trained_state(b200vs.ivf_state_blob(fcent, b200vs.L2))
        fsh = _connect(world, f, r)
        fsh.add(fx[r], np.arange(20, dtype=np.int64) + 100 * r)
        fsh.save(prefix + "f")
        fsh.close()
        ix = _index(BINARY_IVF_FLAT, dim, nlist)
        ix.set_trained_state(blob)
        sh = _connect(world, ix, r)
        sh.add(xs[r], ids[r])
        sh.save(prefix + "b")
        sh.close()
        out = {}
        other = _index(BINARY_IVF_FLAT, dim, nlist + 1)
        osh = _connect(world, other, r)
        out["nlist"] = _status(lambda: osh.load(prefix + "b"))
        out["nlist empty"] = other.get_count()
        osh.close()
        fresh = _index(BINARY_IVF_FLAT, dim, nlist)
        bsh = _connect(world, fresh, r)
        out["float"] = _status(lambda: bsh.load(prefix + "f"))
        out["float empty"] = fresh.get_count()
        bsh.load(prefix + "b")  # still loadable
        out["search"] = bsh.search(xq, 10, nprobe=nlist)
        bsh.close()
        # and a binary snapshot into a float shard
        f2 = b200vs.Index(b200vs.IVF_FLAT, b200vs.L2, dim, nlist=nlist)
        f2sh = _connect(world, f2, r)
        out["binary into float"] = _status(lambda: f2sh.load(prefix + "b"))
        f2sh.close()
        return out

    plain = _index(BINARY_IVF_FLAT, dim, nlist)
    plain.set_trained_state(blob)
    plain.add(allx, alli)
    want = plain.search(xq, 10, nprobe=nlist)
    for r, o in enumerate(run_world(W, rank)):
        assert o["nlist"] == b200vs.EINTERNAL and o["nlist empty"] == 0, f"rank {r}: another nlist returned {o['nlist']}"
        assert o["float"] == b200vs.EINTERNAL and o["float empty"] == 0, f"rank {r}: a float snapshot returned {o['float']}"
        assert o["binary into float"] == b200vs.EINTERNAL, f"rank {r}: a binary snapshot into a float shard returned {o['binary into float']}"
        _assert_same(o["search"], want, f"rank {r}: search after the refused loads")


def each_world(case, worlds, *args):
    for W in worlds:
        try:
            globals()[case](W, *args)
        except AssertionError as e:
            raise AssertionError(f"world {W}: {e}") from e


def _run(case, *args, worlds=WORLDS):
    """Runs each_world(case, worlds, *args) in a subprocess on the loopback NCCL; fails with its output if it failed."""
    assert os.path.exists(LIB), f"{LIB} not built (build() runs make -C tests/nccl_loopback)"
    env = dict(os.environ, B200VS_NCCL_LIB=LIB)
    cmd = [sys.executable, os.path.abspath(__file__), "each_world", json.dumps([case, list(worlds), *args]), str(CASE_TIMEOUT - 20)]
    try:
        p = subprocess.run(cmd, env=env, cwd=ROOT, capture_output=True, text=True, timeout=CASE_TIMEOUT)
    except subprocess.TimeoutExpired as e:  # run() has killed the child
        raise AssertionError(f"{case}{args}: no result within {CASE_TIMEOUT} s\n{e.stdout or ''}\n{e.stderr or ''}")
    if p.returncode != 0 or "LOOPBACK CASE OK" not in p.stdout:
        raise AssertionError(f"{case}{args} failed (exit {p.returncode}):\n{(p.stdout + p.stderr)[-6000:]}")


@pytest.mark.parametrize("lists", ("uneven", "few"))
def test_ivf_matches_plain_index(lists):
    _run("case_ivf", lists, worlds=WORLDS if lists == "uneven" else (5, 8))


def test_flat_matches_plain_index():
    _run("case_flat")


@pytest.mark.parametrize("kind", (BINARY_FLAT, BINARY_IVF_FLAT))
def test_range_matches_plain_index(kind):
    _run("case_range", kind)


def test_delete():
    _run("case_delete")


def test_train():
    _run("case_train")


@pytest.mark.parametrize("kind", (BINARY_FLAT, BINARY_IVF_FLAT))
@pytest.mark.parametrize("worlds", ((3, 3), (3, 2), (2, 5)))
def test_snapshot(kind, worlds, tmp_path):
    W, W2 = worlds
    _run("case_snapshot", W2, kind, str(tmp_path / "snap"), worlds=(W,))


def test_snapshot_refusals(tmp_path):
    _run("case_snapshot_refusals", str(tmp_path / "snap"), worlds=(3,))


def _main():
    """The subprocess of one loopback case: mirrors shard_loopback._main, with this module's cases."""
    case, args, dump_after = sys.argv[1], json.loads(sys.argv[2]), int(sys.argv[3])
    faulthandler.dump_traceback_later(dump_after, exit=True)
    rc = 1
    try:
        globals()[case](*args)
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
