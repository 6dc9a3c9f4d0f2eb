"""Sharded deep top-k: b200vs_shard_search_deep / b200vs_shard_search_binary_deep on list-sharded IVF_FLAT, IVF_PQ and
BINARY_IVF_FLAT and row-sharded FLAT and BINARY_FLAT, for k up to B200VS_DEEP_MAX_K.

World 1 runs in this process (no NCCL).  Worlds 2, 3, 5 and 8 run as threads of one process on one GPU over the loopback
NCCL (tests/shard_loopback.py's World and run_world), each case in a subprocess of its own started through this file's
__main__.  The reference is always a plain index holding every row with the same trained state: distances and ids must equal
its search_deep bit for bit, and the sharded search wherever that answers."""
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
from b200vs import BINARY_FLAT, BINARY_IVF_FLAT, COSINE, FLAT, HAMMING, HNSW, IP, IVF_FLAT, IVF_PQ, L2  # noqa: E402
from gpu_util import require_gpu  # noqa: E402
from shard_loopback import LIB, run_world  # noqa: E402

pytestmark = pytest.mark.gpu
WORLDS = (2, 3, 5, 8)
CASE_TIMEOUT = 900  # seconds of one subprocess; every rendezvous of the loopback library times out after 60 s
KS = (1, 129, 4096, 4097, 8193, 40960)
D, PQ_M, BDIM = 32, 8, 64

# name -> (type, metric, IVF-PQ nbits)
KINDS = {
    "ivf_flat_l2": (IVF_FLAT, L2, 0), "ivf_flat_ip": (IVF_FLAT, IP, 0), "ivf_flat_cosine": (IVF_FLAT, COSINE, 0),
    "ivf_pq8_l2": (IVF_PQ, L2, 8), "ivf_pq8_ip": (IVF_PQ, IP, 8), "ivf_pq4_l2": (IVF_PQ, L2, 4), "ivf_pq4_ip": (IVF_PQ, IP, 4),
    "flat_l2": (FLAT, L2, 0), "flat_ip": (FLAT, IP, 0), "flat_cosine": (FLAT, COSINE, 0),
    "binary_ivf": (BINARY_IVF_FLAT, HAMMING, 0), "binary_flat": (BINARY_FLAT, HAMMING, 0),
}


@pytest.fixture(autouse=True)
def _gpu():
    require_gpu()


def _assert_same(got, want, what):
    assert not isinstance(got, int) and not isinstance(want, int), f"{what}: status {got} / {want}"
    for x, y in zip(got, want):
        assert x.shape == y.shape, f"{what}: shape {x.shape} != {y.shape}"
        bad = np.argwhere((x.view(np.uint32) if x.dtype == np.float32 else x) != (y.view(np.uint32) if y.dtype == np.float32 else y))
        assert bad.size == 0, f"{what}: differs at {bad[:4].tolist()}: got {x[tuple(bad[0])]}, want {y[tuple(bad[0])]}"


def _assert_same_up_to_api_ties(got, want, what):
    """Equal distances bit for bit, and the same ids inside every run of equal distances but the last one of a row (k may cut
    it): the order of b200vs_shard_search on a list-sharded IP / cosine index, whose merge keys on the API distance and so
    orders distinct inner products that round to one 1 - ip by id, where the deep path orders them by -ip."""
    _assert_same((got[0],), (want[0],), what)
    for q in range(got[0].shape[0]):
        d = got[0][q].view(np.uint32)
        starts = np.flatnonzero(np.r_[True, d[1:] != d[:-1]])
        for a, b in zip(starts[:-1], starts[1:]):
            assert np.array_equal(np.sort(got[1][q, a:b]), np.sort(want[1][q, a:b])), f"{what}: query {q} ids of slots [{a}, {b})"


def _status(fn):
    try:
        fn()
        return b200vs.OK
    except b200vs.B200VSError as e:
        return e.code


def _result(fn):
    """fn()'s results, or its status code when refused."""
    try:
        return fn()
    except b200vs.B200VSError as e:
        return e.code


def _pq_blob(cent, metric, nbits, rng):
    """An IVF-PQ trained-state blob: header, centroids [nlist, D], codebooks [M, 2^nbits, D / M]."""
    nlist, d = cent.shape
    cb = (rng.standard_normal((PQ_M, 1 << nbits, d // PQ_M)) * 0.5).astype(np.float32)
    hdr = np.array([0x51505649, nlist, d, metric, PQ_M, nbits], dtype=np.int64)
    return np.concatenate([hdr.view(np.uint8), np.ascontiguousarray(cent, np.float32).reshape(-1).view(np.uint8), cb.reshape(-1).view(np.uint8)])


class Kind:
    """One index kind with its trained state: fresh() makes an index of it, binary / lists tell its row format and sharding."""

    def __init__(self, name, nlist, sample, rng):
        self.t, self.metric, self.nbits = KINDS[name]
        self.binary = self.t in (BINARY_FLAT, BINARY_IVF_FLAT)
        self.lists = self.t in (IVF_FLAT, IVF_PQ, BINARY_IVF_FLAT)
        self.nlist = nlist
        self.dim = BDIM if self.binary else sample.shape[1]
        self.blob = None
        if self.lists:
            cent = sample[rng.choice(len(sample), nlist, replace=False)].copy()
            if self.t == IVF_FLAT:
                self.blob = b200vs.ivf_state_blob(cent, self.metric)
            elif self.t == IVF_PQ:
                self.blob = _pq_blob(cent, self.metric, self.nbits, rng)
            else:
                self.blob = b200vs.binary_ivf_state_blob(cent)

    def fresh(self):
        if self.t == IVF_PQ:
            ix = b200vs.Index(IVF_PQ, self.metric, self.dim, nlist=self.nlist, pq_m=PQ_M, pq_nbits=self.nbits)
        elif self.lists:
            ix = b200vs.Index(self.t, self.metric, self.dim, nlist=self.nlist)
        else:
            ix = b200vs.Index(self.t, self.metric, self.dim)
        if self.blob is not None:
            ix.set_trained_state(self.blob)
        return ix

    def rows(self, rng, n):
        if self.binary:
            return rng.integers(0, 256, (n, self.dim // 8), dtype=np.uint8)
        return rng.standard_normal((n, self.dim)).astype(np.float32)


def _connect(world, ix, rank):
    """The shard of rank `rank`: world None is a world of one, with no communicator."""
    cls = b200vs.BinaryShard if ix.binary else b200vs.Shard
    if world is None:
        return cls(ix, 0, 1, None)
    idb = world.gather(rank, b200vs.Shard.unique_id() if rank == 0 else None)[0]
    return cls(ix, rank, world.W, idb)


def _ranks(W, fn):
    return [fn(0, None)] if W == 1 else run_world(W, fn)


def _split(W, *arrays):
    """Rows each rank sends: uneven contiguous parts, growing with the rank."""
    n = len(arrays[0])
    cuts = [0] + [int(n * (r * r) / (W * W)) for r in range(1, W)] + [n]
    return [[a[cuts[r]:cuts[r + 1]] for a in arrays] for r in range(W)]


# ---------------------------------------------------------------------------------------------
# every kind at every k: padding past the eligible rows, equality with search_deep and shard.search
# ---------------------------------------------------------------------------------------------
def case_kind(W, name):
    rng = np.random.default_rng(sorted(KINDS).index(name) + 17)
    t = KINDS[name][0]
    n = 12000
    sample = (rng.integers(0, 256, (n, BDIM // 8), dtype=np.uint8) if t in (BINARY_FLAT, BINARY_IVF_FLAT)
              else rng.standard_normal((n, D)).astype(np.float32))
    kind = Kind(name, 16, sample, rng)
    x = sample
    ids = rng.permutation(4 * n)[:n].astype(np.int64) + 5
    xq = kind.rows(rng, 3)
    kw = dict(nprobe=5) if kind.lists else {}
    plain = kind.fresh()
    plain.add(x, ids)
    want = {k: plain.search_deep(xq, k, **kw) for k in KS}
    assert (want[40960][1] == -1).any() and (want[40960][1][:, 0] >= 0).all()
    parts = _split(W, x, ids)

    def rank(r, world):
        ix = kind.fresh()
        sh = _connect(world, ix, r)
        sh.add(*parts[r])
        out = {}
        for k in KS:
            out[k] = sh.search_deep(xq, k, **kw)
            if k <= 4096:
                out[("search", k)] = _result(lambda: sh.search(xq, k, **kw))
        sh.close()
        return out

    for r, o in enumerate(_ranks(W, rank)):
        for k in KS:
            _assert_same(o[k], want[k], f"{name} rank {r} k {k}")
            s = o.get(("search", k))
            if s is None or isinstance(s, int):
                continue
            if kind.lists and not kind.binary and kind.metric != L2:
                _assert_same_up_to_api_ties(s, o[k], f"{name} rank {r} k {k}: shard_search vs deep")
            else:
                _assert_same(o[k], s, f"{name} rank {r} k {k}: deep vs shard_search")


# ---------------------------------------------------------------------------------------------
# edges: filters, nprobe = nlist, ranks without lists, nlist % W != 0, tombstones, upserts, a repeated id, non-finite rows
# ---------------------------------------------------------------------------------------------
FILTERS = [dict(), dict(id_range=(300, 4000)), dict(sorted_ids=np.arange(2, 9000, 3)), dict(sorted_ids=np.arange(2, 9000, 3), negate=True)]


def case_ivf_edges(W, lists):
    """IVF_FLAT L2: nlist 3 (< W from W = 5: ranks that own no list) or 2W + 1 (nlist % W != 0)."""
    nlist = 3 if lists == "few" else 2 * W + 1
    rng = np.random.default_rng(300 + W + nlist)
    n = 6000
    x = rng.standard_normal((n, 16)).astype(np.float32)
    ids = rng.permutation(n).astype(np.int64) + 1
    cent = x[rng.choice(n, nlist, replace=False)].copy()
    blob = b200vs.ivf_state_blob(cent, L2)
    dead = ids[::7]
    up_ids = ids[1::11][:300]
    up_x = rng.standard_normal((len(up_ids), 16)).astype(np.float32)
    dup = np.array([10 ** 7], np.int64)  # one id, two rows: list 0 (rank 0) and list nlist - 1 (another rank when W > 1)
    xq = rng.standard_normal((4, 16)).astype(np.float32)
    xq[0] = cent[0]
    plain = b200vs.Index(IVF_FLAT, L2, 16, nlist=nlist)
    plain.set_trained_state(blob)
    plain.add(x, ids)
    plain.delete(dead)
    plain.delete(up_ids)
    plain.add(up_x, up_ids)
    plain.add(cent[:1], dup)
    plain.add(cent[-1:], dup)
    calls = [(nprobe, k, j) for nprobe in (2, nlist) for k in (100, 5000) for j in range(len(FILTERS))]
    want = {c: plain.search_deep(xq, c[1], nprobe=c[0], **FILTERS[c[2]]) for c in calls}
    parts = _split(W, x, ids)

    def rank(r, world):
        ix = b200vs.Index(IVF_FLAT, L2, 16, nlist=nlist)
        ix.set_trained_state(blob)
        sh = _connect(world, ix, r)
        sh.add(*parts[r])
        sh.delete(dead)
        sh.delete(up_ids)
        last = r == W - 1
        sh.add(up_x if last else up_x[:0], up_ids if last else up_ids[:0])
        sh.add(cent[:1] if r == 0 else cent[:0], dup if r == 0 else dup[:0])
        sh.add(cent[-1:] if last else cent[:0], dup if last else dup[:0])
        out = {c: sh.search_deep(xq, c[1], nprobe=c[0], **FILTERS[c[2]]) for c in calls}
        sh.close()
        return out

    for r, o in enumerate(_ranks(W, rank)):
        for c, w in want.items():
            _assert_same(o[c], w, f"rank {r} (nprobe, k, filter) {c}")
    assert (want[(nlist, 5000, 0)][1] == dup[0]).any()


def case_flat_edges(W, metric):
    """Row-sharded FLAT: non-finite rows, tombstones, upserts (delete + add on the shard), every filter."""
    rng = np.random.default_rng(400 + W + metric)
    n, d = 7000, 16
    x = rng.standard_normal((n, d)).astype(np.float32)
    x[::7, 3] = np.inf
    x[::11, 5] = np.nan
    x[::13] *= np.float32(3e38)
    x[::17, 0] = -np.inf
    ids = np.arange(n, dtype=np.int64)
    dead = ids[::5]
    up_ids = ids[1::9][:500]
    up_x = rng.standard_normal((len(up_ids), d)).astype(np.float32)
    xq = rng.standard_normal((3, d)).astype(np.float32)
    xq[1, 2] = 1e30
    plain = b200vs.Index(FLAT, metric, d)
    plain.add(x, ids)
    plain.delete(dead)
    plain.add(up_x, up_ids, upsert=True)
    calls = [(k, j) for k in (129, 4097, 9000) for j in range(len(FILTERS))]
    want = {c: plain.search_deep(xq, c[0], **FILTERS[c[1]]) for c in calls}
    parts = _split(W, x, ids)

    def rank(r, world):
        ix = b200vs.Index(FLAT, metric, d)
        sh = _connect(world, ix, r)
        sh.add(*parts[r])
        sh.delete(dead)
        sh.delete(up_ids)
        sh.add(up_x if r == 0 else up_x[:0], up_ids if r == 0 else up_ids[:0])
        out = {c: sh.search_deep(xq, c[0], **FILTERS[c[1]]) for c in calls}
        sh.close()
        return out

    for r, o in enumerate(_ranks(W, rank)):
        for c, w in want.items():
            _assert_same(o[c], w, f"rank {r} (k, filter) {c}")


# ---------------------------------------------------------------------------------------------
# keys: exact ties across ranks resolve by id; IP keys that share one 1 - ip order by -ip, not by id
# ---------------------------------------------------------------------------------------------
def case_ties(W, t):
    """0/1 rows of 4 dimensions: every distance is shared by hundreds of rows; ids interleave across the sending ranks."""
    rng = np.random.default_rng(500 + W + t)
    n, d, nlist = 3000, 4, 2 * W
    x = rng.integers(0, 2, (n, d)).astype(np.float32)
    ids = np.arange(n, dtype=np.int64)  # rank r sends the ids r, r + W, r + 2W, ...
    blob = b200vs.ivf_state_blob(rng.integers(0, 2, (nlist, d)).astype(np.float32) + 0.01 * np.arange(nlist)[:, None], L2) if t == IVF_FLAT else None
    xq = rng.integers(0, 2, (3, d)).astype(np.float32)
    kw = dict(nprobe=nlist) if t == IVF_FLAT else {}

    def fresh():
        ix = b200vs.Index(t, L2, d, nlist=nlist) if t == IVF_FLAT else b200vs.Index(t, L2, d)
        if blob is not None:
            ix.set_trained_state(blob)
        return ix

    plain = fresh()
    plain.add(x, ids)
    ks = (1, 100, 1000, 2999, 5000)
    want = {k: plain.search_deep(xq, k, **kw) for k in ks}
    parts = [(x[r::W], ids[r::W]) for r in range(W)]

    def rank(r, world):
        ix = fresh()
        sh = _connect(world, ix, r)
        sh.add(*parts[r])
        out = {k: sh.search_deep(xq, k, **kw) for k in ks}
        sh.close()
        return out

    for r, o in enumerate(_ranks(W, rank)):
        for k in ks:
            _assert_same(o[k], want[k], f"rank {r} k {k}")


def case_ip_keys(W, t):
    """Rows (ip_i, cos a_j, sin a_j, 0) against the query (1, 0, 0, 0): ip = ip_i exactly, distinct, all below 2^-25, so every
    API distance 1 - ip rounds to 1.  The larger ip, the better result, has the larger id, and the rows of each list (a_j
    points at centroid j) sit on different ranks.  A merge on the API distance would return the smallest ids instead."""
    n, nlist = 400, 2 * W
    ipv = (np.arange(1, n + 1) * 5e-11).astype(np.float32)
    j = np.arange(n) % nlist
    a = 2 * np.pi * np.arange(nlist) / nlist
    x = np.stack([ipv, np.cos(a[j]), np.sin(a[j]), np.zeros(n)], 1).astype(np.float32)
    ids = np.arange(n, dtype=np.int64) + 1
    cent = np.stack([np.zeros(nlist), np.cos(a), np.sin(a), np.zeros(nlist)], 1).astype(np.float32)
    xq = np.array([[1, 0, 0, 0]], np.float32)
    kw = dict(nprobe=nlist) if t == IVF_FLAT else {}

    def fresh():
        if t == FLAT:
            return b200vs.Index(FLAT, IP, 4)
        ix = b200vs.Index(IVF_FLAT, IP, 4, nlist=nlist)
        ix.set_trained_state(b200vs.ivf_state_blob(cent, IP))
        return ix

    plain = fresh()
    plain.add(x, ids)
    ks = (1, 3, 50, 300, 4097)
    want = {k: plain.search_deep(xq, k, **kw) for k in ks}
    assert (want[300][0] == 1.0).all() and want[300][1][0, 0] == n, "the construction must share one API distance"
    parts = _split(W, x, ids)

    def rank(r, world):
        ix = fresh()
        sh = _connect(world, ix, r)
        sh.add(*parts[r])
        out = {k: sh.search_deep(xq, k, **kw) for k in ks}
        sh.close()
        return out

    for r, o in enumerate(_ranks(W, rank)):
        for k in ks:
            _assert_same(o[k], want[k], f"rank {r} k {k}")


# ---------------------------------------------------------------------------------------------
# gather chunking: W = 8, k = 40960, nq = 256 gathers 8 * 256 * 40960 * 16 B = 1.25 GiB per rank, more than one 1 GiB chunk
# ---------------------------------------------------------------------------------------------
def case_chunks(W):
    rng = np.random.default_rng(600 + W)
    n, d = 5000, 8
    x = rng.standard_normal((n, d)).astype(np.float32)
    ids = np.arange(n, dtype=np.int64)
    xq = rng.standard_normal((256, d)).astype(np.float32)
    plain = b200vs.Index(FLAT, L2, d)
    plain.add(x, ids)
    want = plain.search_deep(xq, 40960)
    parts = _split(W, x, ids)

    def rank(r, world):
        ix = b200vs.Index(FLAT, L2, d)
        sh = _connect(world, ix, r)
        sh.add(*parts[r])
        out = sh.search_deep(xq, 40960)
        sh.close()
        return out

    for r, o in enumerate(_ranks(W, rank)):
        _assert_same(o, want, f"rank {r}")


# ---------------------------------------------------------------------------------------------
# sequencing: deep, top-k and range batches interleaved on one sequence, enqueued from threads started out of order
# ---------------------------------------------------------------------------------------------
def case_sequence(W):
    rng = np.random.default_rng(700 + W)
    n, d, nlist = 8000, 16, 2 * W + 1
    x = rng.standard_normal((n, d)).astype(np.float32)
    ids = np.arange(n, dtype=np.int64) * 3
    blob = b200vs.ivf_state_blob(x[rng.choice(n, nlist, replace=False)], L2)
    xq = rng.standard_normal((5, d)).astype(np.float32)
    plain = b200vs.Index(IVF_FLAT, L2, d, nlist=nlist)
    plain.set_trained_state(blob)
    plain.add(x, ids)
    ops = [("deep", 5000), ("search", 10), ("range", 12.0), ("deep", 40960), ("search", 4096), ("range", 20.0)]

    def call(ix, op, arg, seq=-1):
        if op == "deep":
            return ix.search_deep(xq, arg, nprobe=4, **({"seq": seq} if seq >= 0 else {}))
        if op == "search":
            return ix.search(xq, arg, nprobe=4, **({"seq": seq} if seq >= 0 else {}))
        return ix.range_search(xq, arg, 64, nprobe=4, **({"seq": seq} if seq >= 0 else {}))

    want = [call(plain, op, arg) for op, arg in ops]
    parts = _split(W, x, ids)

    def rank(r, world):
        ix = b200vs.Index(IVF_FLAT, L2, d, nlist=nlist)
        ix.set_trained_state(blob)
        sh = _connect(world, ix, r)
        sh.add(*parts[r])
        got = {}

        def one(s):
            got[s] = call(sh, *ops[s], seq=s)
        ths = [threading.Thread(target=one, args=(s,)) for s in (2, 0, 5, 3, 1, 4)]
        for th in ths:
            th.start()
        for th in ths:
            th.join()
        sh.close()
        return [got.get(s) for s in range(len(ops))]

    for r, o in enumerate(_ranks(W, rank)):
        for s, w in enumerate(want):
            assert o[s] is not None, f"rank {r}: batch {s} did not return"
            _assert_same(o[s], w, f"rank {r} batch {s} {ops[s]}")


# ---------------------------------------------------------------------------------------------
# refusals: the same status on every rank, before the first collective; the sequence number is used up
# ---------------------------------------------------------------------------------------------
def case_refusals(W):
    rng = np.random.default_rng(800 + W)
    n, d, nlist = 3000, 16, 2 * W
    x = rng.standard_normal((n, d)).astype(np.float32)
    ids = np.arange(n, dtype=np.int64)
    blob = b200vs.ivf_state_blob(x[:nlist], L2)
    xq = rng.standard_normal((2, d)).astype(np.float32)
    plain = b200vs.Index(IVF_FLAT, L2, d, nlist=nlist)
    plain.set_trained_state(blob)
    plain.add(x, ids)
    want = plain.search_deep(xq, 3000, nprobe=nlist)
    bx = rng.integers(0, 256, (n, BDIM // 8), dtype=np.uint8)
    bq = bx[:2]
    bplain = b200vs.Index(BINARY_FLAT, HAMMING, BDIM)
    bplain.add(bx, ids)
    bwant = bplain.search_deep(bq, 5000)
    # an IVF-PQ state whose LUT alone (256 sub-quantisers x 256 codes x 4 B = 256 KB) exceeds one SM's 227 KB
    pq_cent = x[:nlist, :1].repeat(256, 1)
    pq_hdr = np.array([0x51505649, nlist, 256, L2, 256, 8], dtype=np.int64)
    pq_blob = np.concatenate([pq_hdr.view(np.uint8), pq_cent.reshape(-1).view(np.uint8),
                              rng.standard_normal(256 * 256).astype(np.float32).view(np.uint8)])
    parts = _split(W, x, ids)
    bparts = _split(W, bx, ids)
    L = b200vs.lib()
    od, oi = np.zeros((2, 10), np.float32), np.zeros((2, 10), np.int64)

    def rank(r, world):
        out = {}
        ix = b200vs.Index(IVF_FLAT, L2, d, nlist=nlist)
        ix.set_trained_state(blob)
        sh = _connect(world, ix, r)
        sh.add(*parts[r])
        out["k"] = _status(lambda: sh.search_deep(xq, b200vs.DEEP_MAX_K + 1, seq=0))
        out["null"] = L.b200vs_shard_search_deep(sh.h, 1, 2, xq.ctypes.data, 10, None, None, None)
        out["binary_call"] = L.b200vs_shard_search_binary_deep(sh.h, 2, 2, bq.ctypes.data, 10, None, od.ctypes.data, oi.ctypes.data)
        out["k0"] = sh.search_deep(xq, 0, seq=3)[1].shape
        out["after"] = sh.search_deep(xq, 3000, seq=4, nprobe=nlist)
        sh.close()
        bix = b200vs.Index(BINARY_FLAT, HAMMING, BDIM)
        bsh = _connect(world, bix, r)
        bsh.add(*bparts[r])
        out["float_call"] = L.b200vs_shard_search_deep(bsh.h, 0, 2, xq.ctypes.data, 10, None, od.ctypes.data, oi.ctypes.data)
        out["b_after"] = bsh.search_deep(bq, 5000, seq=1)
        bsh.close()
        pq = b200vs.Index(IVF_PQ, L2, 256, nlist=nlist, pq_m=256, pq_nbits=8)
        pq.set_trained_state(pq_blob)
        psh = _connect(world, pq, r)
        out["lut"] = _status(lambda: psh.search_deep(np.zeros((1, 256), np.float32), 10, seq=0))
        out["lut_after"] = _status(lambda: psh.search_deep(np.zeros((1, 256), np.float32), 10, seq=1))
        psh.close()
        hn = b200vs.Index(HNSW, L2, d, hnsw_m=16, hnsw_efc=64, max_elements=4000)
        hsh = _connect(world, hn, r)
        hsh.add(*parts[r])
        out["hnsw"] = _status(lambda: hsh.search_deep(xq, 5000, seq=0))
        out["hnsw_after"] = hsh.search(xq, 10, seq=1)
        hsh.close()
        return out

    for r, o in enumerate(_ranks(W, rank)):
        assert o["k"] == b200vs.EILLEGAL_PARAMETERS, f"rank {r}: k above the maximum returned {o['k']}"
        assert o["null"] == b200vs.EILLEGAL_PARAMETERS, f"rank {r}: null outputs returned {o['null']}"
        assert o["binary_call"] == b200vs.EILLEGAL_PARAMETERS, f"rank {r}: binary call on a float shard returned {o['binary_call']}"
        assert o["float_call"] == b200vs.EILLEGAL_PARAMETERS, f"rank {r}: float call on a binary shard returned {o['float_call']}"
        assert o["k0"] == (2, 0)
        assert o["lut"] == b200vs.EILLEGAL_PARAMETERS and o["lut_after"] == b200vs.EILLEGAL_PARAMETERS, f"rank {r}: LUT refusal {o['lut']}"
        assert o["hnsw"] == b200vs.EVECTOR_NOT_SUPPORT, f"rank {r}: HNSW returned {o['hnsw']}"
        assert (o["hnsw_after"][1] >= 0).all(), f"rank {r}: HNSW shard stopped answering"
        _assert_same(o["after"], want, f"rank {r}: the batch after the refusals")
        _assert_same(o["b_after"], bwant, f"rank {r}: the binary batch after the refusal")


# ---------------------------------------------------------------------------------------------
# tests: world 1 in this process, worlds 2, 3, 5, 8 in a loopback subprocess
# ---------------------------------------------------------------------------------------------
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


@pytest.mark.parametrize("name", sorted(KINDS))
def test_world1_kind(name):
    case_kind(1, name)


@pytest.mark.parametrize("name", sorted(KINDS))
def test_kind(name):
    _run("case_kind", name)


def test_world1_edges():
    for lists in ("few", "uneven"):
        case_ivf_edges(1, lists)
    for metric in (L2, IP):
        case_flat_edges(1, metric)
    for t in (FLAT, IVF_FLAT):
        case_ties(1, t)
        case_ip_keys(1, t)
    case_sequence(1)
    case_refusals(1)


@pytest.mark.parametrize("lists", ("few", "uneven"))
def test_ivf_edges(lists):
    _run("case_ivf_edges", lists)


@pytest.mark.parametrize("metric", (L2, IP))
def test_flat_edges(metric):
    _run("case_flat_edges", metric)


@pytest.mark.parametrize("t", (FLAT, IVF_FLAT))
def test_ties_across_ranks(t):
    _run("case_ties", t)


@pytest.mark.parametrize("t", (FLAT, IVF_FLAT))
def test_ip_keys_across_ranks(t):
    _run("case_ip_keys", t)


def test_gather_chunks():
    _run("case_chunks", worlds=(8,))


def test_sequence():
    _run("case_sequence")


def test_refusals():
    _run("case_refusals")


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
