"""Sharded rebuilds: b200vs_shard_need_rebuild (the NeedToRebuild rule over a whole set) and b200vs_shard_rebuild_from (a
collective GPU rebuild of a fresh set from the old set's device rows).

World 1 runs in this process (no NCCL).  Worlds 2, 3 and 5 run as threads of one process on one GPU over the loopback NCCL
(tests/shard_loopback.py's World and run_world), each case in a subprocess of its own started through this file's __main__.
References: at world 1, b200vs_rebuild_from of the same source index; list-sharded sets at world > 1, a fresh shard fed from
the host with shard_train + shard_add of each rank's rows_r; row-sharded HNSW, b200vs_rebuild_from of each rank's index."""
import faulthandler
import json
import os
import shutil
import subprocess
import sys
import tempfile
import threading
import time

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, os.path.join(ROOT, "dingo-store_b200", "python"))
sys.path.insert(0, HERE)

import b200vs  # noqa: E402
from b200vs import (BINARY_FLAT, BINARY_IVF_FLAT, COSINE, EILLEGAL_PARAMETERS, EVECTOR_NOT_SUPPORT, FLAT, HAMMING, HNSW, IP,  # noqa: E402
                    IVF_FLAT, IVF_PQ, L2)
from b200vs.shard import merge_topk, row_owner  # noqa: E402
from gpu_util import require_gpu  # noqa: E402
from shard_loopback import LIB, run_world  # noqa: E402

pytestmark = pytest.mark.gpu
CASE_TIMEOUT = 900  # seconds of one subprocess; every rendezvous of the loopback library times out after 60 s
D, BDIM = 32, 48  # BDIM: 6 bytes per packed row, 2 padded words on the device
TIES = 24  # ids that every rank adds once, each rank's copy a different row


@pytest.fixture(autouse=True)
def _gpu():
    require_gpu()


def _eq(a, b, what):
    if isinstance(a, tuple):
        for x, y in zip(a, b):
            _eq(x, y, what)
        return
    if a is None or b is None:
        assert a is None and b is None, what
        return
    assert a.shape == b.shape, f"{what}: shape {a.shape} != {b.shape}"
    x = a.view(np.uint32) if a.dtype == np.float32 else a
    y = b.view(np.uint32) if b.dtype == np.float32 else b
    bad = np.argwhere(x != y)
    assert bad.size == 0, f"{what}: differs at {bad[:4].tolist()}"


def _status(fn):
    try:
        fn()
        return b200vs.OK
    except b200vs.B200VSError as e:
        return e.code


def _connect(world, ix, rank, lanes=2):
    """The shard of rank `rank`: world None is a world of one, with no communicator."""
    cls = b200vs.BinaryShard if ix.binary else b200vs.Shard
    if world is None:
        return cls(ix, 0, 1, None, lanes=lanes)
    idb = world.gather(rank, b200vs.Shard.unique_id() if rank == 0 else None)[0]
    return cls(ix, rank, world.W, idb, lanes=lanes)


def _ranks(W, fn):
    return [fn(0, None)] if W == 1 else run_world(W, fn)


def _gather(world, rank, v):
    return [v] if world is None else world.gather(rank, v)


def _split(W, n):
    """Uneven contiguous parts of [0, n), growing with the rank."""
    cuts = [0] + [int(n * (r * r) / (W * W)) for r in range(1, W)] + [n]
    return [slice(cuts[r], cuts[r + 1]) for r in range(W)]


def _index(t, metric, dim, nlist=0, **kw):
    if t in (IVF_FLAT, BINARY_IVF_FLAT, IVF_PQ):
        return b200vs.Index(t, metric, dim, nlist=nlist, **kw)
    return b200vs.Index(t, metric, dim, **kw)


def _export(ix, nlist):
    off, vec, codes, ids = ix.export_lists(nlist)
    return off, (codes if ix.binary else vec), ids


def _rows(rng, binary, n):
    if binary:
        return rng.integers(0, 256, (n, BDIM // 8), dtype=np.uint8)
    return rng.standard_normal((n, D)).astype(np.float32)


# ---------------------------------------------------------------------------------------------
# 1. world 1, every type: equal to b200vs_rebuild_from of the same source index
# ---------------------------------------------------------------------------------------------
W1_KINDS = {"ivf_flat_l2": (IVF_FLAT, L2), "ivf_flat_ip": (IVF_FLAT, IP), "ivf_flat_cosine": (IVF_FLAT, COSINE),
            "binary_ivf": (BINARY_IVF_FLAT, HAMMING), "hnsw_l2": (HNSW, L2), "hnsw_cosine": (HNSW, COSINE)}


@pytest.mark.parametrize("name", sorted(W1_KINDS))
def test_world1_equals_single_rebuild(name):
    t, metric = W1_KINDS[name]
    rng = np.random.default_rng(sorted(W1_KINDS).index(name) + 3)
    binary, lists = t == BINARY_IVF_FLAT, t != HNSW
    nlist = 8
    kw = dict(hnsw_m=16, hnsw_efc=64, max_elements=20000) if t == HNSW else {}
    dim = BDIM if binary else D
    n = 5000
    x = _rows(rng, binary, n)
    ids = rng.permutation(3 * n)[:n].astype(np.int64)
    src_ix = _index(t, metric, dim, nlist, **kw)
    src = _connect(None, src_ix, 0)
    if lists:
        src.train(x[:300])
    src.add(x, ids)
    src.delete(ids[::3])
    up = ids[1::7]  # upserts: a delete, then an add of new rows under the same ids
    src.delete(up)
    src.add(_rows(rng, binary, up.size), up)
    if lists:
        src.add(x[:5], ids[1:6])  # repeated ids
    dst_ix = _index(t, metric, dim, nlist, **kw)
    dst = _connect(None, dst_ix, 0)
    n_rows = dst.rebuild_from(src)
    one = _index(t, metric, dim, nlist, **kw)
    want_n = one.rebuild_from(src_ix)
    assert n_rows == want_n == one.get_count() == dst_ix.get_count() > 0
    assert dst_ix.get_deleted_count() == 0
    _eq(dst_ix.get_trained_state(), one.get_trained_state(), "trained state / graph")
    xq = _rows(rng, binary, 7)
    if lists:
        _eq(_export(dst_ix, nlist), _export(one, nlist), "lists")
        ref = _connect(None, one, 0)
        for kw_s in ({}, {"nprobe": 3}):
            _eq(dst.search(xq, 10, **kw_s), ref.search(xq, 10, **kw_s), f"search {kw_s}")
            _eq(dst.search_deep(xq, 300, **kw_s), ref.search_deep(xq, 300, **kw_s), f"deep {kw_s}")
        radius = 20.0 if binary else (40.0 if metric == L2 else 0.5)
        _eq(dst.range_search(xq, radius, 64, nprobe=4), ref.range_search(xq, radius, 64, nprobe=4), "range")
        ref.close()
    else:
        _eq(dst.search(xq, 10, efsearch=64), one.search(xq, 10, efsearch=64), "search")
    assert not dst.need_rebuild()
    dst.close()
    src.close()


def test_world1_empty_src_leaves_dst_untrained():
    src = _connect(None, b200vs.Index(IVF_FLAT, L2, D, nlist=4), 0)
    dst_ix = b200vs.Index(IVF_FLAT, L2, D, nlist=4)
    dst = _connect(None, dst_ix, 0)
    assert dst.rebuild_from(src) == 0
    assert not dst_ix.is_trained() and dst_ix.get_count() == 0
    assert not dst.need_rebuild()


# ---------------------------------------------------------------------------------------------
# 2. list-sharded types at world > 1: byte-equal to the host-fed reference
# ---------------------------------------------------------------------------------------------
# name -> (type, metric, skewed: every live row sits in rank 0's lists)
LIST_KINDS = {"ivf_l2": (IVF_FLAT, L2, False), "ivf_cosine": (IVF_FLAT, COSINE, False), "ivf_ip_skewed": (IVF_FLAT, IP, True),
              "binary": (BINARY_IVF_FLAT, HAMMING, False), "binary_skewed": (BINARY_IVF_FLAT, HAMMING, True)}


def case_lists(W, name):
    t, metric, skewed = LIST_KINDS[name]
    binary = t == BINARY_IVF_FLAT
    rng = np.random.default_rng(sorted(LIST_KINDS).index(name) * 10 + W)
    nlist = 4 * W
    dim = BDIM if binary else D
    n = 1500 * W
    cent = _rows(rng, binary, nlist)
    if skewed:  # rows near centroid 0: rank 0's list 0 takes them all, every other list and rank stays empty
        if binary:
            x = np.repeat(cent[:1], n, axis=0)
            x[np.arange(n), rng.integers(0, BDIM // 8, n)] ^= 1
        else:
            cent[0] *= 30.0 if metric != L2 else 1.0
            x = (cent[:1] + 0.01 * rng.standard_normal((n, dim))).astype(np.float32)
    else:
        x = _rows(rng, binary, n)
    ids = rng.permutation(4 * n)[:n].astype(np.int64)
    blob = b200vs.binary_ivf_state_blob(cent) if binary else b200vs.ivf_state_blob(cent, metric)
    parts = _split(W, n)
    xq = _rows(rng, binary, 9)
    up = ids[2::11]
    up_x = x[rng.permutation(n)[:up.size]]
    ties = not skewed and metric in (L2, HAMMING)
    tie_ids = 10 ** 7 + np.arange(TIES, dtype=np.int64)

    def rank(r, world):
        src_ix = _index(t, metric, dim, nlist)
        if skewed:
            src_ix.set_trained_state(blob)
        src = _connect(world, src_ix, r)
        if not skewed:
            src.train(x[parts[r]][: max(nlist, len(x[parts[r]]) // 2)])
        src.add(x[parts[r]], ids[parts[r]])
        src.delete(ids[::4])
        src.delete(up)
        src.add(up_x[r::W], up[r::W])
        src.add(x[parts[r]][:3], ids[parts[r]][:3])  # repeated ids, on the rank that already sent them
        if ties:  # ids whose copies hold different rows in different ranks' lists: rank r's copy sits on a centroid r owns
            st = src_ix.get_trained_state()[32:]
            c = st.reshape(nlist, dim // 8) if binary else st.view(np.float32).reshape(nlist, dim)
            row = c[r * (nlist // W)][None]
            copies = np.repeat(row, TIES, axis=0)
            if not binary:
                copies = (copies + 1e-4 * rng.standard_normal(copies.shape)).astype(np.float32)
            src.add(copies, tie_ids)
        exp = _export(src_ix, nlist)
        all_exp = _gather(world, r, exp)
        if ties:
            assert all(np.isin(tie_ids, e[2]).all() for e in all_exp), "a tied id is missing from some rank's lists"
        # rows_r in numpy: every rank's live rows in rank order and list-major export order, stable by id, owner r
        all_ids = np.concatenate([e[2] for e in all_exp])
        all_x = np.concatenate([e[1] for e in all_exp])
        order = np.argsort(all_ids, kind="stable")
        mine = order[row_owner(all_ids[order], W) == r]
        rows_r, ids_r = all_x[mine], all_ids[mine]
        ref_ix = _index(t, metric, dim, nlist)
        ref = _connect(world, ref_ix, r)
        ref.train(rows_r)
        ref.add(rows_r, ids_r)
        dst_ix = _index(t, metric, dim, nlist)
        dst = _connect(world, dst_ix, r)
        need_before = src_ix.need_rebuild()
        n_rows = dst.rebuild_from(src)
        out = dict(n_rows=n_rows, count=dst_ix.get_count(), live=src_ix.get_count(), src_lists=len(exp[2]),
                   same_state=np.array_equal(dst_ix.get_trained_state(), ref_ix.get_trained_state()),
                   dst=_export(dst_ix, nlist), ref=_export(ref_ix, nlist), src_after=_export(src_ix, nlist), src_before=exp,
                   search=dst.search(xq, 10, nprobe=3), ref_search=ref.search(xq, 10, nprobe=3),
                   deep=dst.search_deep(xq, 200), ref_deep=ref.search_deep(xq, 200),
                   need=dst.need_rebuild(), src_need=(need_before, src_ix.need_rebuild()))
        for s in (dst, ref, src):
            s.close()
        return out

    outs = _ranks(W, rank)
    total = sum(o["live"] for o in outs)
    assert sum(o["n_rows"] for o in outs) == total > 0
    if skewed:
        assert all(o["src_lists"] == 0 for o in outs[1:]), "the skewed set has rows outside rank 0"
    for r, o in enumerate(outs):
        assert o["n_rows"] == o["count"], f"rank {r}: n_rows {o['n_rows']} != dst count {o['count']}"
        assert o["same_state"], f"{name} rank {r}: trained state differs from the host-fed reference"
        _eq(o["dst"], o["ref"], f"{name} rank {r}: lists")
        _eq(o["src_after"], o["src_before"], f"{name} rank {r}: src changed")
        _eq(o["search"], o["ref_search"], f"{name} rank {r}: search")
        _eq(o["deep"], o["ref_deep"], f"{name} rank {r}: deep search")
        assert not o["need"], f"rank {r}: dst asks for a rebuild right after one"
        assert o["src_need"][0] == o["src_need"][1]


# ---------------------------------------------------------------------------------------------
# 3. row-sharded HNSW at world > 1: each rank's graph is b200vs_rebuild_from of its src index
# ---------------------------------------------------------------------------------------------
def case_hnsw(W, metric):
    rng = np.random.default_rng(W + 100 * metric)
    n = 1200 * W
    x = rng.standard_normal((n, D)).astype(np.float32)
    ids = rng.permutation(3 * n)[:n].astype(np.int64)
    kw = dict(hnsw_m=16, hnsw_efc=64, max_elements=4 * n)
    parts = _split(W, n)
    xq = rng.standard_normal((8, D)).astype(np.float32)
    k = 10

    def rank(r, world):
        src_ix = b200vs.Index(HNSW, metric, D, **kw)
        src = _connect(world, src_ix, r)
        src.add(x[parts[r]], ids[parts[r]])
        up = ids[n // 2::9]  # upserts: a delete, then an add of new rows under the same ids
        src.delete(up)
        src.add(x[: up.size][r::W], up[r::W])
        src.delete(ids[: n // 2])  # then half the rows tombstoned
        dst_ix = b200vs.Index(HNSW, metric, D, **kw)
        dst = _connect(world, dst_ix, r)
        n_rows = dst.rebuild_from(src)
        out = dict(n_rows=n_rows, src_ix=src_ix, dst_ix=dst_ix, search=dst.search(xq, k, efsearch=64))
        dst.close()
        src.close()
        return out

    outs = _ranks(W, rank)
    # the references, one rank index at a time in this thread: its own rebuild_from, and the merge of per-rank searches
    local = [o["dst_ix"].search(xq, k, efsearch=64) for o in outs]
    merged = merge_topk(np.stack([p[0] for p in local]), np.stack([p[1] for p in local]), k)
    for r, o in enumerate(outs):
        one = b200vs.Index(HNSW, metric, D, **kw)
        assert o["n_rows"] == one.rebuild_from(o["src_ix"]), f"rank {r}: n_rows"
        assert np.array_equal(o["dst_ix"].get_trained_state(), one.get_trained_state()), \
            f"rank {r}: graph differs from b200vs_rebuild_from of the rank's index"
        assert o["dst_ix"].get_deleted_count() == 0, f"rank {r}: tombstones left"
        _eq(o["search"], merged, f"rank {r}: shard_search vs the merge of per-rank searches")


# ---------------------------------------------------------------------------------------------
# 4. the set's NeedToRebuild rule
# ---------------------------------------------------------------------------------------------
def _need(world, r, sh, ix):
    """The set's answer, checked equal on every rank, with the rank index's own answer unchanged by the call."""
    before = ix.need_rebuild()
    got = sh.need_rebuild()
    assert ix.need_rebuild() == before, f"rank {r}: b200vs_need_rebuild changed"
    answers = _gather(world, r, got)
    assert len(set(answers)) == 1, f"ranks disagree: {answers}"
    return got, before


def case_need(W):
    rng = np.random.default_rng(7 + W)
    nlist = 2 * W
    tmp = tempfile.mkdtemp(prefix="b200vs_need_")

    def rank(r, world):
        log = {}
        # IVF_FLAT trained on few rows, grown past 256 * nlist and 2 * train_rows_set
        ix = b200vs.Index(IVF_FLAT, L2, D, nlist=nlist)
        sh = _connect(world, ix, r)
        log["untrained"] = _need(world, r, sh, ix)[0]
        sh.train(rng.standard_normal((100, D)).astype(np.float32))
        grow = 256 * nlist // W + 1
        base = r * 10 ** 6
        sh.add(rng.standard_normal((grow - 10, D)).astype(np.float32), base + np.arange(grow - 10))
        log["short"] = _need(world, r, sh, ix)[0]
        sh.add(rng.standard_normal((10, D)).astype(np.float32), base + 10 ** 5 + np.arange(10))
        log["grown"], log["grown_rank"] = _need(world, r, sh, ix)
        # after shard_load: train_rows_set = the live rows
        sh.save(os.path.join(tmp, "set"))
        lx = b200vs.Index(IVF_FLAT, L2, D, nlist=nlist)
        lsh = _connect(world, lx, r)
        lsh.load(os.path.join(tmp, "set"))
        log["loaded"] = _need(world, r, lsh, lx)[0]
        lsh.add(rng.standard_normal((grow + 5, D)).astype(np.float32), base + 2 * 10 ** 5 + np.arange(grow + 5))
        log["loaded_grown"] = _need(world, r, lsh, lx)[0]
        # after shard_broadcast_state: train_rows_set = the live rows then (0)
        bx = b200vs.Index(IVF_FLAT, L2, D, nlist=nlist)
        bsh = _connect(world, bx, r)
        if r == 0:
            bx.set_trained_state(ix.get_trained_state())
        bsh.broadcast_state(0)
        log["broadcast"] = _need(world, r, bsh, bx)[0]
        bsh.add(rng.standard_normal((grow, D)).astype(np.float32), base + np.arange(grow))
        log["broadcast_grown"] = _need(world, r, bsh, bx)[0]
        # HNSW: tombstones crossing half of the nodes, summed over the set
        hx = b200vs.Index(HNSW, L2, D, hnsw_m=8, hnsw_efc=32, max_elements=1000)
        hsh = _connect(world, hx, r)
        hid = np.arange(90, dtype=np.int64)
        hsh.add(rng.standard_normal((90, D)).astype(np.float32)[r::W], hid[r::W])
        hsh.delete(hid[:45])
        log["hnsw_half"] = _need(world, r, hsh, hx)[0]
        hsh.delete(hid[45:46])
        log["hnsw_over"] = _need(world, r, hsh, hx)[0]
        # IVF_PQ: sum(live) / 2 >= train_rows_set
        px = b200vs.Index(IVF_PQ, L2, 16, nlist=nlist, pq_m=4, pq_nbits=4)
        psh = _connect(world, px, r)
        log["pq_untrained"] = _need(world, r, psh, px)[0]
        t_rows = 4096 if r == 0 else 64
        psh.train(rng.standard_normal((t_rows, 16)).astype(np.float32))
        T = 4096 + 64 * (W - 1)
        mine = (2 * T - 2) // W + (1 if r < (2 * T - 2) % W else 0)
        psh.add(rng.standard_normal((mine, 16)).astype(np.float32), base + np.arange(mine))
        log["pq_short"] = _need(world, r, psh, px)[0]
        if r == 0:
            psh.add(rng.standard_normal((2, 16)).astype(np.float32), base + 10 ** 5 + np.arange(2))
        else:
            psh.add(np.zeros((0, 16), np.float32), np.zeros(0, np.int64))
        log["pq_enough"] = _need(world, r, psh, px)[0]
        # FLAT, BINARY_FLAT: never
        for t, dim, rows in ((FLAT, D, rng.standard_normal((50, D)).astype(np.float32)),
                             (BINARY_FLAT, BDIM, rng.integers(0, 256, (50, BDIM // 8), dtype=np.uint8))):
            fx = b200vs.Index(t, L2 if t == FLAT else HAMMING, dim)
            fsh = _connect(world, fx, r)
            fsh.add(rows[r::W], np.arange(50)[r::W])
            fsh.delete(np.arange(40))
            log[f"flat{t}"] = _need(world, r, fsh, fx)[0]
            fsh.close()
        for s in (sh, lsh, bsh, hsh, psh):
            s.close()
        return log

    try:
        outs = _ranks(W, rank)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    want = dict(untrained=False, short=False, grown=True, loaded=False, loaded_grown=True, broadcast=False, broadcast_grown=True,
                hnsw_half=False, hnsw_over=True, pq_untrained=False, pq_short=False, pq_enough=True)
    want.update({f"flat{FLAT}": False, f"flat{BINARY_FLAT}": False})
    for r, o in enumerate(outs):
        for key, v in want.items():
            assert o[key] == v, f"rank {r}: {key} answered {o[key]}, want {v}"
        if W > 1:
            assert not o["grown_rank"], f"rank {r}: the rank index alone asks for a rebuild (the case needs it not to)"


# ---------------------------------------------------------------------------------------------
# 5. refusals: met on one rank, returned by every rank, both sets unchanged and usable
# ---------------------------------------------------------------------------------------------
def case_refusals(W):
    rng = np.random.default_rng(50 + W)
    nlist = 2 * W
    n = 600 * W
    x = rng.standard_normal((n, D)).astype(np.float32)
    ids = np.arange(n, dtype=np.int64)
    parts = _split(W, n)
    bad = min(1, W - 1)  # the rank that meets the refusal
    # few live rows: no rank but the last gets enough training rows
    few = [int(i) for i in np.arange(10 ** 6, 10 ** 6 + 2000) if row_owner([i], W)[0] == 0][:3] if W > 1 else []
    xq = rng.standard_normal((4, D)).astype(np.float32)

    def rank(r, world):
        res = {}
        src_ix = b200vs.Index(IVF_FLAT, L2, D, nlist=nlist)
        src = _connect(world, src_ix, r)
        src.train(x[parts[r]][:200])
        src.add(x[parts[r]], ids[parts[r]])
        snap = [(_export(src_ix, nlist), src_ix.get_trained_state())]
        next_id = [10 ** 8 + 1000 * r]

        def src_after(key):
            """src unchanged by the refusal, then a collective write and a search on it"""
            exp, st = snap[0]
            res[key + "_src_same"] = (np.array_equal(src_ix.get_trained_state(), st) and
                                      all(np.array_equal(a, b) for a, b in zip(_export(src_ix, nlist), exp)))
            src.add(x[:1] + 1, np.array([next_id[0]], np.int64))
            next_id[0] += 1
            res[key + "_src_search"] = src.search(xq, 5, nprobe=nlist)
            snap[0] = (_export(src_ix, nlist), src_ix.get_trained_state())

        def train_add_search(sh, k):
            """a collective write (train + add) and a search on a consistent dst"""
            sh.train(x[parts[r]][:200])
            sh.add(x[parts[r]][:50], 3 * 10 ** 8 + ids[parts[r]][:50])
            return sh.search(xq, k, nprobe=nlist)

        def attempt(key, dst_ix, prepare=None, use=None, dst_rank=None):
            """rebuild into a dst that meets one refusal; use(dst) is the write and search that dst must still serve
            (dsts whose creation parameters differ between ranks are no set to search: they get a delete and the rule)"""
            if dst_rank is None:
                dst = _connect(world, dst_ix, r)
            else:
                idb = world.gather(r, b200vs.Shard.unique_id() if r == 0 else None)[0]
                dst = b200vs.Shard(dst_ix, dst_rank, world.W, idb)
            if prepare:
                prepare(dst_ix)
            st0 = dst_ix.get_trained_state().copy(), dst_ix.get_count()
            res[key] = _status(lambda: dst.rebuild_from(src))
            res[key + "_dst_same"] = np.array_equal(dst_ix.get_trained_state(), st0[0]) and dst_ix.get_count() == st0[1]
            if use is None:
                res[key + "_use"] = _status(lambda: (dst.delete(np.array([12345], np.int64)), dst.need_rebuild()))
            else:
                res[key + "_use"] = _status(lambda: res.__setitem__(key + "_dst_search", use(dst)))
            dst.close()
            src_after(key)

        def add_search(sh):
            sh.add(x[parts[r]][:50], 6 * 10 ** 8 + ids[parts[r]][:50])
            return sh.search(xq, 5, nprobe=nlist)

        # a trained dst on one rank (at world 1 that is a trained set, which takes an add and a search)
        attempt("trained", b200vs.Index(IVF_FLAT, L2, D, nlist=nlist),
                (lambda ix: ix.set_trained_state(src_ix.get_trained_state())) if r == bad else None,
                use=add_search if W == 1 else None)
        # differing creation parameters on one rank
        attempt("params", b200vs.Index(IVF_FLAT, L2, D, nlist=2 * nlist if r == bad else nlist))
        attempt("metric", b200vs.Index(IVF_FLAT, IP if r == bad else L2, D, nlist=nlist))
        # a different rank: dst's ranks are src's shifted by one (a communicator's world is the same on every rank)
        if W > 1:
            attempt("rank", b200vs.Index(IVF_FLAT, L2, D, nlist=nlist), use=lambda sh: train_add_search(sh, 5), dst_rank=(r + 1) % W)
        # the same shard as dst and src, on every rank
        res["same"] = _status(lambda: src.rebuild_from(src))
        src_after("same")
        # a Flat set and an IVF-PQ set
        fsrc = _connect(world, b200vs.Index(FLAT, L2, D), r)
        fsrc.add(x[parts[r]], ids[parts[r]])
        fdst = _connect(world, b200vs.Index(FLAT, L2, D), r)
        res["flat"] = _status(lambda: fdst.rebuild_from(fsrc))
        fdst.add(x[parts[r]][:20], 4 * 10 ** 8 + ids[parts[r]][:20])
        res["flat_use"] = _status(lambda: res.__setitem__("flat_dst_search", fdst.search(xq, 5)))
        fdst.close()
        fsrc.close()
        psrc = _connect(world, b200vs.Index(IVF_PQ, L2, 16, nlist=nlist, pq_m=4, pq_nbits=4), r)
        pdst = _connect(world, b200vs.Index(IVF_PQ, L2, 16, nlist=nlist, pq_m=4, pq_nbits=4), r)
        res["pq"] = _status(lambda: pdst.rebuild_from(psrc))
        pdst.close()
        psrc.close()
        # HNSW: a non-empty dst, and a dst whose max_elements is below the rank's live rows, on one rank
        hkw = dict(hnsw_m=8, hnsw_efc=32)
        hsrc_ix = b200vs.Index(HNSW, L2, D, max_elements=10 * n, **hkw)
        hsrc = _connect(world, hsrc_ix, r)
        hsrc.add(x[:300][r::W], ids[:300][r::W])
        hblob = hsrc_ix.get_trained_state().copy()
        for key, me, fill in (("hnsw_full", 10 * n, True), ("hnsw_small", 1, False)):
            dix = b200vs.Index(HNSW, L2, D, max_elements=me if r == bad else 10 * n, **hkw)
            dsh = _connect(world, dix, r)
            if fill and r == bad:
                dix.add(x[:1], np.array([10 ** 7], np.int64))
            cnt = dix.get_count()
            res[key] = _status(lambda: dsh.rebuild_from(hsrc))
            res[key + "_dst_same"] = dix.get_count() == cnt
            # a write every rank's dst accepts (max_elements 1 on one rank: a delete), then a search
            write = ((lambda: dsh.add(x[300:330][r::W], 5 * 10 ** 8 + ids[300:330][r::W])) if fill
                     else (lambda: dsh.delete(np.array([12345], np.int64))))
            res[key + "_use"] = _status(lambda: (write(), res.__setitem__(key + "_dst_search", dsh.search(xq, 5, efsearch=32))))
            dsh.close()
        res["hnsw_src_same"] = np.array_equal(hsrc_ix.get_trained_state(), hblob)
        hsrc.close()
        # too few training rows for a rank
        if W > 1:
            tsrc_ix = b200vs.Index(IVF_FLAT, L2, D, nlist=nlist)
            tsrc_ix.set_trained_state(src_ix.get_trained_state())
            tsrc = _connect(world, tsrc_ix, r)
            mine = few[r::W]
            tsrc.add(rng.standard_normal((len(mine), D)).astype(np.float32), np.array(mine, np.int64))
            tdst_ix = b200vs.Index(IVF_FLAT, L2, D, nlist=nlist)
            tdst = _connect(world, tdst_ix, r)
            res["few"] = _status(lambda: tdst.rebuild_from(tsrc))
            res["few_dst_same"] = not tdst_ix.is_trained() and tdst_ix.get_count() == 0
            res["few_use"] = _status(lambda: res.__setitem__("few_dst_search", train_add_search(tdst, 5)))
            tdst.close()
            tsrc.close()
        src.close()
        return res

    outs = _ranks(W, rank)
    want = dict(trained=EILLEGAL_PARAMETERS, params=EILLEGAL_PARAMETERS, metric=EILLEGAL_PARAMETERS, same=EILLEGAL_PARAMETERS,
                flat=EVECTOR_NOT_SUPPORT, pq=EVECTOR_NOT_SUPPORT, hnsw_full=EILLEGAL_PARAMETERS, hnsw_small=EILLEGAL_PARAMETERS)
    if W > 1:
        want["few"] = EILLEGAL_PARAMETERS
        want["rank"] = EILLEGAL_PARAMETERS
    for r, o in enumerate(outs):
        for key, v in want.items():
            assert o[key] == v, f"rank {r}: {key} returned {o[key]}, want {v}"
            if key + "_dst_same" in o:
                assert o[key + "_dst_same"], f"rank {r}: {key} changed dst"
            if key + "_use" in o:
                assert o[key + "_use"] == b200vs.OK, f"rank {r}: dst unusable after {key}: status {o[key + '_use']}"
            if key + "_dst_search" in o:
                _eq(o[key + "_dst_search"], outs[0][key + "_dst_search"], f"rank {r}: dst search after {key}")
            if key + "_src_same" in o:
                assert o[key + "_src_same"], f"rank {r}: {key} changed src"
                s = o[key + "_src_search"]
                assert (s[1][:, 0] >= 0).all(), f"rank {r}: src search after {key}"
                _eq(s, outs[0][key + "_src_search"], f"rank {r}: src search after {key}")
        assert o["hnsw_src_same"], f"rank {r}: a refusal changed the HNSW src"


# ---------------------------------------------------------------------------------------------
# 6. concurrency: src's reads go on during the rebuild; src's writes wait for it
# ---------------------------------------------------------------------------------------------
def case_concurrency(W):
    from shard_loopback import World
    rng = np.random.default_rng(90 + W)
    nlist = 4 * W
    n = 150000 * W
    x = rng.standard_normal((n, D)).astype(np.float32)
    ids = np.arange(n, dtype=np.int64)
    parts = _split(W, n)
    xq = rng.standard_normal((16, D)).astype(np.float32)
    new_ids = np.array([5 * 10 ** 8, 5 * 10 ** 8 + 1], np.int64)

    def rank(r, world):
        src_ix = b200vs.Index(IVF_FLAT, L2, D, nlist=nlist)
        src = _connect(world, src_ix, r, lanes=2)
        src.train(x[parts[r]][:2000])
        src.add(x[parts[r]], ids[parts[r]])
        seq = 0
        want = src.search(xq, 10, seq=seq, nprobe=4)
        seq += 1
        # reads on src with consecutive seqs while the rebuild runs
        dst_ix = b200vs.Index(IVF_FLAT, L2, D, nlist=nlist)
        dst = _connect(world, dst_ix, r)
        got, spans, errs = [], [], []
        done = [False]

        def reader(s0):
            # reads go on until every rank's rebuild has returned; the reader threads agree on that after each read (their
            # own World), so every rank issues the same sequence numbers
            try:
                s = s0
                while True:
                    t0 = time.monotonic()
                    got.append(src.search(xq, 10, seq=s, nprobe=4))
                    spans.append((t0, time.monotonic()))
                    s += 1
                    if all(readers.gather(r, done[0])) or s >= s0 + 100000:
                        break
            except Exception as e:  # noqa: BLE001 - reported below
                errs.append(e)

        th = threading.Thread(target=reader, args=(seq,))
        th.start()
        t_rb0 = time.monotonic()
        n_rows = dst.rebuild_from(src)
        t_rb1 = time.monotonic()
        done[0] = True
        th.join()
        during = sum(1 for a, b in spans if a < t_rb1 and b > t_rb0)  # reads that ran while the rebuild did
        # a src write issued during a second rebuild returns after it, and its rows are not in that dst
        dst2_ix = b200vs.Index(IVF_FLAT, L2, D, nlist=nlist)
        dst2 = _connect(world, dst2_ix, r)
        t = {}

        def writer():
            time.sleep(0.02)  # the rebuild, entered first on this thread's rank, holds src's add_mu by then
            t["issued"] = time.monotonic()
            src.add(x[:2] + 1, new_ids if r == 0 else new_ids[:0])
            t["add"] = time.monotonic()

        wt = threading.Thread(target=writer)
        wt.start()
        dst2.rebuild_from(src)
        t["rebuild"] = time.monotonic()
        wt.join()
        in_dst2 = np.isin(new_ids, _export(dst2_ix, nlist)[2]).any()
        out = dict(want=want, got=got, during=during, rebuild_s=t_rb1 - t_rb0, errs=[str(e) for e in errs], n_rows=n_rows,
                   issued_during=t["issued"] < t["rebuild"], add_after=t["add"] >= t["rebuild"], in_dst2=in_dst2)
        for s in (dst, dst2, src):
            s.close()
        return out

    readers = World(W)
    outs = _ranks(W, rank)
    for r, o in enumerate(outs):
        print(f"rank {r}: {len(o['got'])} reads, {o['during']} of them during the {o['rebuild_s'] * 1e3:.1f} ms rebuild", flush=True)
        assert not o["errs"], f"rank {r}: {o['errs']}"
        assert o["during"] >= 1, f"rank {r}: no read ran during the rebuild"
        for i, g in enumerate(o["got"]):
            _eq(g, o["want"], f"rank {r}: read {i} during the rebuild")
        assert o["issued_during"], f"rank {r}: the src add was issued after the rebuild had returned"
        assert o["add_after"], f"rank {r}: a src add returned before the rebuild"
        assert not o["in_dst2"], f"rank {r}: rows added during the rebuild reached dst"
    assert sum(o["n_rows"] for o in outs) == n


# ---------------------------------------------------------------------------------------------
# tests: world 1 in this process, worlds 2, 3, 5 in a loopback subprocess
# ---------------------------------------------------------------------------------------------
def each_world(case, worlds, *args):
    for W in worlds:
        try:
            globals()[case](W, *args)
        except AssertionError as e:
            raise AssertionError(f"world {W}: {e}") from e


def _run(case, *args, worlds=(2, 3, 5)):
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


@pytest.mark.parametrize("name", sorted(LIST_KINDS))
def test_world1_lists(name):
    case_lists(1, name)


@pytest.mark.parametrize("name", sorted(LIST_KINDS))
def test_lists(name):
    _run("case_lists", name)


@pytest.mark.parametrize("metric", (L2, COSINE))
def test_hnsw(metric):
    _run("case_hnsw", metric, worlds=(2, 3))


def test_need_rebuild_world1():
    case_need(1)


def test_need_rebuild_world3():
    _run("case_need", worlds=(3,))


def test_refusals_world1():
    case_refusals(1)


def test_refusals():
    _run("case_refusals", worlds=(2, 3))


def test_concurrency():
    _run("case_concurrency", worlds=(2,))


def _main():
    """The subprocess of one loopback case: mirrors shard_loopback._main, with this module's cases."""
    case, args, dump_after = sys.argv[1], json.loads(sys.argv[2]), int(sys.argv[3])
    faulthandler.enable(all_threads=True)  # a fatal signal prints every rank thread's stack
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
