"""Sharded split and merge rebuilds: b200vs_shard_rebuild_from_range fills a fresh set from an id range of one or more old
sets' device rows.

World 1 runs in this process (no NCCL).  Worlds 2, 3 and 5 run as threads of one process on one GPU over the loopback NCCL
(tests/shard_loopback.py's World and run_world), each case in a subprocess of its own started through this file's __main__,
with a timeout.  References: list-sharded sets, a fresh set fed from the host with shard_train + shard_add of each rank's
rows_r (the rows of R that row_owner gives the rank, in ascending id order) and, at world 1, b200vs_rebuild_from_range of the
rank-0 indexes; row-sharded sets, b200vs_rebuild_from_range of each rank's own source indexes."""
import faulthandler
import json
import os
import subprocess
import sys
import threading
import time

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, os.path.join(ROOT, "dingo-store_b200", "python"))
sys.path.insert(0, HERE)

import b200vs  # noqa: E402
from b200vs import (BINARY_FLAT, BINARY_IVF_FLAT, COSINE, EILLEGAL_PARAMETERS, EVECTOR_ID_DUPLICATED, EVECTOR_NOT_SUPPORT,  # noqa: E402
                    FLAT, HAMMING, HNSW, IP, IVF_FLAT, IVF_PQ, L2)
from b200vs.shard import row_owner  # noqa: E402
from gpu_util import require_gpu  # noqa: E402
from shard_loopback import LIB, World, run_world  # noqa: E402
from test_gpu_shard_rebuild import _connect, _eq, _export, _index, _rows, _split, _status  # noqa: E402

pytestmark = pytest.mark.gpu
CASE_TIMEOUT = 900  # seconds of one subprocess; every rendezvous of the loopback library times out after 60 s
D, BDIM = 32, 48
ALL = 2 ** 63 - 1  # id_max of "every id"
HNSW_KW = dict(hnsw_m=16, hnsw_efc=64)


@pytest.fixture(autouse=True)
def _gpu():
    require_gpu()


def _ranks(W, fn):
    return [fn(0, None)] if W == 1 else run_world(W, fn)


def _gather(world, rank, v):
    return [v] if world is None else world.gather(rank, v)


def _lists(t):
    return t in (IVF_FLAT, BINARY_IVF_FLAT)


def _snap(ix, t, nlist):
    """Everything a rebuild decides about one rank index: its trained state (HNSW: the graph) and, for the row-store types,
    every list's ids and rows."""
    st = ix.get_trained_state().copy()
    if t == HNSW or not ix.is_trained():
        return st, ix.get_count()
    return st, _export(ix, nlist if _lists(t) else 1)


def _snap_eq(a, b, what):
    assert np.array_equal(a[0], b[0]), f"{what}: trained state / graph differs"
    if isinstance(a[1], tuple):
        _eq(a[1], b[1], what + ": lists")
    else:
        assert a[1] == b[1], f"{what}: count {a[1]} != {b[1]}"


def _search(sh, t, xq, nlist):
    if t == HNSW:
        return sh.search(xq, 10, efsearch=64)
    if _lists(t):
        return sh.search(xq, 10, nprobe=min(3, nlist))
    return sh.search(xq, 10)


def _host_rows(all_exps, lo, hi, W, r):
    """rows_r of R: every source set's exported rows (source order, then rank order, then list-major order), filtered to
    lo <= id < hi, stable by id, owner r."""
    ids = np.concatenate([e[2] for exps in all_exps for e in exps])
    x = np.concatenate([e[1] for exps in all_exps for e in exps])
    keep = (ids >= lo) & (ids < hi)
    ids, x = ids[keep], x[keep]
    order = np.argsort(ids, kind="stable")
    mine = order[row_owner(ids[order], W) == r] if ids.size else order
    return x[mine], ids[mine]


# ---------------------------------------------------------------------------------------------
# 1-4, 7. splits, merges and range edges of every type: list-sharded sets against the host-fed reference, row-sharded sets
# against each rank's single-index rebuild_from_range, one source over every id against shard_rebuild_from
# ---------------------------------------------------------------------------------------------
# name -> (type, metric, skewed: every live row of the first set sits in rank 0's lists)
KINDS = {"ivf_l2": (IVF_FLAT, L2, False), "ivf_ip": (IVF_FLAT, IP, False), "ivf_cosine": (IVF_FLAT, COSINE, False),
         "ivf_l2_skewed": (IVF_FLAT, L2, True), "binary_ivf": (BINARY_IVF_FLAT, HAMMING, False),
         "binary_ivf_skewed": (BINARY_IVF_FLAT, HAMMING, True), "flat_l2": (FLAT, L2, False), "flat_ip": (FLAT, IP, False),
         "binary_flat": (BINARY_FLAT, HAMMING, False), "hnsw_l2": (HNSW, L2, False), "hnsw_cosine": (HNSW, COSINE, False)}
LIST_NAMES = sorted(k for k, v in KINDS.items() if _lists(v[0]))
ROW_NAMES = sorted(k for k, v in KINDS.items() if not _lists(v[0]))


def case_ranges(W, name):
    t, metric, skewed = KINDS[name]
    binary, lists = t in (BINARY_IVF_FLAT, BINARY_FLAT), _lists(t)
    rng = np.random.default_rng(sorted(KINDS).index(name) * 10 + W)
    nlist = 4 * W if lists else 0
    dim = BDIM if binary else D
    n = 1200 * W
    kw = dict(HNSW_KW, max_elements=8 * n) if t == HNSW else {}
    # set A holds ids in [0, 4n), set B (the merge sibling) ids in [4n, 8n)
    ids_a = rng.permutation(4 * n)[:n].astype(np.int64)
    ids_b = 4 * n + rng.permutation(4 * n)[: n // 2].astype(np.int64)
    cent = _rows(rng, binary, max(nlist, 1))
    if skewed:  # rows near centroid 0: rank 0's list 0 takes all of A, every other rank of A stays empty
        if binary:
            x_a = np.repeat(cent[:1], n, axis=0)
            x_a[np.arange(n), rng.integers(0, BDIM // 8, n)] ^= 1
        else:
            x_a = (cent[:1] + 0.01 * rng.standard_normal((n, dim))).astype(np.float32)
    else:
        x_a = _rows(rng, binary, n)
    x_b = _rows(rng, binary, ids_b.size)
    blob = (b200vs.binary_ivf_state_blob(cent) if binary else b200vs.ivf_state_blob(cent, metric)) if lists else None
    parts_a, parts_b = _split(W, n), _split(W, ids_b.size)
    up = ids_a[[i for i in range(2, n, 11) if i % 4]]  # upserts, none of them among the ids_a[::4] tombstoned after them
    up_x = _rows(rng, binary, up.size)
    ties = lists and not skewed and metric in (L2, HAMMING)
    tie_ids = 3 * n + 7 + np.arange(8, dtype=np.int64) * 13  # inside A's id range, every copy in a different rank's lists
    mid = int(np.median(ids_a))
    xq = _rows(rng, binary, 9)
    one_id = int(ids_a[5])  # live in A: not deleted below (ids_a[::4] and up are)
    # (key, sources, id_min, id_max): a split child and parent of A, a merge of A and B, and the edges
    jobs = [("child", "a", mid, 4 * n), ("parent", "a", 0, mid), ("merge", "ab", 0, 8 * n), ("empty", "a", mid, mid),
            ("past", "ab", 8 * n, ALL), ("one", "ab", one_id, one_id + 1), ("all", "a", 0, ALL)]
    grow_n = (2 * (n + ids_b.size) + 256 * max(nlist, 1)) // W + 1

    def rank(r, world):
        def make_set(xs, ids, parts, trained_blob):
            ix = _index(t, metric, dim, nlist, **kw)
            if trained_blob is not None:
                ix.set_trained_state(trained_blob)
            sh = _connect(world, ix, r)
            if lists and trained_blob is None:
                sh.train(xs[parts[r]][: max(nlist, len(xs[parts[r]]) // 2)])
            sh.add(xs[parts[r]], ids[parts[r]])  # each row travels to its list's owner, or to row_owner(id)
            return ix, sh

        a_ix, a = make_set(x_a, ids_a, parts_a, blob if skewed else None)
        a.delete(up)  # upserts: a delete, then an add of new rows under the same ids; then a quarter tombstoned
        a.add(up_x[r::W], up[r::W])
        a.delete(ids_a[::4])
        if lists and not skewed:
            a.add(x_a[parts_a[r]][:3], ids_a[parts_a[r]][:3])  # repeated ids inside one set: legal
        if ties:  # ids whose copies hold different rows in different ranks' lists of A
            st = a_ix.get_trained_state()[32:]
            c = st.reshape(nlist, dim // 8) if binary else st.view(np.float32).reshape(nlist, dim)
            copies = np.repeat(c[r * (nlist // W)][None], tie_ids.size, axis=0)
            if not binary:
                copies = (copies + 1e-4 * rng.standard_normal(copies.shape)).astype(np.float32)
            a.add(copies, tie_ids)
        b_ix, b = make_set(x_b, ids_b, parts_b, None)
        b.delete(ids_b[1::5])
        srcs = {"a": [(a_ix, a)], "ab": [(a_ix, a), (b_ix, b)]}
        exps = ({"a": _export(a_ix, nlist), "b": _export(b_ix, nlist)} if lists else None)
        all_exps = {k: _gather(world, r, v) for k, v in exps.items()} if lists else None
        if ties:
            assert all(np.isin(tie_ids, e[2]).all() for e in all_exps["a"]), "a tied id is missing from some rank's lists"
        snaps = [_snap(s_ix, t, nlist) for s_ix, _ in srcs["ab"]]
        want_src = [_search(s, t, xq, nlist) for _, s in srcs["ab"]]
        out = {}
        for key, sk, lo, hi in jobs:
            dst_ix = _index(t, metric, dim, nlist, **kw)
            dst = _connect(world, dst_ix, r)
            st = _status(lambda: out.__setitem__(key + "_n", dst.rebuild_from_range([s for _, s in srcs[sk]], lo, hi)))
            o = dict(status=st, count=dst_ix.get_count(), trained=dst_ix.is_trained(), snap=_snap(dst_ix, t, nlist))
            if lists:  # the host-fed reference
                rows_r, ids_r = _host_rows([all_exps[c] for c in sk], lo, hi, W, r)
                total = sum(_gather(world, r, ids_r.size))
                ref_ix = _index(t, metric, dim, nlist)
                ref = _connect(world, ref_ix, r)
                ref_st = b200vs.OK
                if total:
                    ref_st = _status(lambda: ref.train(rows_r))
                    if ref_st == b200vs.OK:
                        ref.add(rows_r, ids_r)
                o.update(ref_status=ref_st, ref_snap=_snap(ref_ix, t, nlist), want_n=ref_ix.get_count())
                if st == b200vs.OK and total:
                    o.update(search=_search(dst, t, xq, nlist), ref_search=_search(ref, t, xq, nlist),
                             deep=dst.search_deep(xq, 200), ref_deep=ref.search_deep(xq, 200))
                if key == "merge":  # 7. the set's rule on the rebuilt set, as on the host-fed reference, as the sets grow
                    g = _rows(rng, binary, grow_n)
                    g_ids = 10 ** 9 + r * grow_n + np.arange(grow_n, dtype=np.int64)
                    need = [(dst.need_rebuild(), ref.need_rebuild())]
                    dst.add(g, g_ids)
                    ref.add(g, g_ids)
                    need.append((dst.need_rebuild(), ref.need_rebuild()))
                    o["need"] = need
                ref.close()
            else:  # each rank's single-index rebuild_from_range of its own source indexes
                one = _index(t, metric, dim, nlist, **kw)
                one_st = _status(lambda: out.__setitem__(key + "_one_n", one.rebuild_from_range([s_ix for s_ix, _ in srcs[sk]], lo, hi)))
                o.update(ref_status=one_st, ref_snap=_snap(one, t, nlist), want_n=out.get(key + "_one_n", 0))
                if st == b200vs.OK and one.get_count():
                    o.update(search=dst_ix.search(xq, 10, **({"efsearch": 64} if t == HNSW else {})),
                             ref_search=one.search(xq, 10, **({"efsearch": 64} if t == HNSW else {})))
                if t == HNSW and key == "merge":
                    o["need"] = [(dst.need_rebuild(), False)]
            if key == "all" and t != FLAT and t != BINARY_FLAT:  # 4. one source, every id: shard_rebuild_from
                fx = _index(t, metric, dim, nlist, **kw)
                fsh = _connect(world, fx, r)
                o["from_n"] = fsh.rebuild_from(a)
                o["from_snap"] = _snap(fx, t, nlist)
                fsh.close()
            if W == 1 and lists:  # world 1: b200vs_rebuild_from_range of the rank-0 indexes
                one = _index(t, metric, dim, nlist)
                o["one_status"] = _status(lambda: one.rebuild_from_range([s_ix for s_ix, _ in srcs[sk]], lo, hi))
                o["one_snap"] = _snap(one, t, nlist)
                if o["one_status"] == b200vs.OK and st == b200vs.OK and one.get_count():
                    o["one_search"] = (one.search(xq, 10, nprobe=min(3, nlist)), one.search_deep(xq, 200))
            o["n"] = out.get(key + "_n", 0)
            out[key] = o
            dst.close()
        for i, (s_ix, s) in enumerate(srcs["ab"]):
            _snap_eq(_snap(s_ix, t, nlist), snaps[i], f"rank {r}: source {i} after the rebuilds")
            _eq(_search(s, t, xq, nlist), want_src[i], f"rank {r}: source {i} search after the rebuilds")
        a.close()
        b.close()
        return out

    outs = _ranks(W, rank)
    for key, sk, lo, hi in jobs:
        for r, o in enumerate(outs):
            what = f"{name} W={W} rank {r} {key}"
            o = o[key]
            if key in ("empty", "past"):
                assert o["status"] == b200vs.OK and o["n"] == 0 and o["count"] == 0, what
                if lists:
                    assert not o["trained"], f"{what}: an empty R trained dst"
            assert o["status"] == o["ref_status"], f"{what}: status {o['status']}, reference {o['ref_status']}"
            if o["status"] != b200vs.OK:  # the single id at world > 1 on list types: shard_train's refusal
                assert key == "one" and lists and o["count"] == 0 and not o["trained"], what
                continue
            assert o["n"] == o["count"] == o["want_n"], f"{what}: n_rows {o['n']}, count {o['count']}, want {o['want_n']}"
            _snap_eq(o["snap"], o["ref_snap"], what)
            for k in ("search", "deep"):
                if k in o:
                    _eq(o[k], o["ref_" + k], f"{what}: {k}")
            if "need" in o:
                for got, want in o["need"]:
                    assert got == want, f"{what}: need_rebuild {got}, reference {want}"
                if lists:
                    assert o["need"][-1][0], f"{what}: the grown set does not ask for a rebuild"
            if "from_snap" in o:
                assert o["from_n"] == o["n"], what
                _snap_eq(o["snap"], o["from_snap"], f"{what} vs shard_rebuild_from")
            if "one_snap" in o:
                assert o["one_status"] == o["status"], what
                _snap_eq(o["snap"], o["one_snap"], f"{what} vs b200vs_rebuild_from_range")
                if "one_search" in o:
                    _eq(o["search"], o["one_search"][0], f"{what}: search vs the single index")
                    _eq(o["deep"], o["one_search"][1], f"{what}: deep vs the single index")
    for key in ("child", "parent", "merge"):
        assert sum(o[key]["n"] for o in outs) > 0, f"{name} W={W}: {key} rebuilt no rows"


# ---------------------------------------------------------------------------------------------
# 5. refusals: met on one rank, returned by every rank, dst fresh, dst and sources still serve
# ---------------------------------------------------------------------------------------------
def case_refusals(W):
    rng = np.random.default_rng(70 + W)
    nlist = 2 * W
    n = 600 * W
    x = rng.standard_normal((n, D)).astype(np.float32)
    ids = np.arange(n, dtype=np.int64)
    parts = _split(W, n)
    bad = min(1, W - 1)  # the rank that meets the refusal
    xq = rng.standard_normal((4, D)).astype(np.float32)
    few = [int(i) for i in np.arange(10 ** 6, 10 ** 6 + 2000) if row_owner([i], W)[0] == 0][:3] if W > 1 else []
    dup_id = 10 ** 7

    def rank(r, world):
        res = {}
        src_ix = b200vs.Index(IVF_FLAT, L2, D, nlist=nlist)
        src = _connect(world, src_ix, r)
        src.train(x[parts[r]][:200])
        src.add(x[parts[r]], ids[parts[r]])
        # a second set that holds dup_id too: src's copy sits on a centroid of rank bad's lists, sib's on one of rank
        # (bad + 1) % W's, so the two copies meet only after the routing
        sib_ix = b200vs.Index(IVF_FLAT, L2, D, nlist=nlist)
        sib = _connect(world, sib_ix, r)
        sib.train(x[parts[r]][:200])
        sib.add(x[parts[r]][:100] + 5, 2 * 10 ** 6 + ids[parts[r]][:100])
        per = nlist // W
        for sh, ix, owner in ((src, src_ix, bad), (sib, sib_ix, (bad + 1) % W)):
            row = ix.get_trained_state()[32:].view(np.float32).reshape(nlist, D)[owner * per][None]
            sh.add(row if r == 0 else row[:0], np.array([dup_id] if r == 0 else [], np.int64))
        res["dup_holders"] = (dup_id in _export(src_ix, nlist)[2], dup_id in _export(sib_ix, nlist)[2])
        state = {k: (_export(v, nlist), v.get_trained_state().copy()) for k, v in (("src", src_ix), ("sib", sib_ix))}
        want = {k: s.search(xq, 5, nprobe=nlist) for k, s in (("src", src), ("sib", sib))}

        def sources_after(key):
            """the sources unchanged by the refusal and still serving searches"""
            res[key + "_src_same"] = all(
                np.array_equal(v.get_trained_state(), state[k][1]) and all(np.array_equal(p, q) for p, q in zip(_export(v, nlist), state[k][0]))
                for k, v in (("src", src_ix), ("sib", sib_ix)))
            res[key + "_src_search"] = all(np.array_equal(s.search(xq, 5, nprobe=nlist)[1], want[k][1]) for k, s in (("src", src), ("sib", sib)))

        def attempt(key, dst_ix, srcs, lo=0, hi=ALL, prepare=None, dst_rank=None, consistent=True):
            if dst_rank is None:
                dst = _connect(world, dst_ix, r)
            else:
                idb = world.gather(r, b200vs.Shard.unique_id() if r == 0 else None)[0]
                dst = b200vs.Shard(dst_ix, dst_rank, world.W, idb)
            if prepare:
                prepare(dst_ix)
            st0 = dst_ix.get_trained_state().copy(), dst_ix.get_count()
            res[key] = _status(lambda: dst.rebuild_from_range(srcs, lo, hi(r) if callable(hi) else hi))
            res[key + "_dst_same"] = np.array_equal(dst_ix.get_trained_state(), st0[0]) and dst_ix.get_count() == st0[1]
            if consistent:  # a collective write and a search on dst
                def use():
                    if not dst_ix.is_trained():
                        dst.train(x[parts[r]][:200])
                    dst.add(x[parts[r]][:50], 3 * 10 ** 8 + ids[parts[r]][:50])
                    res[key + "_dst_search"] = dst.search(xq, 5, nprobe=nlist)
                res[key + "_use"] = _status(use)
            else:
                res[key + "_use"] = _status(lambda: (dst.delete(np.array([12345], np.int64)), dst.need_rebuild()))
            dst.close()
            sources_after(key)

        ivf = lambda **kw: b200vs.Index(IVF_FLAT, kw.get("metric", L2), D, nlist=kw.get("nlist", nlist))  # noqa: E731
        attempt("range", ivf(), [src], 10, lambda rr: 5 if rr == bad else 100)  # id_min > id_max on one rank
        attempt("trained", ivf(), [src], prepare=(lambda ix: ix.set_trained_state(src_ix.get_trained_state())) if r == bad else None,
                consistent=W == 1)
        attempt("params", ivf(nlist=2 * nlist if r == bad else nlist), [src], consistent=False)
        attempt("metric", ivf(metric=IP if r == bad else L2), [src, sib], consistent=False)
        attempt("dup", ivf(), [src, sib])  # an id live in two sets, its copies on two ranks
        if W > 1:
            attempt("rank", ivf(), [src], dst_rank=(r + 1) % W)
            tsrc_ix = ivf()
            tsrc_ix.set_trained_state(src_ix.get_trained_state())
            tsrc = _connect(world, tsrc_ix, r)
            mine = few[r::W]
            tsrc.add(rng.standard_normal((len(mine), D)).astype(np.float32), np.array(mine, np.int64))
            attempt("few", ivf(), [tsrc, src], 10 ** 6, 10 ** 6 + 2000)
            tsrc.close()
        # the empty R: OK, dst untrained
        e_ix = ivf()
        e = _connect(world, e_ix, r)
        res["empty"] = _status(lambda: res.__setitem__("empty_n", e.rebuild_from_range([src, sib], 5 * 10 ** 8, 6 * 10 ** 8)))
        res["empty_fresh"] = not e_ix.is_trained() and e_ix.get_count() == 0 and res.get("empty_n") == 0
        e.close()
        # argument errors, refused by the library on the rank that meets them (every rank passes them alike here)
        a_ix = ivf()
        a = _connect(world, a_ix, r)
        L = b200vs.lib()
        import ctypes
        n_rows = ctypes.c_int64(0)

        def call(handles, n_src=None):
            arr = (ctypes.c_void_p * max(1, len(handles)))(*handles) if handles else None
            return L.b200vs_shard_rebuild_from_range(a.h, len(handles) if n_src is None else n_src, arr, 0, ALL, ctypes.byref(n_rows))
        res["args"] = [call([src.h], n_src=0), call([src.h] * 17, n_src=17), call([src.h, None]), call([a.h]), call([src.h, src.h]),
                       L.b200vs_shard_rebuild_from_range(a.h, 1, None, 0, ALL, ctypes.byref(n_rows))]
        res["args_fresh"] = not a_ix.is_trained() and a_ix.get_count() == 0
        a.close()
        # IVF_PQ sets keep only codes
        psrc = _connect(world, b200vs.Index(IVF_PQ, L2, 16, nlist=nlist, pq_m=4, pq_nbits=4), r)
        pdst = _connect(world, b200vs.Index(IVF_PQ, L2, 16, nlist=nlist, pq_m=4, pq_nbits=4), r)
        res["pq"] = _status(lambda: pdst.rebuild_from_range([psrc], 0, ALL))
        pdst.close()
        psrc.close()
        # row-sharded: an HNSW dst below its rank's share of R on one rank, and an id held by two sets
        hkw = dict(hnsw_m=8, hnsw_efc=32)
        h1_ix = b200vs.Index(HNSW, L2, D, max_elements=10 * n, **hkw)
        h1 = _connect(world, h1_ix, r)
        h1.add(x[:300][r::W], ids[:300][r::W])
        h2_ix = b200vs.Index(HNSW, L2, D, max_elements=10 * n, **hkw)
        h2 = _connect(world, h2_ix, r)
        h2.add(x[300:400][r::W], ids[300:400][r::W])
        hblob = (h1_ix.get_trained_state().copy(), h2_ix.get_trained_state().copy())
        for key, me, srcs, lo, hi in (("hnsw_small", 1, [h1], 0, ALL), ("hnsw_dup", 10 * n, [h1, h2], 0, ALL)):
            if key == "hnsw_dup":  # ids[250:260] live in both sets, each copy on its owner rank
                h2.add(x[250:260][r::W], ids[250:260][r::W])
                hblob = (hblob[0], h2_ix.get_trained_state().copy())
            dix = b200vs.Index(HNSW, L2, D, max_elements=me if r == bad else 10 * n, **hkw)
            dsh = _connect(world, dix, r)
            res[key] = _status(lambda: dsh.rebuild_from_range(srcs, lo, hi))
            res[key + "_dst_same"] = dix.get_count() == 0
            res[key + "_use"] = _status(lambda: (dsh.delete(np.array([12345], np.int64)), res.__setitem__(key + "_dst_search", dsh.search(xq, 5, efsearch=32))))
            dsh.close()
        res["hnsw_src_same"] = np.array_equal(h1_ix.get_trained_state(), hblob[0]) and np.array_equal(h2_ix.get_trained_state(), hblob[1])
        h1.close()
        h2.close()
        src.close()
        sib.close()
        return res

    outs = _ranks(W, rank)
    holders = [o["dup_holders"] for o in outs]
    assert any(h[0] for h in holders) and any(h[1] for h in holders)
    if W > 1:
        assert [h[0] for h in holders].index(True) != [h[1] for h in holders].index(True), "the dup copies share a rank"
    want = dict(range=EILLEGAL_PARAMETERS, trained=EILLEGAL_PARAMETERS, params=EILLEGAL_PARAMETERS, metric=EILLEGAL_PARAMETERS,
                dup=EVECTOR_ID_DUPLICATED, pq=EVECTOR_NOT_SUPPORT, hnsw_small=EILLEGAL_PARAMETERS, hnsw_dup=EVECTOR_ID_DUPLICATED,
                empty=b200vs.OK)
    if W > 1:
        want.update(rank=EILLEGAL_PARAMETERS, few=EILLEGAL_PARAMETERS)
    for r, o in enumerate(outs):
        for key, v in want.items():
            assert o[key] == v, f"W={W} rank {r}: {key} returned {o[key]}, want {v}"
            if key + "_dst_same" in o:
                assert o[key + "_dst_same"], f"rank {r}: {key} changed dst"
            if key + "_use" in o:
                assert o[key + "_use"] == b200vs.OK, f"rank {r}: dst unusable after {key}: status {o[key + '_use']}"
            if key + "_dst_search" in o:
                _eq(o[key + "_dst_search"], outs[0][key + "_dst_search"], f"rank {r}: dst search after {key}")
            if key + "_src_same" in o:
                assert o[key + "_src_same"], f"rank {r}: {key} changed a source"
                assert o[key + "_src_search"], f"rank {r}: a source searches differently after {key}"
        assert o["empty_fresh"], f"rank {r}: the empty R trained or filled dst"
        assert o["args"] == [EILLEGAL_PARAMETERS] * 6, f"rank {r}: argument refusals {o['args']}"
        assert o["args_fresh"], f"rank {r}: an argument refusal changed dst"
        assert o["hnsw_src_same"], f"rank {r}: a refusal changed an HNSW source"


# ---------------------------------------------------------------------------------------------
# 6. concurrency: a split's child and parent at once from one set, started in opposite orders on the two ranks, while the
# set serves searches; then a merge at once with a split of one of its sources.  The loopback ranks meet on the host, so this
# checks the locks (no rebuild waits for another's gate, reads go on, results equal the sequential ones), not the device
# synchronisation that makes interleaved collectives unsafe on NCCL over real GPUs (include/b200vs.h)
# ---------------------------------------------------------------------------------------------
def case_concurrency(W):
    rng = np.random.default_rng(130 + W)
    nlist = 4 * W
    n = 60000 * W
    x = rng.standard_normal((n, D)).astype(np.float32)
    ids = np.arange(n, dtype=np.int64)
    parts = _split(W, n)
    xq = rng.standard_normal((16, D)).astype(np.float32)
    mid = n // 2
    readers = World(W)

    def rank(r, world):
        def set_of(xs, ids_, train):
            ix = b200vs.Index(IVF_FLAT, L2, D, nlist=nlist)
            sh = _connect(world, ix, r)
            sh.train(train)
            sh.add(xs, ids_)
            return ix, sh

        a_ix, a = set_of(x[parts[r]], ids[parts[r]], x[parts[r]][:2000])
        b_ix, b = set_of(x[parts[r]][:5000] + 1, n + ids[parts[r]][:5000], x[parts[r]][:2000] + 1)
        want = a.search(xq, 10, seq=0, nprobe=4)
        got, errs, done = [], [], [False]

        def reader():
            try:
                s = 1
                while True:
                    got.append(a.search(xq, 10, seq=s, nprobe=4))
                    s += 1
                    if all(readers.gather(r, done[0])) or s >= 100000:
                        break
            except Exception as e:  # noqa: BLE001 - reported below
                errs.append(e)

        def fresh():
            ix = b200vs.Index(IVF_FLAT, L2, D, nlist=nlist)
            return ix, _connect(world, ix, r)

        def at_once(jobs):
            """runs (dst, srcs, lo, hi) jobs on one thread each, started in rank order on even ranks and reversed on odd ones"""
            res = [None] * len(jobs)

            def run(i):
                dst, srcs, lo, hi = jobs[i]
                res[i] = _status(lambda: dst.rebuild_from_range(srcs, lo, hi))
            order = list(range(len(jobs)))
            if r % 2:
                order.reverse()
            ths = []
            for i in order:
                th = threading.Thread(target=run, args=(i,), daemon=True)
                th.start()
                ths.append(th)
                time.sleep(0.05)  # the first job holds its gates by the time the second starts
            for th in ths:
                th.join(timeout=CASE_TIMEOUT - 60)
            return res

        rd = threading.Thread(target=reader, daemon=True)
        rd.start()
        (c_ix, c), (p_ix, p) = fresh(), fresh()
        split = at_once([(c, [a], mid, ALL), (p, [a], 0, mid)])
        (m_ix, m), (c2_ix, c2) = fresh(), fresh()
        merge = at_once([(m, [a, b], 0, ALL), (c2, [a], mid, ALL)])
        done[0] = True
        rd.join()
        # the sequential references
        outs = {}
        for key, ix, srcs, lo, hi in (("c", c_ix, [a], mid, ALL), ("p", p_ix, [a], 0, mid), ("m", m_ix, [a, b], 0, ALL),
                                      ("c2", c2_ix, [a], mid, ALL)):
            rix, rsh = fresh()
            rsh.rebuild_from_range(srcs, lo, hi)
            outs[key] = (_snap(ix, IVF_FLAT, nlist), _snap(rix, IVF_FLAT, nlist))
            rsh.close()
        for s in (c, p, m, c2, a, b):
            s.close()
        return dict(split=split, merge=merge, want=want, got=got, errs=[str(e) for e in errs], snaps=outs)

    outs = _ranks(W, rank)
    for r, o in enumerate(outs):
        assert o["split"] == [b200vs.OK] * 2 and o["merge"] == [b200vs.OK] * 2, f"rank {r}: {o['split']} {o['merge']}"
        assert not o["errs"], f"rank {r}: {o['errs']}"
        assert len(o["got"]) >= 1
        for i, g in enumerate(o["got"]):
            _eq(g, o["want"], f"rank {r}: read {i} during the rebuilds")
        for key, (got, ref) in o["snaps"].items():
            _snap_eq(got, ref, f"rank {r}: {key} vs its sequential rebuild")


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


@pytest.mark.parametrize("name", sorted(KINDS))
def test_world1(name):
    case_ranges(1, name)


@pytest.mark.parametrize("name", LIST_NAMES)
def test_lists(name):
    _run("case_ranges", name)


@pytest.mark.parametrize("name", ROW_NAMES)
def test_rows(name):
    _run("case_ranges", name, worlds=(2, 3))


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
