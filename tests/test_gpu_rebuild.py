"""Index rebuilds: b200vs_need_rebuild follows the reference plugins' NeedToRebuild rule for every type, flipping exactly at
its thresholds, and b200vs_rebuild_from gives an index equal, byte for byte, to a fresh train + add of the old index's live
rows in ascending id order (trained state, lists, ids, rows, search and range results, and for HNSW the graph), while the
old index keeps serving."""
import os
import tempfile
import threading
import time

import numpy as np
import pytest

import b200vs
import kmeans_restate as kr
import oracle_lib
from b200vs import (BINARY_FLAT, BINARY_IVF_FLAT, COSINE, EILLEGAL_PARAMETERS, EVECTOR_NOT_SUPPORT, FLAT, HAMMING, HNSW, IP,
                    IVF_FLAT, IVF_PQ, L2)
from gpu_util import require_gpu

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _gpu():
    require_gpu()


def rows(rng, n, d):
    return rng.standard_normal((n, d)).astype(np.float32)


def nlist_of(ix):
    st = ix.get_trained_state()
    return int(st[:32].view(np.int64)[1]) if st.size >= 32 else 1


def sorted_live(ix):
    """(rows, ids) of every live row in ascending id order (rows sharing an id keep their export order)."""
    if ix.type == HNSW:
        _, _, _, ids = ix.export_lists(1, with_vectors=False)
        ids = np.sort(ids)
        x, found = ix.reconstruct(ids)
        assert found.all()
        return x, ids
    nl = nlist_of(ix) if ix.type != IVF_PQ else 1
    _, vec, codes, ids = ix.export_lists(nl)
    order = np.argsort(ids, kind="stable")
    return (codes if ix.binary else vec)[order], ids[order]


def fresh_build(src, **params):
    """A fresh index of src's kind trained and filled with src's live rows in ascending id order."""
    x, ids = sorted_live(src)
    f = b200vs.Index(src.type, src.metric, src.dim, **params)
    if src.type == HNSW:
        f.add_batched(x, ids)
        return f
    f.train(x)
    f.add(x, ids)
    return f


def assert_same_index(a, b, queries, k=10):
    """Trained state, lists and every read of a and b agree bit for bit."""
    assert a.get_count() == b.get_count() and a.get_deleted_count() == b.get_deleted_count()
    sa, sb = a.get_trained_state(), b.get_trained_state()
    assert np.array_equal(sa, sb), "trained states differ"
    if a.type != HNSW:
        nl = nlist_of(a) if a.type != IVF_PQ or a.sub_type() == IVF_PQ else 1
        cs = 0
        if a.type == IVF_PQ and a.sub_type() == IVF_PQ:
            cs = (a.params.pq_m * (a.params.pq_nbits or 8) + 7) // 8
        ea = a.export_lists(nl, with_vectors=cs == 0, code_size=cs)
        eb = b.export_lists(nl, with_vectors=cs == 0, code_size=cs)
        for u, v in zip(ea, eb):
            assert (u is None and v is None) or np.array_equal(u, v), "exported lists differ"
    for kw in ({}, {"exact_only": True}, {"nprobe": 4}):
        Da, Ia = a.search(queries, k, **kw)
        Db, Ib = b.search(queries, k, **kw)
        assert np.array_equal(Ia, Ib) and np.array_equal(Da.view(np.uint32), Db.view(np.uint32)), f"search {kw} differs"
    if a.type != HNSW:
        radius = 40.0 if a.binary else (float(np.median(a.search(queries, k)[0][:, -1])) if a.metric == L2 else 0.6)
        ra, rb = a.range_search(queries, radius, 256), b.range_search(queries, radius, 256)
        for u, v in zip(ra, rb):
            assert np.array_equal(u.view(np.uint32) if u.dtype == np.float32 else u, v.view(np.uint32) if v.dtype == np.float32 else v)


# ---------------------------------------------------------------------------------------------------------------- the rule

def test_need_rebuild_ivf_flat_degenerate_and_trained():
    rng = np.random.default_rng(1)
    d, nlist = 16, 8
    thr = 256 * nlist
    # degenerate: trained on fewer rows than nlist -> nlist 1; rebuild from 256 * nlist_org rows on
    ix = b200vs.Index(IVF_FLAT, L2, d, nlist=nlist)
    ix.train(rows(rng, 5, d))
    assert nlist_of(ix) == 1 and not ix.need_rebuild()
    ix.add(rows(rng, thr - 1, d), np.arange(thr - 1))
    assert not ix.need_rebuild()
    ix.add(rows(rng, 1, d), [thr - 1])
    assert ix.need_rebuild()
    ix.delete([0])
    assert not ix.need_rebuild()
    # trained on t rows: from 256 * nlist rows on, once t <= count / 2
    t = 3000
    iv = b200vs.Index(IVF_FLAT, L2, d, nlist=nlist)
    x = rows(rng, t, d)
    iv.train(x)
    iv.train(rows(rng, 9000, d))  # ignored: the index is trained, train_rows stays t
    iv.add(rows(rng, 2 * t - 1, d), np.arange(2 * t - 1))
    assert not iv.need_rebuild()
    iv.add(rows(rng, 1, d), [10 ** 6])
    assert iv.need_rebuild()
    # count-based after save / load: train_rows becomes the loaded count
    with tempfile.TemporaryDirectory() as td:
        p = os.path.join(td, "ivf.idx")
        iv.save(p)
        lo = b200vs.Index(IVF_FLAT, L2, d, nlist=nlist)
        lo.load(p)
        assert lo.get_count() == 2 * t and not lo.need_rebuild()
        lo.add(rows(rng, 2 * t - 1, d), np.arange(2 * 10 ** 6, 2 * 10 ** 6 + 2 * t - 1))
        assert not lo.need_rebuild()
        lo.add(rows(rng, 1, d), [3 * 10 ** 6])
        assert lo.need_rebuild()
    # created with nlist 1: never
    one = b200vs.Index(IVF_FLAT, L2, d, nlist=1)
    one.train(rows(rng, 10, d))
    one.add(rows(rng, 600, d), np.arange(600))
    assert not one.need_rebuild()
    # untrained: never
    assert not b200vs.Index(IVF_FLAT, L2, d, nlist=nlist).need_rebuild()


def test_need_rebuild_after_set_trained_state():
    # set_trained_state takes the live count of the call as train_rows: 0 on a fresh index, so the rule then waits for
    # 256 * nlist rows only
    rng = np.random.default_rng(6)
    d, nlist = 16, 8
    thr = 256 * nlist
    iv = b200vs.Index(IVF_FLAT, L2, d, nlist=nlist)
    iv.train(rows(rng, 3000, d))
    st = iv.get_trained_state()
    ix = b200vs.Index(IVF_FLAT, L2, d, nlist=nlist)
    ix.set_trained_state(st)
    ix.add(rows(rng, thr - 1, d), np.arange(thr - 1))
    assert not ix.need_rebuild()
    ix.add(rows(rng, 1, d), [thr - 1])
    assert ix.need_rebuild()
    # the same index loaded from a file: train_rows = the loaded count, so it no longer needs one
    with tempfile.TemporaryDirectory() as td:
        p = os.path.join(td, "ivf.idx")
        ix.save(p)
        lo = b200vs.Index(IVF_FLAT, L2, d, nlist=nlist)
        lo.load(p)
        assert not lo.need_rebuild()


def test_need_rebuild_binary_ivf():
    rng = np.random.default_rng(2)
    dim, nlist = 64, 4
    thr = 256 * nlist
    ix = b200vs.Index(BINARY_IVF_FLAT, HAMMING, dim, nlist=nlist)
    ix.train(rng.integers(0, 256, (3, dim // 8), dtype=np.uint8))
    ix.add(rng.integers(0, 256, (thr - 1, dim // 8), dtype=np.uint8), np.arange(thr - 1))
    assert not ix.need_rebuild()
    ix.add(rng.integers(0, 256, (1, dim // 8), dtype=np.uint8), [thr])
    assert ix.need_rebuild()
    t = 1500
    tr = b200vs.Index(BINARY_IVF_FLAT, HAMMING, dim, nlist=nlist)
    tr.train(rng.integers(0, 256, (t, dim // 8), dtype=np.uint8))
    tr.add(rng.integers(0, 256, (2 * t - 1, dim // 8), dtype=np.uint8), np.arange(2 * t - 1))
    assert not tr.need_rebuild()
    tr.add(rng.integers(0, 256, (1, dim // 8), dtype=np.uint8), [10 ** 6])
    assert tr.need_rebuild()


def test_need_rebuild_ivf_pq():
    rng = np.random.default_rng(3)
    d, nlist, M, nbits = 16, 4, 4, 4
    need = max(256 * nlist, 256 * (1 << nbits))  # 4096
    ix = b200vs.Index(IVF_PQ, L2, d, nlist=nlist, pq_m=M, pq_nbits=nbits)
    assert not ix.need_rebuild()
    ix.train(rows(rng, 100, d))
    assert ix.sub_type() == FLAT
    ix.add(rows(rng, need - 1, d), np.arange(need - 1))
    assert not ix.need_rebuild()
    ix.add(rows(rng, 1, d), [need - 1])
    assert ix.need_rebuild()
    ix.delete([5])
    assert not ix.need_rebuild()
    pq = b200vs.Index(IVF_PQ, L2, d, nlist=nlist, pq_m=M, pq_nbits=nbits)
    t = need
    pq.train(rows(rng, t, d))
    assert pq.sub_type() == IVF_PQ
    pq.add(rows(rng, 2 * t - 1, d), np.arange(2 * t - 1))
    assert not pq.need_rebuild()
    pq.add(rows(rng, 1, d), [10 ** 6])
    assert pq.need_rebuild()
    with tempfile.TemporaryDirectory() as td:
        p = os.path.join(td, "pq.idx")
        pq.save(p)
        lo = b200vs.Index(IVF_PQ, L2, d, nlist=nlist, pq_m=M, pq_nbits=nbits)
        lo.load(p)
        assert not lo.need_rebuild()  # train_rows = 2t: needs 4t rows
        lo.add(rows(rng, 2 * t - 1, d), np.arange(2 * 10 ** 6, 2 * 10 ** 6 + 2 * t - 1))
        assert not lo.need_rebuild()
        lo.add(rows(rng, 1, d), [3 * 10 ** 6])
        assert lo.need_rebuild()


def test_need_rebuild_hnsw_deletes_and_upserts():
    rng = np.random.default_rng(4)
    d, n = 16, 100
    for via_upsert in (False, True):
        ix = b200vs.Index(HNSW, L2, d, hnsw_m=8, hnsw_efc=40, max_elements=1000)
        ix.add(rows(rng, n, d), np.arange(n))
        assert not ix.need_rebuild()
        # deleted > (live + deleted) / 2: with 100 nodes and only tombstones added by upserts, after u upserts there are
        # 100 + u nodes and u tombstones
        if via_upsert:
            for u in range(1, 200):
                ix.upsert(rows(rng, 1, d), [u % n])
                e = n + u
                assert ix.need_rebuild() == (u > e // 2), u
        else:
            for u in range(1, n + 1):
                ix.delete([u - 1])
                assert ix.need_rebuild() == (u > n // 2), u


def test_need_rebuild_flat_types_never():
    rng = np.random.default_rng(5)
    f = b200vs.Index(FLAT, L2, 8)
    f.add(rows(rng, 10, 8), np.arange(10))
    f.delete(np.arange(9))
    assert not f.need_rebuild()
    b = b200vs.Index(BINARY_FLAT, HAMMING, 64)
    b.add(rng.integers(0, 256, (10, 8), dtype=np.uint8), np.arange(10))
    b.delete(np.arange(9))
    assert not b.need_rebuild()


# -------------------------------------------------------------------------------------------------- equality with a fresh build

def ivf_history(ix, rng, d, binary=False):
    """Adds with ids out of order, deletes, upserts and enough deletes to compact the arena."""
    def gen(n):
        return rng.integers(0, 256, (n, d // 8), dtype=np.uint8) if binary else rows(rng, n, d)
    ids = rng.permutation(12000)[:9000] + 5
    ix.add(gen(ids.size), ids)
    ix.delete(ids[:2500])
    ix.upsert(gen(700), ids[3000:3700])
    ix.add(gen(300), np.arange(20000, 20300)[::-1])
    ix.delete(ids[4000:7800])  # garbage + tombstones past the live rows: compaction


@pytest.mark.parametrize("metric", [L2, IP])
@pytest.mark.parametrize("degenerate", [False, True])
def test_rebuild_ivf_flat_equals_fresh(metric, degenerate):
    rng = np.random.default_rng(10 + metric)
    d, nlist = 32, 16
    src = b200vs.Index(IVF_FLAT, metric, d, nlist=nlist)
    src.train(rows(rng, 7 if degenerate else 2000, d))
    ivf_history(src, rng, d)
    dst = b200vs.Index(IVF_FLAT, metric, d, nlist=nlist)
    n = dst.rebuild_from(src)
    assert n == src.get_count()
    assert nlist_of(dst) == nlist  # the rows are now enough to train every list
    assert_same_index(dst, fresh_build(src, nlist=nlist), rows(rng, 40, d))


def test_rebuild_ivf_flat_large_subsample():
    rng = np.random.default_rng(11)
    d, nlist = 64, 8  # 256 * 8 = 2048 < count: k-means draws its subsample on the device
    src = b200vs.Index(IVF_FLAT, L2, d, nlist=nlist)
    src.train(rows(rng, 500, d))
    ids = rng.permutation(40000)[:30000]
    src.add(rows(rng, ids.size, d), ids)
    dst = b200vs.Index(IVF_FLAT, L2, d, nlist=nlist)
    assert dst.rebuild_from(src) == 30000
    assert_same_index(dst, fresh_build(src, nlist=nlist), rows(rng, 64, d))


def test_rebuild_ivf_flat_cosine_rows_as_stored():
    rng = np.random.default_rng(12)
    d, nlist = 32, 8
    oracle = oracle_lib.load()
    src = b200vs.Index(IVF_FLAT, COSINE, d, nlist=nlist)
    src.train(rows(rng, 1000, d))
    ids = rng.permutation(5000)[:3000]
    src.add(rows(rng, ids.size, d) * 3.0, ids)
    src.delete(ids[:200])
    dst = b200vs.Index(IVF_FLAT, COSINE, d, nlist=nlist)
    dst.rebuild_from(src)
    x, sids = sorted_live(src)  # stored rows: already normalised
    cent = kr.kmeans(oracle, IP, x, nlist)  # k-means on the stored rows as they are (IP assignment = cosine's)
    assert np.array_equal(dst.get_trained_state(), b200vs.ivf_state_blob(cent, COSINE))
    labels = oracle.assign(IP, x, cent, nthreads=8)
    off, vec, _, got_ids = dst.export_lists(nlist)
    for l in range(nlist):
        want = labels == l
        assert np.array_equal(got_ids[off[l]:off[l + 1]], sids[want])
        assert np.array_equal(vec[off[l]:off[l + 1]].view(np.uint32), x[want].view(np.uint32))


def test_rebuild_hnsw_cosine_rows_as_stored():
    # faiss's normaliser leaves rows whose squared norm is within 1e-5 of 1 alone, so a second pass over IVF rows is
    # invisible; hnswlib's divides every row again, and on these rows that changes bits
    rng = np.random.default_rng(18)
    d, n = 32, 3000
    kw = dict(hnsw_m=8, hnsw_efc=40, max_elements=10000)
    src = b200vs.Index(HNSW, COSINE, d, **kw)
    ids = rng.permutation(8000)[:n]
    src.add_batched(rows(rng, n, d) * 3.0, ids)
    src.delete(ids[:300])
    dst = b200vs.Index(HNSW, COSINE, d, **kw)
    assert dst.rebuild_from(src) == n - 300
    x, sids = sorted_live(src)
    got, found = dst.reconstruct(sids)
    assert found.all() and np.array_equal(got.view(np.uint32), x.view(np.uint32))
    twice = oracle_lib.load().normalize_hnsw(x)
    assert not np.array_equal(twice.view(np.uint32), x.view(np.uint32))


def test_rebuild_binary_ivf_equals_fresh():
    rng = np.random.default_rng(13)
    dim, nlist = 128, 8
    src = b200vs.Index(BINARY_IVF_FLAT, HAMMING, dim, nlist=nlist)
    src.train(rng.integers(0, 256, (3, dim // 8), dtype=np.uint8))  # degenerate: nlist 1
    ivf_history(src, rng, dim, binary=True)
    dst = b200vs.Index(BINARY_IVF_FLAT, HAMMING, dim, nlist=nlist)
    assert dst.rebuild_from(src) == src.get_count()
    assert nlist_of(dst) == nlist
    assert_same_index(dst, fresh_build(src, nlist=nlist), rng.integers(0, 256, (40, dim // 8), dtype=np.uint8))


@pytest.mark.parametrize("enough", [True, False])
def test_rebuild_ivf_pq_inner_flat(enough):
    rng = np.random.default_rng(14)
    d, nlist, M, nbits = 32, 4, 8, 4
    need = max(256 * nlist, 256 * (1 << nbits))
    kw = dict(nlist=nlist, pq_m=M, pq_nbits=nbits)
    src = b200vs.Index(IVF_PQ, L2, d, **kw)
    src.train(rows(rng, 10, d))
    ids = rng.permutation(3 * need)[:need + 500] + 1
    src.add(rows(rng, ids.size, d), ids)
    src.delete(ids[:(200 if enough else 1000)])
    assert src.sub_type() == FLAT
    dst = b200vs.Index(IVF_PQ, L2, d, **kw)
    assert dst.rebuild_from(src) == src.get_count()
    assert dst.sub_type() == (IVF_PQ if enough else FLAT)
    assert_same_index(dst, fresh_build(src, **kw), rows(rng, 40, d))
    if enough:  # IVF-PQ mode stores only codes: no rebuild from it
        with pytest.raises(b200vs.B200VSError) as e:
            b200vs.Index(IVF_PQ, L2, d, **kw).rebuild_from(dst)
        assert e.value.code == EVECTOR_NOT_SUPPORT


def test_rebuild_hnsw_equals_fresh():
    rng = np.random.default_rng(15)
    d, n = 32, 6000
    kw = dict(hnsw_m=16, hnsw_efc=64, max_elements=20000)
    src = b200vs.Index(HNSW, L2, d, **kw)
    ids = rng.permutation(10000)[:n]
    src.add_batched(rows(rng, n, d), ids)
    src.upsert(rows(rng, 500, d), ids[:500])
    src.delete(ids[1000:4000])
    assert src.need_rebuild()
    dst = b200vs.Index(HNSW, L2, d, **kw)
    assert dst.rebuild_from(src) == src.get_count()
    assert dst.get_deleted_count() == 0 and not dst.need_rebuild()
    f = fresh_build(src, **kw)
    assert np.array_equal(dst.get_trained_state(), f.get_trained_state()), "graph blobs differ"
    assert_same_index(dst, f, rows(rng, 40, d))


# ------------------------------------------------------------------------------------------------------ src keeps serving

def test_src_keeps_serving_during_rebuild():
    rng = np.random.default_rng(16)
    d, nlist = 64, 64
    src = b200vs.Index(IVF_FLAT, L2, d, nlist=nlist)
    src.train(rows(rng, 20000, d))
    src.add(rows(rng, 300000, d), np.arange(300000))
    q = rows(rng, 16, d)
    D0, I0 = src.search(q, 10, nprobe=8)
    before = src.export_lists(nlist)
    stop, started, bad, spans = threading.Event(), threading.Event(), [], []

    def reader():
        while not stop.is_set():
            t0 = time.perf_counter()
            D, I = src.search(q, 10, nprobe=8)
            spans.append((t0, time.perf_counter()))
            started.set()
            if not (np.array_equal(I, I0) and np.array_equal(D.view(np.uint32), D0.view(np.uint32))):
                bad.append(1)

    t = threading.Thread(target=reader)
    t.start()
    try:
        started.wait(60)
        dst = b200vs.Index(IVF_FLAT, L2, d, nlist=nlist)
        r0 = time.perf_counter()
        dst.rebuild_from(src)
        r1 = time.perf_counter()
    finally:
        stop.set()
        t.join()
    assert not bad
    inside = [s for s in spans if s[0] > r0 and s[1] < r1]
    assert inside, f"no search ran while the rebuild ran ({len(spans)} searches, rebuild {r1 - r0:.3f} s)"
    for u, v in zip(before, src.export_lists(nlist)):
        assert np.array_equal(u, v)


def test_writers_on_inner_flat_ivf_pq_wait_for_the_rebuild():
    # an IVF-PQ region in inner-Flat mode takes its writes under the inner index's lock: the rebuild must read one
    # consistent state of it, whichever writes it came between
    rng = np.random.default_rng(19)
    d, n0, nops = 32, 3000, 600
    kw = dict(nlist=4, pq_m=8, pq_nbits=4)  # need = 4096 > n0 + nops: dst stays inner Flat, its rows exportable
    src = b200vs.Index(IVF_PQ, L2, d, **kw)
    src.train(rows(rng, 10, d))
    x0, y = rows(rng, n0, d), rows(rng, nops, d)
    src.add(x0, np.arange(n0))
    done, stop, first = [0], threading.Event(), threading.Event()

    def writer():
        for j in range(nops):
            if stop.is_set():
                break
            src.add(y[j:j + 1], [10 ** 6 + j])
            src.delete([j])
            done[0] = j + 1
            first.set()

    t = threading.Thread(target=writer)
    t.start()
    try:
        first.wait(60)
        at_start = done[0]
        dst = b200vs.Index(IVF_PQ, L2, d, **kw)
        dst.rebuild_from(src)
    finally:
        stop.set()
        t.join()
    assert done[0] > at_start  # the writer went on after the rebuild began
    assert dst.sub_type() == FLAT
    _, vec, _, ids = dst.export_lists(1)
    assert np.all(np.diff(ids) > 0)  # ascending id order
    a = int((ids >= 10 ** 6).sum())  # adds the rebuild saw; it saw a - 1 or a deletes
    r = n0 - int((ids < n0).sum())
    assert r in (a - 1, a), (a, r)
    want_ids = np.concatenate([np.arange(r, n0), 10 ** 6 + np.arange(a)])
    want_rows = np.concatenate([x0[r:], y[:a]])
    assert np.array_equal(ids, want_ids)
    assert np.array_equal(vec.view(np.uint32), want_rows.view(np.uint32))


# --------------------------------------------------------------------------------------------------------------- refusals

def snapshot(ix):
    return (ix.get_count(), ix.get_deleted_count(), ix.is_trained(), bytes(ix.get_trained_state()))


def test_refusals_leave_both_unchanged():
    rng = np.random.default_rng(17)
    d, nlist = 16, 4
    src = b200vs.Index(IVF_FLAT, L2, d, nlist=nlist)
    src.train(rows(rng, 500, d))
    src.add(rows(rng, 500, d), np.arange(500))

    def refused(dst, s, code):
        a, b = snapshot(dst), snapshot(s)
        with pytest.raises(b200vs.B200VSError) as e:
            dst.rebuild_from(s)
        assert e.value.code == code, e.value.msg
        assert snapshot(dst) == a and snapshot(s) == b

    refused(src, src, EILLEGAL_PARAMETERS)
    trained = b200vs.Index(IVF_FLAT, L2, d, nlist=nlist)
    trained.train(rows(rng, 100, d))
    refused(trained, src, EILLEGAL_PARAMETERS)
    for other in (b200vs.Index(IVF_FLAT, IP, d, nlist=nlist), b200vs.Index(IVF_FLAT, L2, d + 8, nlist=nlist),
                  b200vs.Index(IVF_FLAT, L2, d, nlist=nlist + 1), b200vs.Index(IVF_PQ, L2, d, nlist=nlist, pq_m=4)):
        refused(other, src, EILLEGAL_PARAMETERS)
    pq_a = b200vs.Index(IVF_PQ, L2, d, nlist=nlist, pq_m=4, pq_nbits=4)
    pq_a.train(rows(rng, 10, d))
    pq_a.add(rows(rng, 100, d), np.arange(100))
    refused(b200vs.Index(IVF_PQ, L2, d, nlist=nlist, pq_m=8, pq_nbits=4), pq_a, EILLEGAL_PARAMETERS)
    refused(b200vs.Index(IVF_PQ, L2, d, nlist=nlist, pq_m=4, pq_nbits=8), pq_a, EILLEGAL_PARAMETERS)
    pq_mode = b200vs.Index(IVF_PQ, L2, d, nlist=nlist, pq_m=4, pq_nbits=4)
    pq_mode.train(rows(rng, 4096, d))
    pq_mode.add(rows(rng, 100, d), np.arange(100))
    refused(b200vs.Index(IVF_PQ, L2, d, nlist=nlist, pq_m=4, pq_nbits=4), pq_mode, EVECTOR_NOT_SUPPORT)
    hs = b200vs.Index(HNSW, L2, d, hnsw_m=8, hnsw_efc=40, max_elements=1000)
    hs.add(rows(rng, 300, d), np.arange(300))
    refused(b200vs.Index(HNSW, L2, d, hnsw_m=8, hnsw_efc=40, max_elements=299), hs, EILLEGAL_PARAMETERS)
    refused(b200vs.Index(HNSW, L2, d, hnsw_m=12, hnsw_efc=40, max_elements=1000), hs, EILLEGAL_PARAMETERS)
    refused(b200vs.Index(HNSW, L2, d, hnsw_m=8, hnsw_efc=50, max_elements=1000), hs, EILLEGAL_PARAMETERS)
    full = b200vs.Index(HNSW, L2, d, hnsw_m=8, hnsw_efc=40, max_elements=1000)
    full.add(rows(rng, 1, d), [7])
    refused(full, hs, EILLEGAL_PARAMETERS)
    refused(b200vs.Index(FLAT, L2, d), src, EILLEGAL_PARAMETERS)  # a type mismatch, whichever side is Flat
    fl = b200vs.Index(FLAT, L2, d)
    fl.add(rows(rng, 10, d), np.arange(10))
    refused(b200vs.Index(FLAT, L2, d), fl, EVECTOR_NOT_SUPPORT)
    bf = b200vs.Index(BINARY_FLAT, HAMMING, 64)
    refused(b200vs.Index(BINARY_FLAT, HAMMING, 64), bf, EVECTOR_NOT_SUPPORT)
    # the exact max_elements fits
    ok = b200vs.Index(HNSW, L2, d, hnsw_m=8, hnsw_efc=40, max_elements=300)
    assert ok.rebuild_from(hs) == 300


def test_default_and_explicit_default_parameters_match():
    rng = np.random.default_rng(20)
    d = 16
    src = b200vs.Index(IVF_FLAT, L2, d)  # nlist 0 = 2048
    src.train(rows(rng, 100, d))
    src.add(rows(rng, 100, d), np.arange(100))
    assert b200vs.Index(IVF_FLAT, L2, d, nlist=2048).rebuild_from(src) == 100
    pq = b200vs.Index(IVF_PQ, L2, d, nlist=4, pq_m=16, pq_nbits=0)  # nbits 0 = 8
    pq.train(rows(rng, 10, d))
    pq.add(rows(rng, 50, d), np.arange(50))
    assert b200vs.Index(IVF_PQ, L2, d, nlist=4, pq_m=16, pq_nbits=8).rebuild_from(pq) == 50


def test_empty_src_leaves_dst_untrained():
    for kind, kw in ((IVF_FLAT, dict(nlist=4)), (IVF_PQ, dict(nlist=4, pq_m=4)), (HNSW, dict(hnsw_m=8, hnsw_efc=40))):
        src = b200vs.Index(kind, L2, 16, **kw)
        dst = b200vs.Index(kind, L2, 16, **kw)
        assert dst.rebuild_from(src) == 0
        assert dst.get_count() == 0 and (kind == HNSW or not dst.is_trained())
    src = b200vs.Index(IVF_FLAT, L2, 16, nlist=4)
    src.train(np.ones((10, 16), np.float32))
    src.add(np.ones((3, 16), np.float32), [1, 2, 3])
    src.delete([1, 2, 3])
    dst = b200vs.Index(IVF_FLAT, L2, 16, nlist=4)
    assert dst.rebuild_from(src) == 0 and not dst.is_trained()
