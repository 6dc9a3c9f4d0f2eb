"""Split and merge rebuilds: b200vs_rebuild_from_range fills a fresh index from the live rows with id_min <= id < id_max of
one or more old indexes, and the result equals, bit for bit, a fresh index trained and filled through the ordinary host ABI
with those rows in ascending id order (trained state, lists, ids, rows, search and range results, and for HNSW the graph).
Refusals leave every index as it was, and two rebuilds from one source can run at once while it keeps serving reads."""
import ctypes
import threading
import time

import numpy as np
import pytest

import b200vs
from b200vs import (BINARY_FLAT, BINARY_IVF_FLAT, COSINE, EILLEGAL_PARAMETERS, EVECTOR_ID_DUPLICATED, EVECTOR_NOT_SUPPORT, FLAT,
                    HAMMING, HNSW, IP, IVF_FLAT, IVF_PQ, L2)
from gpu_util import require_gpu
from test_gpu_rebuild import assert_same_index, fresh_build, ivf_history, nlist_of, rows, sorted_live

pytestmark = pytest.mark.gpu

I64_MAX = 2 ** 63 - 1


@pytest.fixture(autouse=True)
def _gpu():
    require_gpu()


def gen(rng, kind, n, d):
    return rng.integers(0, 256, (n, d // 8), dtype=np.uint8) if kind in b200vs.BINARY_TYPES else rows(rng, n, d)


def rows_in(srcs, lo, hi):
    """R: the live rows with lo <= id < hi of every source, in ascending id order (ties: source order, then export order)."""
    xs, ids = [], []
    for s in srcs:
        x, i = sorted_live(s)
        keep = (i >= lo) & (i < hi)
        xs.append(x[keep])
        ids.append(i[keep])
    x, ids = np.concatenate(xs), np.concatenate(ids)
    order = np.argsort(ids, kind="stable")
    return x[order], ids[order]


def fresh_range(srcs, lo, hi, **params):
    """A fresh index of the sources' kind trained and filled through the host ABI with R in ascending id order."""
    x, ids = rows_in(srcs, lo, hi)
    s = srcs[0]
    f = b200vs.Index(s.type, s.metric, s.dim, **params)
    if s.type == HNSW:
        f.add_batched(x, ids)
        return f
    f.train(x)
    f.add(x, ids)
    return f


def queries(rng, ix, n=40):
    return gen(rng, ix.type, n, ix.dim)


def history(ix, rng):
    """A long history: ids out of order, deletes, upserts and (IVF types) a compaction.  Live ids lie in [5, 20300)."""
    if ix.type == HNSW:
        ids = rng.permutation(12000)[:5000] + 5
        ix.add_batched(rows(rng, ids.size, ix.dim) * 3.0, ids)
        ix.upsert(rows(rng, 400, ix.dim), ids[:400])
        ix.delete(ids[1000:2500])
        ix.add_batched(rows(rng, 300, ix.dim), np.arange(20000, 20300)[::-1].copy())
        return
    ivf_history(ix, rng, ix.dim, binary=ix.binary)


SPLIT_KINDS = [
    (IVF_FLAT, L2, dict(nlist=16)), (IVF_FLAT, IP, dict(nlist=16)), (IVF_FLAT, COSINE, dict(nlist=16)),
    (BINARY_IVF_FLAT, HAMMING, dict(nlist=16)), (FLAT, L2, {}), (FLAT, COSINE, {}), (BINARY_FLAT, HAMMING, {}),
    (HNSW, L2, dict(hnsw_m=12, hnsw_efc=48, max_elements=20000)),
]


@pytest.mark.parametrize("kind,metric,kw", SPLIT_KINDS)
@pytest.mark.parametrize("at", ["median", "tiny"])
def test_split_equals_fresh(kind, metric, kw, at):
    rng = np.random.default_rng(100 + kind * 7 + metric)
    d = 128 if kind in b200vs.BINARY_TYPES else 32
    src = b200vs.Index(kind, metric, d, **kw)
    if kind in (IVF_FLAT, BINARY_IVF_FLAT):
        src.train(gen(rng, kind, 3000, d))
    history(src, rng)
    before = src.get_count()
    _, live_ids = sorted_live(src)
    # "tiny": the child [0, s) holds 7 rows, fewer than nlist, so its nlist degenerates to 1
    s = int(live_ids[7] if at == "tiny" else np.median(live_ids))
    q = queries(rng, src)
    for lo, hi in ((0, s), (s, I64_MAX)):
        dst = b200vs.Index(kind, metric, d, **kw)
        want = int(((live_ids >= lo) & (live_ids < hi)).sum())
        assert dst.rebuild_from_range([src], lo, hi) == want
        _, got_ids = sorted_live(dst)
        assert got_ids.size == want and got_ids.min() >= lo and got_ids.max() < hi
        if kind in (IVF_FLAT, BINARY_IVF_FLAT):
            assert nlist_of(dst) == (1 if want < kw["nlist"] else kw["nlist"])
        f = fresh_range([src], lo, hi, **kw)
        if kind == HNSW:
            assert np.array_equal(dst.get_trained_state(), f.get_trained_state()), "graph blobs differ"
        assert_same_index(dst, f, q)
    assert src.get_count() == before


@pytest.mark.parametrize("enough", [True, False])
def test_split_ivf_pq_inner_flat(enough):
    rng = np.random.default_rng(14)
    d, nlist, M, nbits = 32, 4, 8, 4
    need = max(256 * nlist, 256 * (1 << nbits))  # 4096
    kw = dict(nlist=nlist, pq_m=M, pq_nbits=nbits)
    src = b200vs.Index(IVF_PQ, L2, d, **kw)
    src.train(rows(rng, 10, d))
    ids = rng.permutation(4 * need)[:need + 3000] + 1
    src.add(rows(rng, ids.size, d), ids)
    src.delete(ids[:500])
    assert src.sub_type() == FLAT
    _, live_ids = sorted_live(src)
    # the child [s, max) holds `need` rows (IVF-PQ) or one fewer (inner Flat again)
    s = int(live_ids[live_ids.size - need + (0 if enough else 1)])
    dst = b200vs.Index(IVF_PQ, L2, d, **kw)
    assert dst.rebuild_from_range([src], s, I64_MAX) == need - (0 if enough else 1)
    assert dst.sub_type() == (IVF_PQ if enough else FLAT)
    q = rows(rng, 40, d)
    assert_same_index(dst, fresh_range([src], s, I64_MAX, **kw), q)
    parent = b200vs.Index(IVF_PQ, L2, d, **kw)
    parent.rebuild_from_range([src], 0, s)
    assert parent.sub_type() == FLAT
    assert_same_index(parent, fresh_range([src], 0, s, **kw), q)


def test_split_hnsw_cosine_rows_as_stored():
    # hnswlib's normaliser divides every row again, so a host build from R would not keep R's bits: the rebuilt index is
    # compared with b200vs_rebuild_from of the source once every row outside the range is deleted, and with the stored rows
    rng = np.random.default_rng(18)
    d = 32
    kw = dict(hnsw_m=8, hnsw_efc=40, max_elements=20000)
    src = b200vs.Index(HNSW, COSINE, d, **kw)
    history(src, rng)
    _, live_ids = sorted_live(src)
    s = int(np.median(live_ids))
    dst = b200vs.Index(HNSW, COSINE, d, **kw)
    assert dst.rebuild_from_range([src], s, I64_MAX) == int((live_ids >= s).sum())
    x, sids = rows_in([src], s, I64_MAX)
    got, found = dst.reconstruct(sids)
    assert found.all() and np.array_equal(got.view(np.uint32), x.view(np.uint32))
    src.delete(live_ids[live_ids < s])
    ref = b200vs.Index(HNSW, COSINE, d, **kw)
    ref.rebuild_from(src)
    assert np.array_equal(dst.get_trained_state(), ref.get_trained_state()), "graph blobs differ"
    assert_same_index(dst, ref, rows(rng, 40, d))


MERGE_KINDS = [(IVF_FLAT, L2, dict(nlist=16)), (BINARY_IVF_FLAT, HAMMING, dict(nlist=16)), (FLAT, IP, {}),
               (HNSW, L2, dict(hnsw_m=12, hnsw_efc=48, max_elements=20000))]


@pytest.mark.parametrize("kind,metric,kw", MERGE_KINDS)
def test_merge_equals_fresh(kind, metric, kw):
    # the target's own index holds [0, 6000), the sibling [6000, 12000); the merged range is [2000, 10000), so each source
    # also holds rows outside it (as a split parent's index does), and those must stay out of dst
    rng = np.random.default_rng(200 + kind)
    d = 128 if kind in b200vs.BINARY_TYPES else 32
    own, sib = b200vs.Index(kind, metric, d, **kw), b200vs.Index(kind, metric, d, **kw)
    for ix, base in ((own, 0), (sib, 6000)):
        if kind in (IVF_FLAT, BINARY_IVF_FLAT):
            ix.train(gen(rng, kind, 1000, d))
        ids = rng.permutation(6000) + base
        if kind == HNSW:
            ix.add_batched(gen(rng, kind, 6000, d), ids)
        else:
            ix.add(gen(rng, kind, 6000, d), ids)
        ix.delete(ids[:700])
    dst = b200vs.Index(kind, metric, d, **kw)
    n = dst.rebuild_from_range([sib, own], 2000, 10000)  # source order does not matter: the ids are disjoint
    _, got = sorted_live(dst)
    assert n == got.size and got.min() >= 2000 and got.max() < 10000
    f = fresh_range([own, sib], 2000, 10000, **kw)
    if kind == HNSW:
        assert np.array_equal(dst.get_trained_state(), f.get_trained_state()), "graph blobs differ"
    assert_same_index(dst, f, queries(rng, own))


@pytest.mark.parametrize("kind,metric,kw", [(IVF_FLAT, L2, dict(nlist=16)), (IVF_FLAT, COSINE, dict(nlist=16)),
                                            (BINARY_IVF_FLAT, HAMMING, dict(nlist=16)),
                                            (IVF_PQ, L2, dict(nlist=4, pq_m=8, pq_nbits=4)),
                                            (HNSW, L2, dict(hnsw_m=12, hnsw_efc=48, max_elements=20000))])
def test_one_source_whole_range_equals_rebuild_from(kind, metric, kw):
    rng = np.random.default_rng(300 + kind)
    d = 128 if kind in b200vs.BINARY_TYPES else 32
    src = b200vs.Index(kind, metric, d, **kw)
    if kind != HNSW:
        src.train(gen(rng, kind, 10 if kind == IVF_PQ else 3000, d))
    history(src, rng)
    a, b = b200vs.Index(kind, metric, d, **kw), b200vs.Index(kind, metric, d, **kw)
    assert a.rebuild_from_range([src], 0, I64_MAX) == b.rebuild_from(src) == src.get_count()
    assert np.array_equal(a.get_trained_state(), b.get_trained_state())
    assert_same_index(a, b, queries(rng, src))
    assert_same_index(a, fresh_build(src, **kw), queries(rng, src))


# --------------------------------------------------------------------------------------------------------------- range edges

@pytest.mark.parametrize("kind", [IVF_FLAT, FLAT, HNSW])
def test_range_edges(kind):
    rng = np.random.default_rng(400 + kind)
    d = 16
    kw = dict(nlist=4) if kind == IVF_FLAT else dict(hnsw_m=8, hnsw_efc=40, max_elements=1000) if kind == HNSW else {}
    src = b200vs.Index(kind, L2, d, **kw)
    if kind == IVF_FLAT:
        src.train(rows(rng, 100, d))
    ids = np.array([3, 10, 11, 50, 99, 100, 400, I64_MAX], np.int64)
    src.add(rows(rng, ids.size, d), ids)

    def got(lo, hi):
        dst = b200vs.Index(kind, L2, d, **kw)
        n = dst.rebuild_from_range([src], lo, hi)
        live = sorted_live(dst)[1] if n else np.zeros(0, np.int64)
        assert n == live.size == dst.get_count()
        if n == 0 and kind == IVF_FLAT:
            assert not dst.is_trained()
        return live.tolist()

    assert got(10, 100) == [10, 11, 50, 99]  # id_min included, id_max excluded
    assert got(11, 11) == []  # id_min == id_max
    assert got(0, 0) == [] and got(-5, -5) == []
    assert got(12, 50) == []  # a range that holds no rows
    assert got(101, 400) == []
    assert got(0, I64_MAX) == [3, 10, 11, 50, 99, 100, 400]  # INT64_MAX is never inside [id_min, id_max)
    assert got(-(2 ** 63), I64_MAX) == [3, 10, 11, 50, 99, 100, 400]
    if kind != FLAT:  # b200vs_rebuild_from keeps every live row, INT64_MAX's too
        dst = b200vs.Index(kind, L2, d, **kw)
        assert dst.rebuild_from(src) == ids.size


# ------------------------------------------------------------------------------------------------------------------ refusals

def fingerprint(ix, q):
    fp = [ix.get_count(), ix.get_deleted_count(), ix.is_trained(), bytes(ix.get_trained_state())]
    if ix.get_count():
        if ix.type != IVF_PQ or ix.sub_type() == FLAT:  # IVF-PQ mode exports codes, not rows
            x, ids = sorted_live(ix)
            fp += [x.tobytes(), ids.tobytes()]
        D, I = ix.search(q, 10)
        fp += [D.tobytes(), I.tobytes()]
    return fp


def test_refusals_leave_everything_unchanged():
    rng = np.random.default_rng(17)
    d, nlist = 16, 4
    q = rows(rng, 8, d)

    def ivf(lo, n, train=True, **kw):
        ix = b200vs.Index(IVF_FLAT, L2, d, nlist=nlist, **kw)
        if train:
            ix.train(rows(rng, 200, d))
            ix.add(rows(rng, n, d), np.arange(lo, lo + n))
        return ix

    a, b = ivf(0, 500), ivf(500, 500)
    overlap = ivf(400, 200)  # shares ids 400 .. 499 with a

    def refused(dst, srcs, lo, hi, code):
        every = [dst] + [s for s in srcs if s is not None]
        before = [fingerprint(ix, q) for ix in every]
        with pytest.raises(b200vs.B200VSError) as e:
            dst.rebuild_from_range(srcs, lo, hi)
        assert e.value.code == code, e.value.msg
        assert [fingerprint(ix, q) for ix in every] == before

    fresh = lambda **kw: ivf(0, 0, train=False, **kw)  # noqa: E731
    refused(fresh(), [], 0, 10, EILLEGAL_PARAMETERS)
    many = [ivf(1000 * i + 10000, 2) for i in range(17)]
    refused(fresh(), many, 0, I64_MAX, EILLEGAL_PARAMETERS)
    assert fresh().rebuild_from_range(many[:16], 0, I64_MAX) == 32  # 16 sources are served
    refused(fresh(), [a, None], 0, 10, EILLEGAL_PARAMETERS)
    refused(fresh(), [a], 10, 9, EILLEGAL_PARAMETERS)
    refused(a, [a], 0, 10, EILLEGAL_PARAMETERS)
    refused(a, [b, a], 0, 10, EILLEGAL_PARAMETERS)
    refused(fresh(), [a, b, a], 0, 10, EILLEGAL_PARAMETERS)
    refused(b200vs.Index(IVF_FLAT, IP, d, nlist=nlist), [a, b], 0, 10, EILLEGAL_PARAMETERS)
    refused(b200vs.Index(IVF_FLAT, L2, d + 8, nlist=nlist), [a], 0, 10, EILLEGAL_PARAMETERS)
    refused(b200vs.Index(IVF_FLAT, L2, d, nlist=nlist + 1), [a, b], 0, 10, EILLEGAL_PARAMETERS)
    refused(b200vs.Index(FLAT, L2, d), [a], 0, 10, EILLEGAL_PARAMETERS)
    refused(ivf(5000, 10), [a], 0, 10, EILLEGAL_PARAMETERS)  # dst not empty
    trained = fresh()
    trained.train(rows(rng, 100, d))
    refused(trained, [a], 0, 10, EILLEGAL_PARAMETERS)
    refused(fresh(), [a, overlap], 0, 1000, EVECTOR_ID_DUPLICATED)
    refused(fresh(), [overlap, a], 450, 460, EVECTOR_ID_DUPLICATED)
    assert fresh().rebuild_from_range([a, overlap], 0, 400) == 400  # the shared ids lie outside this range
    assert fresh().rebuild_from_range([a, b], 0, 1000) == 1000
    # a null source list
    n = ctypes.c_int64(-1)
    dst = fresh()
    assert b200vs.lib().b200vs_rebuild_from_range(dst.h, 1, None, 0, 10, ctypes.byref(n)) == EILLEGAL_PARAMETERS and n.value == 0
    # IVF-PQ: a source in IVF-PQ mode keeps only codes
    pq_kw = dict(nlist=nlist, pq_m=4, pq_nbits=4)
    pq_flat = b200vs.Index(IVF_PQ, L2, d, **pq_kw)
    pq_flat.train(rows(rng, 10, d))
    pq_flat.add(rows(rng, 100, d), np.arange(100))
    pq_mode = b200vs.Index(IVF_PQ, L2, d, **pq_kw)
    pq_mode.train(rows(rng, 4096, d))
    pq_mode.add(rows(rng, 100, d), np.arange(100, 200))
    refused(b200vs.Index(IVF_PQ, L2, d, **pq_kw), [pq_flat, pq_mode], 0, 150, EVECTOR_NOT_SUPPORT)
    # HNSW: max_elements below |R| (R, not the sources' live rows, decides)
    hkw = dict(hnsw_m=8, hnsw_efc=40)
    h1, h2 = b200vs.Index(HNSW, L2, d, max_elements=1000, **hkw), b200vs.Index(HNSW, L2, d, max_elements=1000, **hkw)
    h1.add(rows(rng, 300, d), np.arange(300))
    h2.add(rows(rng, 300, d), np.arange(300, 600))
    refused(b200vs.Index(HNSW, L2, d, max_elements=399, **hkw), [h1, h2], 100, 500, EILLEGAL_PARAMETERS)
    assert b200vs.Index(HNSW, L2, d, max_elements=400, **hkw).rebuild_from_range([h1, h2], 100, 500) == 400
    h3 = b200vs.Index(HNSW, L2, d, max_elements=1000, **hkw)
    h3.add(rows(rng, 10, d), np.arange(295, 305))
    refused(b200vs.Index(HNSW, L2, d, max_elements=1000, **hkw), [h1, h3], 0, 1000, EVECTOR_ID_DUPLICATED)
    # Flat types are served here; b200vs_rebuild_from keeps refusing them
    fl = b200vs.Index(FLAT, L2, d)
    fl.add(rows(rng, 10, d), np.arange(10))
    assert b200vs.Index(FLAT, L2, d).rebuild_from_range([fl], 0, 5) == 5
    with pytest.raises(b200vs.B200VSError) as e:
        b200vs.Index(FLAT, L2, d).rebuild_from(fl)
    assert e.value.code == EVECTOR_NOT_SUPPORT


# --------------------------------------------------------------------------------------------------------------- concurrency

def same_rows(a, b):
    """a and b hold the same trained state and the same lists (ids and rows)."""
    if not np.array_equal(a.get_trained_state(), b.get_trained_state()) or a.get_count() != b.get_count():
        return False
    return all(np.array_equal(u, v) for u, v in zip(a.export_lists(nlist_of(a)), b.export_lists(nlist_of(b))))


def test_children_rebuild_at_once_while_the_source_serves():
    # Both children of a split are rebuilt from one source at once, while a third thread searches it and a writer adds one
    # row into each child's range.  A rebuild holds the source for its whole call, so each child either was copied before
    # the write (and then the write finished only after that rebuild ended) or began after the write had finished (and then
    # holds the new row).  The writer starts once both calls are under way, so normally it waits for both; a rebuild thread
    # that a loaded host starts late takes the second branch, which is still checked.
    rng = np.random.default_rng(16)
    d, nlist, n = 64, 512, 600000
    src = b200vs.Index(IVF_FLAT, L2, d, nlist=nlist)
    src.train(rows(rng, 20000, d))
    src.add(rows(rng, n, d), np.arange(n))
    s = n // 2
    ranges = ((0, s), (s, I64_MAX))

    def sequential():
        out = []
        for lo, hi in ranges:
            w = b200vs.Index(IVF_FLAT, L2, d, nlist=nlist)
            w.rebuild_from_range([src], lo, hi)
            out.append(w)
        return out

    pre = sequential()
    q = rows(rng, 16, d)
    stop, seen, spans = threading.Event(), [], []
    kids = [b200vs.Index(IVF_FLAT, L2, d, nlist=nlist) for _ in range(2)]
    ends, errors, wrote = [0.0, 0.0], [], [0.0]
    new_rows = rows(rng, 2, d)

    def reader():
        while not stop.is_set():
            t0 = time.perf_counter()
            D, I = src.search(q, 10, nprobe=8)
            spans.append((t0, time.perf_counter()))
            seen.append((D.tobytes(), I.tobytes()))

    def rebuild(i):
        try:
            kids[i].rebuild_from_range([src], *ranges[i])
        except Exception as e:  # noqa: BLE001
            errors.append(e)
        ends[i] = time.perf_counter()

    def writer():
        src.add(new_rows, [7, s + 7])  # one write with a row in each child's range
        wrote[0] = time.perf_counter()

    D0, I0 = src.search(q, 10, nprobe=8)
    rt = threading.Thread(target=reader)
    rt.start()
    try:
        r0 = time.perf_counter()
        ts = [threading.Thread(target=rebuild, args=(i,)) for i in range(2)]
        for t in ts:
            t.start()
        time.sleep(0.05)
        wt = threading.Thread(target=writer)
        wt.start()
        for t in ts:
            t.join()
        r1 = time.perf_counter()
        wt.join()
    finally:
        stop.set()
        rt.join()
    assert not errors, errors
    assert src.get_count() == n + 2
    post = sequential()
    D1, I1 = src.search(q, 10, nprobe=8)
    # every search saw the source either before or after the one write, never anything else
    allowed = {(D0.tobytes(), I0.tobytes()), (D1.tobytes(), I1.tobytes())}
    assert all(r in allowed for r in seen)
    assert [s_ for s_ in spans if s_[0] > r0 and s_[1] < r1], "no search ran while the rebuilds ran"
    for i in range(2):
        if same_rows(kids[i], pre[i]):
            assert wrote[0] >= ends[i], f"the write finished while rebuild {i} held the source"
            assert_same_index(kids[i], pre[i], q)
        else:
            assert ends[i] >= wrote[0], f"rebuild {i} holds the write, but ended before it"
            assert_same_index(kids[i], post[i], q)
