"""Deep top-k (b200vs_search_deep / b200vs_search_binary_deep, Index.search_deep): exact searches for k up to 40960.

Every supported type against the oracle bit for bit (ids and distance bits, -1 / 0 padding included), and against
b200vs_search bit for bit wherever that answers (k <= 4096, and k = 8192 on a small-d Flat); exact ties that cross the k-th
boundary, non-finite rows, every filter, tombstones and upserts, empty probed lists, query chunking, refusals and
concurrent readers."""
import os
import subprocess
import threading

import numpy as np
import pytest

import b200vs
import binary_oracle as bo
import pq_codes
from b200vs import BINARY_FLAT, BINARY_IVF_FLAT, COSINE, FLAT, HNSW, IP, IVF_FLAT, IVF_PQ, L2
from gpu_util import assert_same_results, require_gpu

pytestmark = pytest.mark.gpu

KS = (1, 129, 4096, 4097, 8193, 40960)


@pytest.fixture(autouse=True)
def _gpu():
    require_gpu()


def rows(n, d, seed):
    return np.random.default_rng(seed).standard_normal((n, d)).astype(np.float32)


def same_as_search(ix, xq, k, **kw):
    """deep == b200vs_search bit for bit, with and without exact_only"""
    for exact in (False, True):
        Ds, Is = ix.search(xq, k, exact_only=exact, **kw)
        Dd, Id = ix.search_deep(xq, k, exact_only=exact, **kw)
        assert_same_results(Dd, Id, Ds, Is)


@pytest.mark.parametrize("metric", [L2, IP, COSINE])
def test_flat_oracle(oracle, metric):
    n, d = 50000, 24
    xb, ids = rows(n, d, 1), np.random.default_rng(2).permutation(n).astype(np.int64) * 3 + 1
    xq = rows(3, d, 3)
    stored = oracle.normalize_faiss(xb) if metric == COSINE else xb  # the rows a cosine index stores
    ix = b200vs.Index(FLAT, metric, d)
    ix.add(xb, ids)
    for k in KS:
        Dd, Id = ix.search_deep(xq, k)
        Do, Io = oracle.flat_search(metric, stored, ids, xq, k, nthreads=8)
        assert_same_results(Dd, Id, Do, Io)
        st = ix.stats()
        assert st[0] > 0 and st[1] == 0
        if k <= 4096:
            same_as_search(ix, xq, k)


def test_flat_k8192_small_d_equals_search():
    xb = rows(30000, 8, 4)
    ix = b200vs.Index(FLAT, L2, 8)
    ix.add(xb, np.arange(30000, dtype=np.int64))
    same_as_search(ix, rows(2, 8, 5), 8192)


def ivf_flat(oracle, metric, n, d, nlist, seed):
    xb = rows(n, d, seed)
    stored = oracle.normalize_faiss(xb) if metric == COSINE else xb
    cent = stored[np.random.default_rng(seed).choice(n, nlist, replace=False)].copy()
    ix = b200vs.Index(IVF_FLAT, metric, d, nlist=nlist)
    ix.set_trained_state(b200vs.ivf_state_blob(cent, metric))
    ix.add(xb, np.arange(5, n + 5, dtype=np.int64))
    off, lx, _, lids = ix.export_lists(nlist)
    return ix, cent, off, lx, lids


@pytest.mark.parametrize("metric", [L2, IP, COSINE])
def test_ivf_flat_oracle(oracle, metric):
    nlist = 16
    ix, cent, off, lx, lids = ivf_flat(oracle, metric, 60000, 32, nlist, 10 + metric)
    xq = rows(3, 32, 11)
    for k in KS:
        for nprobe in (4, nlist):
            Dd, Id = ix.search_deep(xq, k, nprobe=nprobe)
            Do, Io = oracle.ivfflat_search(metric, cent, off, lx, lids, xq, k, nprobe, nthreads=8)
            assert_same_results(Dd, Id, Do, Io)
            if k <= 4096:
                same_as_search(ix, xq, k, nprobe=nprobe)


@pytest.mark.parametrize("metric", [L2, IP, COSINE])
@pytest.mark.parametrize("nbits", [8, 4])
def test_ivf_pq_oracle(oracle, metric, nbits):
    from test_gpu_ivf_pq_nbits import SynthN
    s = SynthN(oracle, metric, 20000, 64, 8, 16, nbits, seed=7 * nbits + metric)
    s.export()
    xq = rows(3, 64, 12)
    for k in KS:
        Dd, Id = s.ix.search_deep(xq, k, nprobe=5)
        Do, Io = pq_codes.ivfpq_search(oracle, metric, s.cent, s.cb, s.off, s.packed, s.lids, xq, k, 5, nthreads=8)
        assert_same_results(Dd, Id, Do, Io)
        if k <= 4096:
            same_as_search(s.ix, xq, k, nprobe=5)


@pytest.mark.parametrize("metric", [L2, IP, COSINE])
def test_ivf_pq_inner_flat(oracle, metric):
    # fewer than max(256 * nlist, 256 * 2^nbits) training rows: the index serves an inner Flat index
    xb = rows(3000, 32, 13)
    ix = b200vs.Index(IVF_PQ, metric, 32, nlist=16, pq_m=8, pq_nbits=8)
    ix.train(xb)
    ids = np.arange(3000, dtype=np.int64)
    ix.add(xb, ids)
    xq = rows(2, 32, 14)
    stored = oracle.normalize_faiss(xb) if metric == COSINE else xb
    for k in KS:
        Dd, Id = ix.search_deep(xq, k)
        Do, Io = oracle.flat_search(metric, stored, ids, xq, k, nthreads=8)
        assert_same_results(Dd, Id, Do, Io)
    same_as_search(ix, xq, 2000)


def test_binary_flat_oracle():
    rng = np.random.default_rng(20)
    n, dim = 30000, 256
    xb = rng.integers(0, 256, (n, dim // 8), dtype=np.uint8)
    ids = rng.permutation(n).astype(np.int64)
    xq = rng.integers(0, 256, (3, dim // 8), dtype=np.uint8)
    ix = b200vs.Index(BINARY_FLAT, b200vs.HAMMING, dim)
    ix.add(xb, ids)
    for k in KS:
        Dd, Id = ix.search_deep(xq, k)
        Do, Io = bo.flat_search(xb, ids, xq, k)
        assert_same_results(Dd, Id, Do, Io)
        if k <= 4096:
            same_as_search(ix, xq, k)


def test_binary_ivf_oracle():
    rng = np.random.default_rng(21)
    n, dim, nlist = 30000, 128, 8
    xb = rng.integers(0, 256, (n, dim // 8), dtype=np.uint8)
    cent = xb[rng.choice(n, nlist, replace=False)].copy()
    ix = b200vs.Index(BINARY_IVF_FLAT, b200vs.HAMMING, dim, nlist=nlist)
    ix.set_trained_state(b200vs.binary_ivf_state_blob(cent))
    ix.add(xb, np.arange(n, dtype=np.int64))
    off, _, codes, lids = ix.export_lists(nlist)
    xq = rng.integers(0, 256, (3, dim // 8), dtype=np.uint8)
    for k in KS:
        Dd, Id = ix.search_deep(xq, k, nprobe=3)
        Do, Io = bo.ivf_search(cent, off, codes, lids, xq, k, 3)
        assert_same_results(Dd, Id, Do, Io)
        if k <= 4096:
            same_as_search(ix, xq, k, nprobe=3)


def test_fewer_rows_than_k_pads(oracle):
    xb = rows(5000, 16, 30)
    ids = np.arange(100, 5100, dtype=np.int64)
    ix = b200vs.Index(FLAT, L2, 16)
    ix.add(xb, ids)
    xq = rows(2, 16, 31)
    Dd, Id = ix.search_deep(xq, 40960)
    assert (Id[:, 5000:] == -1).all() and (Dd[:, 5000:] == 0).all()
    Do, Io = oracle.flat_search(L2, xb, ids, xq, 40960, nthreads=8)
    assert_same_results(Dd, Id, Do, Io)


@pytest.mark.parametrize("metric", [L2, IP])
def test_exact_ties_take_smallest_ids(oracle, metric):
    # 6000 identical rows under shuffled ids among distinct ones: every key digit ties, the k-th boundary falls inside the
    # tie, so the id select decides which of them survive
    rng = np.random.default_rng(40)
    d = 16
    near = rows(1000, d, 41) * 0.01
    same = np.tile(rows(1, d, 42), (6000, 1))
    far = rows(3000, d, 43) * 100
    xb = np.concatenate([near, same, far])
    ids = rng.permutation(10000).astype(np.int64) * 7
    xq = np.zeros((2, d), np.float32)
    ix = b200vs.Index(FLAT, metric, d)
    ix.add(xb, ids)
    for k in (4096, 5000, 8193):
        Dd, Id = ix.search_deep(xq[:1] if metric == IP else xq, k)
        Do, Io = oracle.flat_search(metric, xb, ids, xq[:1] if metric == IP else xq, k, nthreads=8)
        assert_same_results(Dd, Id, Do, Io)
    # the whole candidate set ties: the answer is the k smallest ids
    ix2 = b200vs.Index(FLAT, L2, d)
    ix2.add(same, ids[:6000])
    Dd, Id = ix2.search_deep(xq[:1], 4500)
    assert np.array_equal(Id[0], np.sort(ids[:6000])[:4500])
    same_as_search(ix2, xq[:1], 4096)


def test_non_finite_rows_match_search():
    rng = np.random.default_rng(50)
    d = 16
    xb = rng.standard_normal((6000, d)).astype(np.float32)
    xb[::7, 3] = np.inf
    xb[::11, 5] = np.nan
    xb[::13] *= np.float32(3e38)
    xb[::17, 0] = -np.inf
    xq = rng.standard_normal((3, d)).astype(np.float32)
    xq[1, 2] = 1e30
    for metric in (L2, IP):
        ix = b200vs.Index(FLAT, metric, d)
        ix.add(xb, np.arange(6000, dtype=np.int64))
        same_as_search(ix, xq, 4096)
        Dd, Id = ix.search_deep(xq, 6000)
        Ds, Is = ix.search(xq, 4096)
        assert_same_results(Dd[:, :4096], Id[:, :4096], Ds, Is)
        assert (Id >= 0).all()  # NaN distances are results too, as in the shared-memory select


def test_filters_tombstones_upserts(oracle):
    n, d = 40000, 16
    xb = rows(n, d, 60)
    ids = np.arange(n, dtype=np.int64)
    ix = b200vs.Index(FLAT, L2, d)
    ix.add(xb, ids)
    dead = ids[::5]
    ix.delete(dead)
    up = rows(2000, d, 61)
    up_ids = ids[1::9][:2000]
    ix.add(up, up_ids, upsert=True)
    live = np.ones(n, bool)
    live[dead] = False
    cur = xb.copy()
    cur[up_ids] = up
    live[up_ids] = True
    xl, il = cur[live], ids[live]
    xq = rows(3, d, 62)
    sorted_ids = np.arange(3, n, 3, dtype=np.int64)
    for filt in ({}, {"id_range": (1000, 30000)}, {"sorted_ids": sorted_ids}, {"sorted_ids": sorted_ids, "negate": True}):
        for k in (4096, 9000):
            Dd, Id = ix.search_deep(xq, k, **filt)
            Do, Io = oracle.flat_search(L2, xl, il, xq, k, nthreads=8, **filt)
            assert_same_results(Dd, Id, Do, Io)
            if k <= 4096:
                same_as_search(ix, xq, k, **filt)


def test_ivf_empty_lists_and_all_probes(oracle):
    # most lists empty: probes cover empty lists; nprobe = nlist covers every row
    d, nlist = 16, 64
    xb = rows(9000, d, 70)
    cent = np.concatenate([xb[:8], rows(nlist - 8, d, 71) * 1000])
    ix = b200vs.Index(IVF_FLAT, L2, d, nlist=nlist)
    ix.set_trained_state(b200vs.ivf_state_blob(cent, L2))
    ix.add(xb, np.arange(9000, dtype=np.int64))
    off, lx, _, lids = ix.export_lists(nlist)
    assert (np.diff(off) == 0).sum() >= nlist - 8
    xq = rows(2, d, 72) * 1000
    for nprobe in (20, nlist):
        for k in (4096, 8192, 40960):
            Dd, Id = ix.search_deep(xq, k, nprobe=nprobe)
            Do, Io = oracle.ivfflat_search(L2, cent, off, lx, lids, xq, k, nprobe, nthreads=8)
            assert_same_results(Dd, Id, Do, Io)


def test_query_chunks_match_single_queries():
    # 64 queries x 4M candidates x 5 B of keys and eligibility is ~1.3 GB: more than one query chunk
    n, d = 4_000_000, 8
    xb = rows(n, d, 80)
    ix = b200vs.Index(FLAT, L2, d)
    ix.add(xb, np.arange(n, dtype=np.int64))
    xq = rows(64, d, 81)
    D, I = ix.search_deep(xq, 40960)
    for i in range(0, 64, 9):
        D1, I1 = ix.search_deep(xq[i:i + 1], 40960)
        assert_same_results(D[i:i + 1], I[i:i + 1], D1, I1)
    assert np.all(np.diff(D, axis=1) >= 0)


def test_refusals_leave_the_index_answering():
    xb = rows(3000, 16, 90)
    ix = b200vs.Index(FLAT, L2, 16)
    ix.add(xb, np.arange(3000, dtype=np.int64))
    xq = rows(1, 16, 91)
    ref = ix.search_deep(xq, 100)
    with pytest.raises(b200vs.B200VSError) as e:
        ix.search_deep(xq, 40961)
    assert e.value.code == b200vs.EILLEGAL_PARAMETERS
    od, oi = np.zeros(10, np.float32), np.zeros(10, np.int64)
    rc = ix.L.b200vs_search_binary_deep(ix.h, 1, np.zeros(2, np.uint8).ctypes.data, 10, None, od.ctypes.data, oi.ctypes.data)
    assert rc == b200vs.EILLEGAL_PARAMETERS  # a binary call on a float index
    D0, I0 = ix.search_deep(xq, 0)
    assert D0.shape == (1, 0)
    assert_same_results(*ix.search_deep(xq, 100), *ref)
    hn = b200vs.Index(HNSW, L2, 16, hnsw_m=16, hnsw_efc=64, max_elements=4000)
    hn.add(xb, np.arange(3000, dtype=np.int64))
    with pytest.raises(b200vs.B200VSError) as e:
        hn.search_deep(xq, 5000)
    assert e.value.code == b200vs.EVECTOR_NOT_SUPPORT
    D, I = hn.search(xq, 10)
    assert (I >= 0).all()


def test_concurrent_deep_and_ordinary_searches():
    n, d = 60000, 16
    ix = b200vs.Index(FLAT, L2, d)
    ix.add(rows(n, d, 100), np.arange(n, dtype=np.int64))
    qs = [rows(2, d, 101 + t) for t in range(6)]
    want = [(ix.search_deep(q, 8193), ix.search(q, 100)) for q in qs]
    errs = []

    def work(t):
        try:
            for _ in range(3):
                Dd, Id = ix.search_deep(qs[t], 8193)
                Ds, Is = ix.search(qs[t], 100)
                assert_same_results(Dd, Id, *want[t][0])
                assert_same_results(Ds, Is, *want[t][1])
        except Exception as ex:  # noqa: BLE001 - collected and re-raised on the main thread
            errs.append(ex)

    th = [threading.Thread(target=work, args=(t,)) for t in range(6)]
    for t in th:
        t.start()
    for t in th:
        t.join()
    assert not errs, errs[0]


def test_binary_query_chunks_match_single_queries():
    # 64 queries x 4M candidates x 5 B is ~1.3 GB of keys and eligibility: more than one query chunk on Hamming rows
    rng = np.random.default_rng(110)
    n, dim = 4_000_000, 64
    xb = rng.integers(0, 256, (n, dim // 8), dtype=np.uint8)
    ix = b200vs.Index(BINARY_FLAT, b200vs.HAMMING, dim)
    ix.add(xb, np.arange(n, dtype=np.int64))
    xq = rng.integers(0, 256, (64, dim // 8), dtype=np.uint8)
    D, I = ix.search_deep(xq, 40960)
    for i in (0, 31, 63):
        D1, I1 = ix.search_deep(xq[i:i + 1], 40960)
        assert_same_results(D[i:i + 1], I[i:i + 1], D1, I1)


@pytest.mark.parametrize("metric", [L2, IP, COSINE])
def test_bruteforce_scan_deep_k(metric):
    # k = 40960 is past the exact scan's shared-memory select: every tile's top-k and the running merge take the deep path.
    # Uneven tiles must give one deep Flat search over their concatenation.
    d, k = 16, 40960
    sizes = [30000, 1, 52345, 7000, 41000]
    xb = rows(sum(sizes), d, 120)
    ids = np.random.default_rng(121).permutation(len(xb)).astype(np.int64) * 5 + 2
    xq = rows(3, d, 122)
    sc = b200vs.BruteForceScan(metric, d, xq, k)
    o = 0
    for m in sizes:
        sc.push(xb[o:o + m], ids[o:o + m])
        o += m
    Ds, Is = sc.finish()
    ix = b200vs.Index(FLAT, metric, d)
    ix.add(xb, ids)
    Dd, Id = ix.search_deep(xq, k)
    if metric == L2:
        assert_same_results(Ds, Is, Dd, Id)
    else:
        # the running merge ranks API distances 1 - ip, ties to the smaller id (the reference's priority queues), while one
        # index ranks ip itself: two ips may round to one 1 - ip, so equal distances may come in another id order, and a
        # tie at the k-th distance may keep other ids.  Distances are equal bit for bit, ids below the last distance too.
        assert np.array_equal(Ds.view(np.uint32), Dd.view(np.uint32))
        for q in range(len(xq)):
            below = Dd[q] < Dd[q, -1]
            assert set(Is[q][below].tolist()) == set(Id[q][below].tolist())
    # below the select's limit the scan keeps its kernels and equals b200vs_search
    sc = b200vs.BruteForceScan(metric, d, xq, 500)
    o = 0
    for m in sizes:
        sc.push(xb[o:o + m], ids[o:o + m])
        o += m
    assert_same_results(*sc.finish(), *ix.search(xq, 500))


def test_cpp_plugin_routes_deep_topk():
    exe = os.path.join(b200vs.PKG_ROOT, "host", "test_plugin_deep")
    assert os.path.exists(exe), "build it with: make -C dingo-store_b200/host"
    r = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    print(r.stdout[-3000:])
    assert r.returncode == 0 and "PLUGIN DEEP TESTS OK" in r.stdout, r.stdout[-3000:] + r.stderr[-1000:]
