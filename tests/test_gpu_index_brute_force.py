"""Brute-force search over an index's own device rows (b200vs_brute_force_search / b200vs_brute_force_range_search): the
answer of b200vs_scan_* / b200vs_scan_range_* fed the index's live rows in ascending id order, without the RocksDB scan.

The expected answer comes from BruteForceScan / BruteForceRangeScan fed a host model of the live rows (the raw rows as
added, after adds, deletes and upserts) in ascending id order and a random chunking, with rows sharing an id (IVF-Flat
adds without upsert) in separate chunks.  Ids, distance bits and counts must be equal.

Under IP / COSINE the chunked scan carries one ambiguity of its own: where 1 - ip rounds two different ip values to one
distance at the k-th slot, a chunking that splits the two rows keeps the smaller id, one chunk the larger ip.  The chunked
comparisons under IP / COSINE therefore use rows on a grid where every ip and 1 - ip is exact (ties then fall to the id on
both sides); random rows under IP / COSINE are compared with the scan fed the same rows as one chunk."""
import numpy as np
import pytest

import b200vs
from b200vs import COSINE, FLAT, HNSW, IP, IVF_FLAT, IVF_PQ, L2, BINARY_FLAT, BINARY_IVF_FLAT
from gpu_util import require_gpu

pytestmark = pytest.mark.gpu

D = 64


@pytest.fixture(autouse=True)
def _gpu():
    require_gpu()


def make_rows(rng, n, metric, grid):
    if not grid:
        return rng.standard_normal((n, D)).astype(np.float32)
    if metric == IP:  # integers in [-4, 4] * 2^-6: every ip is a multiple of 2^-12 with |ip| <= 1/4, so 1 - ip is exact
        return (rng.integers(-4, 5, (n, D)) * 2.0 ** -6).astype(np.float32)
    # COSINE: 16 entries of +-1/4, norm exactly 1 (not normalised again), every ip a multiple of 1/16
    x = np.zeros((n, D), np.float32)
    for i in range(n):
        x[i, rng.choice(D, 16, replace=False)] = rng.choice([-0.25, 0.25], 16)
    return x


class Model:
    """The live rows as (id, row) entries in the order an index stores rows sharing an id."""

    def __init__(self):
        self.entries = []

    def add(self, ids, x, replace):
        if replace:
            self.delete(ids)
        self.entries += list(zip(ids.tolist(), list(x)))

    def delete(self, ids):
        s = set(ids.tolist())
        self.entries = [e for e in self.entries if e[0] not in s]

    def sorted(self):
        order = sorted(range(len(self.entries)), key=lambda i: self.entries[i][0])  # stable: equal ids keep storage order
        ids = np.array([self.entries[i][0] for i in order], np.int64)
        x = np.array([self.entries[i][1] for i in order], np.float32).reshape(-1, D)
        return ids, x

    def chunks(self, rng, one=False):
        ids, x = self.sorted()
        n = len(ids)
        cuts = set() if one else set(rng.choice(np.arange(1, max(n, 2)), size=min(6, max(n - 1, 0)), replace=False).tolist())
        cuts |= {i for i in range(1, n) if ids[i] == ids[i - 1]}  # a tile never repeats an id
        b = [0] + sorted(cuts) + [n]
        return [(x[b[i]:b[i + 1]], ids[b[i]:b[i + 1]]) for i in range(len(b) - 1) if b[i + 1] > b[i]]


def build(itype, metric, rng, n, grid):
    """An index after adds, deletes and upserts (IVF-Flat: tombstones, list compaction, a repeated id), and its model."""
    m = Model()
    if itype == HNSW:
        ix = b200vs.Index(HNSW, metric, D, hnsw_m=16, hnsw_efc=64, max_elements=4 * n)
    elif itype == IVF_FLAT:
        ix = b200vs.Index(IVF_FLAT, metric, D, nlist=32)
        ix.train(make_rows(rng, 4096, metric, grid))
    else:
        ix = b200vs.Index(FLAT, metric, D)
    ids = rng.permutation(np.arange(10, 10 + 2 * n, 2, dtype=np.int64))
    x = make_rows(rng, n, metric, grid)
    if itype == HNSW:
        ix.add_batched(x, ids)
    else:
        ix.add(x, ids)
    m.add(ids, x, True)
    dead = rng.choice(ids, n // 3, replace=False)
    ix.delete(dead)
    m.delete(dead)
    up = rng.choice(ids, n // 10, replace=False)
    xu = make_rows(rng, len(up), metric, grid)
    if itype == HNSW:
        ix.add_batched(xu, up)  # Add == Upsert on HNSW
    else:
        ix.upsert(xu, up)
    m.add(up, xu, True)
    new = np.arange(3, 3 + 2 * (n // 20), 2, dtype=np.int64)
    xn = make_rows(rng, len(new), metric, grid)
    if itype == HNSW:
        ix.add_batched(xn, new)
    else:
        ix.add(xn, new)
    m.add(new, xn, True)
    if itype == IVF_FLAT:  # an add without upsert keeps the old row beside the new one; the same row lands in the same list
        again = new[:5]
        xa = xn[:5].copy()
        ix.add(xa, again)
        m.add(again, xa, False)
    return ix, m


def scan_topk(metric, m, xq, k, rng, one=False, **filt):
    sc = b200vs.BruteForceScan(metric, D, xq, k, **filt)
    for x, ids in m.chunks(rng, one):
        sc.push(x, ids)
    return sc.finish()


def scan_range(metric, m, xq, radius, max_results, rng, **filt):
    sc = b200vs.BruteForceRangeScan(metric, D, xq, radius, max_results, **filt)
    for x, ids in m.chunks(rng):
        sc.push(x, ids)
    return sc.finish()


def same(a, b):
    assert np.array_equal(a[1], b[1]), f"ids differ at {np.argwhere(a[1] != b[1])[:5].tolist()}"
    assert np.array_equal(a[0].view(np.uint32), b[0].view(np.uint32)), "distance bits differ"
    if len(a) > 2:
        assert np.array_equal(a[2], b[2]), "counts differ"


CASES = [(FLAT, L2), (FLAT, IP), (FLAT, COSINE), (IVF_FLAT, L2), (IVF_FLAT, IP), (IVF_FLAT, COSINE), (HNSW, L2), (HNSW, IP)]
IDS = [f"{['flat', 'ivf', 'pq', 'hnsw'][t]}-{['', 'l2', 'ip', 'cos'][m]}" for t, m in CASES]


@pytest.fixture(scope="module", params=CASES, ids=IDS)
def built(request):
    require_gpu()  # a module fixture is set up before the autouse one
    itype, metric = request.param
    rng = np.random.default_rng(100 + 10 * itype + metric)
    grid = metric != L2
    ix, m = build(itype, metric, rng, 48000, grid)
    return itype, metric, ix, m, grid, rng


@pytest.mark.parametrize("nq,k", [(1, 1), (8, 100), (64, 100), (1024, 10), (8, 4096), (4, 5000), (2, 40960)])
def test_topk_equals_chunked_scan(built, nq, k):
    itype, metric, ix, m, grid, rng = built
    xq = make_rows(rng, nq, metric, grid)
    got = ix.brute_force_search(xq, k, nprobe=3, efsearch=7)  # both ignored
    same(got, scan_topk(metric, m, xq, k, rng))
    assert (got[1] >= 0).sum() == nq * min(k, len(m.entries))
    if k <= 100:
        same(ix.brute_force_search(xq, k, exact_only=True), got)


@pytest.mark.parametrize("max_results", [10, 8192])
@pytest.mark.parametrize("nq", [1, 64, 1024])
def test_range_equals_chunked_scan(built, nq, max_results):
    itype, metric, ix, m, grid, rng = built
    xq = make_rows(rng, nq, metric, grid)
    ids, x = m.sorted()
    # a radius that admits a few hundred rows of the first query
    sample = x[rng.choice(len(x), 2000, replace=False)].astype(np.float64)
    q0 = xq[0].astype(np.float64)
    if metric == L2:
        dist = ((sample - q0) ** 2).sum(1)
    else:
        dist = 1 - sample @ (q0 / np.linalg.norm(q0) if metric == COSINE else q0)
    radius = float(np.quantile(dist, 0.01))
    got = ix.brute_force_range_search(xq, radius, max_results)
    same(got, scan_range(metric, m, xq, radius, max_results, rng))
    assert got[2].max() > 0
    if max_results == 10:
        assert got[2].max() == 10


@pytest.mark.parametrize("kind", ["range", "list", "negate"])
def test_filters(built, kind):
    itype, metric, ix, m, grid, rng = built
    xq = make_rows(rng, 32, metric, grid)
    ids, _ = m.sorted()
    if kind == "range":
        filt = dict(id_range=(int(ids[len(ids) // 4]), int(ids[3 * len(ids) // 4])))
    else:
        filt = dict(sorted_ids=np.unique(rng.choice(ids, 5000, replace=False)), negate=kind == "negate")
    for k in (10, 4096):
        same(ix.brute_force_search(xq, k, **filt), scan_topk(metric, m, xq, k, rng, **filt))
    radius = {L2: 90.0, IP: 0.98, COSINE: 0.8}[metric]  # a few percent of the rows
    got = ix.brute_force_range_search(xq, radius, 64, **filt)
    same(got, scan_range(metric, m, xq, radius, 64, rng, **filt))
    assert got[2].max() > 0


@pytest.mark.parametrize("itype,metric", [(FLAT, L2), (IVF_FLAT, IP), (HNSW, L2)], ids=["flat-l2", "ivf-ip", "hnsw-l2"])
def test_range_against_float64(itype, metric):
    """Every hit's distance is its float64 distance to FP32 accuracy, inside the radius; every row clearly inside the
    radius is a hit; hits come in ascending id order."""
    rng = np.random.default_rng(17 + itype)
    ix, m = build(itype, metric, rng, 8000, False)
    ids, x = m.sorted()
    xq = make_rows(rng, 16, metric, False)
    X, Q = x.astype(np.float64), xq.astype(np.float64)
    dist = ((X ** 2).sum(1)[None, :] + (Q ** 2).sum(1)[:, None] - 2 * Q @ X.T) if metric == L2 else 1 - Q @ X.T
    radius = float(np.quantile(dist, 0.01))
    Dg, Ig, Cg = ix.brute_force_range_search(xq, radius, len(ids))
    tol = 1e-5 * (np.abs(dist).max() + 1)
    for q in range(len(xq)):
        hits = Ig[q, :Cg[q]]
        assert (np.diff(hits) >= 0).all()  # an IVF-Flat id added twice comes twice
        pos = np.searchsorted(ids, hits)
        assert np.allclose(Dg[q, :Cg[q]], dist[q, pos], rtol=0, atol=tol)
        assert (dist[q, pos] < radius + tol).all()
        assert set(ids[dist[q] < radius - tol].tolist()) <= set(hits.tolist())
    assert Cg.sum() > 0  # one radius for every query: some queries hold no row inside it


@pytest.mark.parametrize("itype,metric", [(t, mt) for t, mt in CASES if mt != L2], ids=[i for (t, mt), i in zip(CASES, IDS) if mt != L2])
def test_random_rows_equal_one_chunk_scan(itype, metric):
    rng = np.random.default_rng(7 + itype + metric)
    ix, m = build(itype, metric, rng, 20000, False)
    for nq, k in [(8, 100), (64, 50), (4, 9000)]:
        xq = make_rows(rng, nq, metric, False)
        same(ix.brute_force_search(xq, k), scan_topk(metric, m, xq, k, rng, one=True))


def test_flat_l2_equals_oracle(oracle):
    rng = np.random.default_rng(3)
    ix, m = build(FLAT, L2, rng, 6000, False)
    ids, x = m.sorted()
    xq = make_rows(rng, 16, L2, False)
    Do, Io = oracle.flat_search(L2, x, ids, xq, 50, nthreads=8)
    same(ix.brute_force_search(xq, 50), (Do, Io))


def test_refusals_launch_nothing():
    rng = np.random.default_rng(5)
    x = rng.random((5000, D)).astype(np.float32)
    ids = np.arange(5000, dtype=np.int64)
    xq = x[:4]
    pq_flat = b200vs.Index(IVF_PQ, L2, D, nlist=4, pq_m=8, pq_nbits=4)
    pq_flat.train(x[:100])  # too few rows: the inner Flat index
    pq = b200vs.Index(IVF_PQ, L2, D, nlist=4, pq_m=8, pq_nbits=4)
    pq.train(x)
    assert pq_flat.L.b200vs_sub_type(pq_flat.h) == FLAT and pq.L.b200vs_sub_type(pq.h) == IVF_PQ
    hc = b200vs.Index(HNSW, COSINE, D, hnsw_m=8, hnsw_efc=32, max_elements=10000)
    float_ix = [pq_flat, pq, hc]
    for ix in float_ix:
        ix.add(x, ids)
    bx = rng.integers(0, 256, (5000, D // 8), dtype=np.uint8)
    bf = b200vs.Index(BINARY_FLAT, b200vs.HAMMING, D)
    bi = b200vs.Index(BINARY_IVF_FLAT, b200vs.HAMMING, D, nlist=4)
    bi.train(bx)
    for ix in (bf, bi):
        ix.add(bx, ids)
    for ix in float_ix + [bf, bi]:
        q = bx[:4] if ix in (bf, bi) else xq
        ix.search(q, 5)  # stats of an earlier read
        for call in (lambda: ix.brute_force_search(q, 10), lambda: ix.brute_force_range_search(q, 1.0, 10)):
            with pytest.raises(b200vs.B200VSError) as e:
                call()
            assert e.value.code == b200vs.EVECTOR_NOT_SUPPORT
            assert ix.stats()[0] == 0
        _, I = ix.search(q, 5)
        assert (I >= 0).all() and ix.get_count() == 5000


def test_edges():
    rng = np.random.default_rng(9)
    xq = rng.random((3, D)).astype(np.float32)
    for ix in (b200vs.Index(FLAT, L2, D), b200vs.Index(IVF_FLAT, IP, D, nlist=8), b200vs.Index(HNSW, L2, D, hnsw_m=8, hnsw_efc=32)):
        Dd, I = ix.brute_force_search(xq, 7)  # empty (or untrained): empty results
        assert (I == -1).all() and (Dd == 0).all()
        Dd, I, C = ix.brute_force_range_search(xq, 1e9, 7)
        assert (C == 0).all() and (I == -1).all()
        Dd, I = ix.brute_force_search(xq, 0)  # k <= 0: OK, nothing done
        assert I.shape == (3, 0)
        with pytest.raises(b200vs.B200VSError) as e:
            ix.brute_force_range_search(xq, 1.0, 0)
        assert e.value.code == b200vs.EILLEGAL_PARAMETERS
        with pytest.raises(b200vs.B200VSError) as e:
            ix.brute_force_search(xq, b200vs.DEEP_MAX_K + 1)
        assert e.value.code == b200vs.EILLEGAL_PARAMETERS
    fl = b200vs.Index(FLAT, L2, D)
    fl.add(rng.random((100, D)).astype(np.float32), np.arange(100, dtype=np.int64))
    Dd, I, C = fl.brute_force_range_search(xq, float("nan"), 5)
    assert (C == 0).all() and (I == -1).all() and fl.stats()[0] == 0
    Dd, I, C = fl.brute_force_range_search(xq, 1e9, 500)  # every row, in id order
    assert (C == 100).all() and (I[:, :100] == np.arange(100)).all()
