"""Streaming brute-force range scan (b200vs_scan_range_*), the GPU counterpart of VectorReader::BruteForceRangeSearch
(src/vector/vector_reader.cc:2050-2202).  Per query the result is the first max_results hits in scan order (tiles in push
order, rows in order within a tile), a hit being a row with id >= 0 that passes the filters and whose FP32 value is
strictly inside the radius (L2: dist < radius; IP / cosine: ip > 1 - radius).  Every case compares ids, counts, padding
and distance bits with a numpy restatement of that rule built on raw_fp32 / api_of, whose summation order is the
kernel's; cosine rows and queries go through the oracle's NormalizeVectorForFaiss first."""
import ctypes

import numpy as np
import pytest

import b200vs
import oracle_lib
from b200vs import COSINE, IP, L2
from gpu_util import require_gpu
from test_gpu_exact_edges import api_of, raw_fp32

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _gpu():
    require_gpu()


def prep(metric, x):
    x = np.ascontiguousarray(x, np.float32)
    return oracle_lib.load().normalize_faiss(x) if metric == COSINE else x


def raw_matrix(X, Q, metric):
    """raw_fp32 of every (query, row) pair: [nq, n]."""
    n, d = X.shape
    out = np.empty((len(Q), n), np.float32)
    step = max(1, (1 << 23) // max(1, n * d))
    for a in range(0, len(Q), step):
        q = Q[a:a + step]
        out[a:a + len(q)] = raw_fp32(np.tile(X, (len(q), 1)), np.repeat(q, n, axis=0), metric).reshape(len(q), n)
    return out


def cand_mask(ids, id_range=None, sorted_ids=None, negate=False):
    m = ids >= 0
    if id_range is not None:
        m &= (ids >= id_range[0]) & (ids < id_range[1])
    if sorted_ids is not None:
        m &= np.isin(ids, sorted_ids) != negate
    return m


def restate(metric, xq, tiles, radius, max_results, **filters):
    """The rule, tile by tile: (D, I, C) as scan_range_finish returns them."""
    Q = prep(metric, xq)
    nq = len(Q)
    thr = np.float32(radius) if metric == L2 else np.float32(1) - np.float32(radius)
    D = np.zeros((nq, max_results), np.float32)
    I = np.full((nq, max_results), -1, np.int64)
    C = np.zeros(nq, np.int32)
    for x, ids in tiles:
        if len(ids) == 0:
            continue
        raw = raw_matrix(prep(metric, x), Q, metric)
        hit = (raw < thr if metric == L2 else raw > thr) & cand_mask(ids, **filters)[None, :]
        for q in range(nq):
            room = max_results - C[q]
            if room <= 0:
                continue
            r = np.flatnonzero(hit[q])[:room]
            D[q, C[q]:C[q] + len(r)] = api_of(raw[q, r], metric)
            I[q, C[q]:C[q] + len(r)] = ids[r]
            C[q] += len(r)
    return D, I, C


def run(metric, d, xq, tiles, radius, max_results, **filters):
    sc = b200vs.BruteForceRangeScan(metric, d, xq, radius, max_results, **filters)
    for x, ids in tiles:
        sc.push(x, ids)
    return sc.finish()


def check(metric, d, xq, tiles, radius, max_results, **filters):
    gd, gi, gc = run(metric, d, xq, tiles, radius, max_results, **filters)
    wd, wi, wc = restate(metric, xq, tiles, radius, max_results, **filters)
    assert np.array_equal(gc, wc), f"counts differ at queries {np.flatnonzero(gc != wc)[:5]}"
    assert np.array_equal(gi, wi), f"ids differ at {np.argwhere(gi != wi)[:5].tolist()}"
    assert np.array_equal(gd.view(np.uint32), wd.view(np.uint32)), "distance bits differ"
    return gd, gi, gc


def make_tiles(rng, sizes, d, id0=1):
    n = sum(sizes)
    xb = rng.random((n, d), dtype=np.float32)
    ids = rng.permutation(n).astype(np.int64) + id0
    tiles, a = [], 0
    for t in sizes:
        tiles.append((xb[a:a + t], ids[a:a + t]))
        a += t
    return tiles


def radius_for(metric, xq, tiles, frac):
    """A radius that keeps about `frac` of the rows for query 0."""
    X = np.concatenate([t[0] for t in tiles])
    raw = np.sort(raw_matrix(prep(metric, X), prep(metric, xq[:1]), metric)[0])
    i = int(frac * len(raw))
    return float(raw[i]) if metric == L2 else float(np.float32(1) - raw[len(raw) - 1 - i])


SIZES = {"2048-2048-777": [2048, 2048, 777], "5-1-300": [5, 1, 300], "4096": [4096], "200-ones": [1] * 200,
         "empty-in-middle": [700, 0, 600]}


@pytest.mark.parametrize("metric", [L2, IP, COSINE])
@pytest.mark.parametrize("d", [96, 13, 768])
def test_metrics_and_dims(metric, d):
    rng = np.random.default_rng(d * 10 + metric)
    xq = rng.random((9, d), dtype=np.float32)
    tiles = make_tiles(rng, SIZES["2048-2048-777"], d)
    _, _, gc = check(metric, d, xq, tiles, radius_for(metric, xq, tiles, 0.02), 1024)
    assert gc[0] > 0


@pytest.mark.parametrize("metric", [L2, IP, COSINE])
@pytest.mark.parametrize("layout", list(SIZES))
def test_tile_layouts(metric, layout):
    d = 96
    rng = np.random.default_rng(len(layout) + metric)
    xq = rng.random((6, d), dtype=np.float32)
    tiles = make_tiles(rng, SIZES[layout], d)
    _, _, gc = check(metric, d, xq, tiles, radius_for(metric, xq, tiles, 0.1), 1024)
    assert gc.max() > 0


@pytest.mark.parametrize("metric", [L2, IP])
@pytest.mark.parametrize("max_results", [1, 7, 1024, 100000])
def test_max_results(metric, max_results):
    d = 32
    rng = np.random.default_rng(max_results + metric)
    xq = rng.random((5, d), dtype=np.float32)
    tiles = make_tiles(rng, [2048, 2048, 777], d)
    _, _, gc = check(metric, d, xq, tiles, radius_for(metric, xq, tiles, 0.3), max_results)
    if max_results <= 1024:
        assert gc[0] == max_results  # query 0 has ~30 % of 4873 rows as hits: the cap is reached
    else:
        assert (gc < max_results).all() and gc[0] > 1024


@pytest.mark.parametrize("cap", [10, 15])
def test_cap_mid_tile_and_at_boundary(cap):
    """Every row is a hit: cap 10 fills exactly at the end of the first tile, cap 15 inside the second; later pushes add
    nothing."""
    d = 24
    rng = np.random.default_rng(cap)
    xq = rng.random((3, d), dtype=np.float32)
    tiles = make_tiles(rng, [10, 10, 10, 10], d)
    gd, gi, gc = check(L2, d, xq, tiles, 1e30, cap)
    assert (gc == cap).all()
    expect = np.concatenate([t[1] for t in tiles])[:cap]
    assert (gi == expect[None, :]).all()


@pytest.mark.parametrize("metric", [L2, IP])
def test_threshold_is_strict(metric):
    """A row whose raw value equals the threshold is not a hit; one just inside it is."""
    d = 16
    q = np.zeros((1, d), np.float32)
    x = np.zeros((4, d), np.float32)
    if metric == L2:  # q = 0: dist = x0^2 exactly; radius 0.25
        x[:, 0] = [0.5, np.nextafter(np.float32(0.5), np.float32(0)), 0.75, 0.25]
        radius = 0.25
    else:             # q = e0: ip = x0 exactly; radius 0.5 -> threshold 1 - 0.5 = 0.5
        q[0, 0] = 1.0
        x[:, 0] = [0.5, np.nextafter(np.float32(0.5), np.float32(1)), 0.25, 0.75]
        radius = 0.5
    ids = np.array([11, 12, 13, 14], np.int64)
    gd, gi, gc = check(metric, d, q, [(x, ids)], radius, 8)
    assert 11 not in gi[0] and 12 in gi[0]


def test_filters():
    d = 40
    rng = np.random.default_rng(7)
    xq = rng.random((8, d), dtype=np.float32)
    tiles = make_tiles(rng, [2048, 2048, 777], d)
    radius = radius_for(L2, xq, tiles, 0.2)
    allow = np.sort(rng.choice(np.arange(1, 4874), 1500, replace=False)).astype(np.int64)
    for kw in ({"id_range": (500, 3000)}, {"sorted_ids": allow}, {"sorted_ids": allow, "negate": True},
               {"id_range": (500, 3000), "sorted_ids": allow, "negate": True}, {"id_range": (500, 3000), "sorted_ids": allow}):
        _, _, gc = check(L2, d, xq, tiles, radius, 1024, **kw)
        assert gc.max() > 0, kw


def test_negative_ids_are_never_hits():
    d = 20
    rng = np.random.default_rng(8)
    xq = rng.random((4, d), dtype=np.float32)
    tiles = make_tiles(rng, [300, 300], d)
    for x, ids in tiles:
        ids[::3] = -ids[::3]
    gd, gi, gc = check(L2, d, xq, tiles, 1e30, 1024)
    assert (gc == 400).all() and not (gi[:, :400] < 0).any()


def test_duplicate_id_in_one_push():
    d = 20
    rng = np.random.default_rng(9)
    xq = rng.random((4, d), dtype=np.float32)
    tiles = make_tiles(rng, [100, 50, 100], d)
    radius = radius_for(IP, xq, tiles, 0.3)
    dup_x, dup_ids = tiles[1][0], tiles[1][1].copy()
    dup_ids[7] = dup_ids[3]
    sc = b200vs.BruteForceRangeScan(IP, d, xq, radius, 64)
    sc.push(*tiles[0])
    with pytest.raises(b200vs.B200VSError) as e:
        sc.push(dup_x, dup_ids)
    assert e.value.code == b200vs.EVECTOR_ID_DUPLICATED
    sc.push(*tiles[2])
    gd, gi, gc = sc.finish()
    wd, wi, wc = restate(IP, xq, [tiles[0], tiles[2]], radius, 64)
    assert np.array_equal(gc, wc) and np.array_equal(gi, wi) and np.array_equal(gd.view(np.uint32), wd.view(np.uint32))


@pytest.mark.parametrize("nq", [1, 70000])
def test_query_counts(nq):
    """nq = 70000 is past the 65535 limit of a grid's y dimension: one CTA per query in grid.x."""
    d = 8
    rng = np.random.default_rng(nq)
    xq = rng.random((nq, d), dtype=np.float32)
    tiles = make_tiles(rng, [30, 20], d)
    _, _, gc = check(L2, d, xq, tiles, 0.6, 1)
    assert gc.sum() > nq // 2


def test_finish_without_push():
    xq = np.random.default_rng(0).random((3, 16), dtype=np.float32)
    sc = b200vs.BruteForceRangeScan(L2, 16, xq, 1.0, 5)
    gd, gi, gc = sc.finish()
    assert (gc == 0).all() and (gi == -1).all() and (gd == 0).all()
    sc = b200vs.BruteForceRangeScan(L2, 16, xq, 1.0, 5)
    sc.push(np.zeros((0, 16), np.float32), np.zeros(0, np.int64))  # n = 0: a no-op
    gd, gi, gc = sc.finish()
    assert (gc == 0).all() and (gi == -1).all()


def test_error_statuses():
    xq = np.random.default_rng(0).random((2, 8), dtype=np.float32)

    def code(fn):
        with pytest.raises(b200vs.B200VSError) as e:
            fn()
        return e.value.code

    assert code(lambda: b200vs.BruteForceRangeScan(L2, 0, xq, 1.0)) == b200vs.EVECTOR_INVALID
    assert code(lambda: b200vs.BruteForceRangeScan(b200vs.HAMMING, 8, xq, 1.0)) == b200vs.EVECTOR_NOT_SUPPORT
    assert code(lambda: b200vs.BruteForceRangeScan(7, 8, xq, 1.0)) == b200vs.EILLEGAL_PARAMETERS
    assert code(lambda: b200vs.BruteForceRangeScan(L2, 8, np.zeros((0, 8), np.float32), 1.0)) == b200vs.EILLEGAL_PARAMETERS
    assert code(lambda: b200vs.BruteForceRangeScan(L2, 8, xq, 1.0, max_results=0)) == b200vs.EILLEGAL_PARAMETERS
    L = b200vs.lib()
    sp = b200vs.SearchParams()
    assert L.b200vs_scan_range_begin(0, L2, 8, 2, xq.ctypes.data, 1.0, 4, ctypes.byref(sp), None) == b200vs.EILLEGAL_PARAMETERS
    sc = b200vs.BruteForceRangeScan(L2, 8, xq, 1.0, 4)
    ids = np.arange(3, dtype=np.int64)
    assert L.b200vs_scan_range_push(sc.h, 3, None, ids.ctypes.data) == b200vs.EILLEGAL_PARAMETERS
    assert L.b200vs_scan_range_push(sc.h, 3, xq.ctypes.data, None) == b200vs.EILLEGAL_PARAMETERS
    assert L.b200vs_scan_range_push(sc.h, -1, None, None) == b200vs.OK
    h, sc.h = sc.h, None
    assert L.b200vs_scan_range_finish(h, None, None, None) == b200vs.EILLEGAL_PARAMETERS  # and the handle is freed
    assert L.b200vs_scan_range_push(None, 1, xq.ctypes.data, ids.ctypes.data) == b200vs.EILLEGAL_PARAMETERS


@pytest.mark.parametrize("metric", [L2, IP, COSINE])
def test_same_hits_as_flat_range_search(metric):
    """With the cap not reached, each query's (id, distance bits) set equals b200vs_range_search on a Flat index holding
    the concatenation of the tiles."""
    d = 64
    rng = np.random.default_rng(40 + metric)
    xq = rng.random((12, d), dtype=np.float32)
    tiles = make_tiles(rng, [2048, 2048, 777], d)
    radius = radius_for(metric, xq, tiles, 0.03)
    cap = sum(len(t[1]) for t in tiles)  # never reached: the Flat search keeps the closest hits, the scan the first
    gd, gi, gc = run(metric, d, xq, tiles, radius, cap)
    ix = b200vs.Index(b200vs.FLAT, metric, d)
    ix.add(np.concatenate([t[0] for t in tiles]), np.concatenate([t[1] for t in tiles]))
    fd, fi, fc = ix.range_search(xq, radius, cap)
    assert np.array_equal(gc, fc) and gc[0] > 0
    for q in range(len(xq)):
        a = set(zip(gi[q, :gc[q]].tolist(), gd[q, :gc[q]].view(np.uint32).tolist()))
        b = set(zip(fi[q, :fc[q]].tolist(), fd[q, :fc[q]].view(np.uint32).tolist()))
        assert a == b, f"query {q}"
