"""HNSW search at the edges of hnsw_search_kernel: tombstones (against the oracle with the same nodes filtered out), both
forms around the merged-array / candidate-heap switch, k > ef, odd dimensions (scalar distance tail), a candidate heap that
spills past its shared-memory part, and a filtered walk that floods a graph of 200k nodes.  Every search equals the oracle
bit for bit; returned distances are also checked against float64."""
import heapq

import numpy as np
import pytest

import b200vs
import oracle_lib
from b200vs import COSINE, HNSW, IP, L2
from gpu_util import assert_same_results, require_gpu

pytestmark = pytest.mark.gpu

HNSW_CAND_SMEM = 1024  # csrc/hnsw.cu: candidate-heap entries kept in shared memory; ef_run + 1 <= this runs the merged-array form
HNSW_CAND_POOL_BYTES = 512 << 20  # csrc/hnsw.cu: candidate-pool budget of one heap-form launch


@pytest.fixture(autouse=True)
def _gpu():
    require_gpu()


def pair(oracle, metric, n, d, M=16, efc=100, seed=0, data=None):
    """The same graph on both sides: single writer, same insertion order."""
    rng = np.random.default_rng(seed)
    xb = rng.random((n, d)).astype(np.float32) if data is None else data
    labels = np.arange(1000, 1000 + n, dtype=np.int64)
    ix = b200vs.Index(HNSW, metric, d, hnsw_m=M, hnsw_efc=efc, max_elements=n)
    ix.add(xb, labels)
    h = oracle_lib.OracleHnsw(oracle, metric, d, n, M, efc)
    h.add(xb, labels)
    assert np.array_equal(ix.get_trained_state(), h.export())
    return ix, h, xb, labels


def adopted(oracle, metric, n, d, M=16, efc=40, seed=0, threads=16):
    """A graph built by concurrent writers and adopted by the oracle (faster to build at large n)."""
    rng = np.random.default_rng(seed)
    xb = rng.random((n, d)).astype(np.float32)
    labels = np.arange(1, n + 1, dtype=np.int64)
    ix = b200vs.Index(HNSW, metric, d, hnsw_m=M, hnsw_efc=efc, max_elements=n, hnsw_build_threads=threads)
    ix.add(xb, labels)
    h = oracle_lib.OracleHnsw(oracle, metric, d, n, M, efc)
    h.load(ix.get_trained_state())
    return ix, h, xb, labels


def parse_graph(blob):
    """The HNSW state blob (DESIGN §5) -> (enterpoint, maxlevel, maxM, link0 [n, 2M+1], up_off, linkup, data, labels)."""
    b = np.ascontiguousarray(blob, dtype=np.uint8)
    hdr = b[:64].view(np.int64)
    n, d, M, maxM0, maxlevel, ep = (int(v) for v in hdr[1:7])
    pad8 = lambda v: (v + 7) // 8 * 8
    p = pad8(64 + 4 * n)
    up_off = b[p:p + 8 * (n + 1)].view(np.int64)
    p += 8 * (n + 1)
    link0 = b[p:p + 4 * n * (maxM0 + 1)].view(np.uint32).reshape(n, maxM0 + 1)
    p += 4 * n * (maxM0 + 1)
    linkup = b[p:p + 4 * int(up_off[n])].view(np.uint32)
    p = pad8(p + 4 * int(up_off[n]))
    data = b[p:p + 4 * n * d].view(np.float32).reshape(n, d)
    p = pad8(p + 4 * n * d)
    labels = b[p:p + 8 * n].view(np.int64)
    return ep, maxlevel, M, link0, up_off, linkup, data, labels


def flooded_walk(blob, q):
    """(peak, reached): the largest candidate-heap size of a base-layer walk in which no node ever enters the result set (a filter that passes
    fewer labels than ef): every fresh neighbour is pushed and the walk ends only when the heap is empty.  Float32 L2
    distances; the walk starts where the greedy descent of the upper layers ends, as the kernel's does.  `reached` marks
    the nodes the walk visits."""
    ep, maxlevel, M, link0, up_off, linkup, data, _ = parse_graph(blob)
    dist = ((data - q[None, :]) ** 2).sum(axis=1, dtype=np.float32)
    cur = ep
    for level in range(maxlevel, 0, -1):
        changed = True
        while changed:
            changed = False
            base = int(up_off[cur]) + (level - 1) * (M + 1)
            nb = linkup[base + 1:base + 1 + int(linkup[base])]
            for c in nb:
                if dist[c] < dist[cur]:
                    cur, changed = int(c), True
    vis = np.zeros(len(dist), bool)
    vis[cur] = True
    heap = [(float(dist[cur]), cur)]
    peak = 1
    while heap:
        _, c = heapq.heappop(heap)
        nb = link0[c, 1:1 + link0[c, 0]]
        nb = nb[~vis[nb]]
        vis[nb] = True
        for x in nb.tolist():
            heapq.heappush(heap, (float(dist[x]), x))
        peak = max(peak, len(heap))
    return peak, vis


def stored_rows(oracle, metric, xb):
    return oracle.normalize_hnsw(xb) if metric == COSINE else xb


def check_f64(oracle, metric, xb, labels, xq, D, I):
    """Every returned distance equals the float64 distance to the stored row within (d + 2) 2^-24 of the summed
    magnitudes; rows come back ascending by (distance, label)."""
    X = stored_rows(oracle, metric, xb).astype(np.float64)
    Q = stored_rows(oracle, metric, xq).astype(np.float64)
    pos = {int(l): i for i, l in enumerate(labels)}
    gamma = (xb.shape[1] + 2) * 2.0 ** -24
    for qi in range(len(xq)):
        valid = I[qi] >= 0
        assert valid.all() or not valid[np.argmin(valid):].any(), "-1 padding must come last"
        ids, ds = I[qi][valid], D[qi][valid].astype(np.float64)
        rows = X[[pos[int(i)] for i in ids]]
        if metric == L2:
            t = (rows - Q[qi]) ** 2
            want, S = t.sum(axis=1), t.sum(axis=1)
        else:
            t = rows * Q[qi]
            want, S = 1.0 - t.sum(axis=1), np.abs(t).sum(axis=1) + 1.0
        assert (np.abs(ds - want) <= gamma * S).all(), f"query {qi}: |gpu - f64| {np.abs(ds - want).max()} over the bound"
        key = list(zip(D[qi][valid].tolist(), ids.tolist()))
        assert key == sorted(key), f"query {qi}: not ascending by (distance, label)"


def brute_f64(oracle, metric, xb, labels, xq, k):
    X = stored_rows(oracle, metric, xb).astype(np.float64)
    Q = stored_rows(oracle, metric, xq).astype(np.float64)
    if metric == L2:
        dm = (Q * Q).sum(1)[:, None] - 2 * Q @ X.T + (X * X).sum(1)[None, :]
    else:
        dm = 1.0 - Q @ X.T
    return labels[np.argsort(dm, axis=1, kind="stable")[:, :k]]


@pytest.mark.parametrize("metric", [L2, IP, COSINE])
def test_tombstones_equal_oracle_with_negated_filter(oracle, metric):
    """hnswlib traverses a tombstoned node but never returns it, with the strict stop rule: exactly what an id filter does.
    So the engine after delete(dead) equals the oracle filtering the dead labels out."""
    n, d = 3000, 24
    ix, h, xb, labels = pair(oracle, metric, n, d, seed=metric)
    ep = int(ix.get_trained_state()[:64].view(np.int64)[6])
    rng = np.random.default_rng(5)
    dead = np.union1d(rng.choice(labels, 700, replace=False), labels[[ep]])  # the entry point is among the dead
    assert ix.delete(dead) == len(dead)
    xq = rng.random((32, d)).astype(np.float32)
    for k, ef in ((10, 64), (50, 0), (5, 1024)):
        Dg, Ig = ix.search(xq, k, efsearch=ef)
        Do, Io, _, _ = h.search(xq, k, ef=ef, nthreads=8, sorted_ids=dead, negate=True)
        assert_same_results(Dg, Ig, Do, Io)
        assert ix.stats()[6] == len(xq), "tombstones must run the candidate-heap form"
        check_f64(oracle, metric, xb, labels, xq, Dg, Ig)
    rmin, rmax = 1500, 3200
    Dg, Ig = ix.search(xq, 10, efsearch=64, id_range=(rmin, rmax))
    Do, Io, _, _ = h.search(xq, 10, ef=64, nthreads=8, id_range=(rmin, rmax), sorted_ids=dead, negate=True)
    assert_same_results(Dg, Ig, Do, Io)
    allow = np.arange(1000, 1000 + n, 3, dtype=np.int64)
    Dg, Ig = ix.search(xq, 10, efsearch=64, sorted_ids=allow)
    Do, Io, _, _ = h.search(xq, 10, ef=64, nthreads=8, sorted_ids=np.setdiff1d(allow, dead))
    assert_same_results(Dg, Ig, Do, Io)
    assert not np.isin(Ig, dead).any()
    # every row deleted: the walk still runs, nothing comes back
    ix.delete(labels)
    assert ix.get_count() == 0
    Dg, Ig = ix.search(xq, 10, efsearch=64)
    assert (Ig == -1).all()


@pytest.mark.parametrize("metric", [L2, IP, COSINE])
def test_ef_and_k_around_the_form_switch(oracle, metric):
    """ef = 1023 is the largest merged-array walk, ef = 1024 the smallest unfiltered heap walk (non-strict stop); k > ef
    runs with ef_run = k.  ef is sticky on both sides, so the calls run in the same order."""
    n, d = 3000, 32
    ix, h, xb, labels = pair(oracle, metric, n, d, seed=10 + metric)
    xq = np.random.default_rng(11).random((24, d)).astype(np.float32)
    sticky = 10
    for k, ef in ((10, HNSW_CAND_SMEM - 1), (10, HNSW_CAND_SMEM), (200, 16), (1024, 0)):
        Dg, Ig = ix.search(xq, k, efsearch=ef)
        sticky = ef if ef > 0 else sticky
        heap_form = max(k, sticky) + 1 > HNSW_CAND_SMEM
        assert ix.stats()[6] == (len(xq) if heap_form else 0), f"k={k} ef={ef}: wrong kernel form"
        Do, Io, _, _ = h.search(xq, k, ef=ef, nthreads=8)
        assert_same_results(Dg, Ig, Do, Io)
        assert (Ig >= 0).all()
        check_f64(oracle, metric, xb, labels, xq, Dg, Ig)
        if ef == HNSW_CAND_SMEM:
            want = brute_f64(oracle, metric, xb, labels, xq, 10)
            rec = np.mean([len(set(a) & set(b)) / 10 for a, b in zip(Ig, want)])
            assert rec >= 0.99, rec


@pytest.mark.parametrize("d,ef", [(1, 64), (7, 64), (33, 64), (33, HNSW_CAND_SMEM), (1536, HNSW_CAND_SMEM), (4096, HNSW_CAND_SMEM)])
def test_dimensions(oracle, d, ef):
    """d % 4 != 0 takes the scalar tail of quad_distance; d = 1536 / 4096 with ef = 1024 sizes the query row plus both heaps
    in shared memory."""
    n = 1500 if d < 1000 else 600
    for metric in ((L2,) if d == 1 else (L2, COSINE)):  # at d = 1 every positive row normalises to 1.0
        ix, h, xb, labels = pair(oracle, metric, n, d, M=8, efc=48, seed=d)
        xq = np.random.default_rng(d).random((64 if d == 1 else 16, d)).astype(np.float32)
        if d == 1:  # keep queries whose squared differences are all distinct (no exact ties to break)
            sq = (xb[None, :, 0] - xq[:, None, 0]) ** 2
            xq = xq[[len(np.unique(r)) == n for r in sq]][:16]
            assert len(xq) >= 8
        for kw in ({}, {"id_range": (1100, 1000 + n)}):
            Dg, Ig = ix.search(xq, 10, efsearch=ef, **kw)
            Do, Io, _, _ = h.search(xq, 10, ef=ef, nthreads=8, **kw)
            assert_same_results(Dg, Ig, Do, Io)
            check_f64(oracle, metric, xb, labels, xq, Dg, Ig)


def test_candidate_heap_spills_to_global_memory(oracle):
    """A filter that passes 3 labels keeps the result set below ef, so every fresh neighbour enters the candidate heap:
    on 20k nodes it grows far past its 1024 shared-memory entries."""
    n, d = 20000, 16
    ix, h, xb, labels = adopted(oracle, L2, n, d, seed=3)
    rng = np.random.default_rng(4)
    xq = rng.random((8, d)).astype(np.float32)
    allow = np.sort(rng.choice(labels, 3, replace=False))
    peak, reached = flooded_walk(ix.get_trained_state(), xq[0])
    assert peak > HNSW_CAND_SMEM
    Dg, Ig = ix.search(xq, 5, efsearch=32, sorted_ids=allow)
    Do, Io, _, _ = h.search(xq, 5, ef=32, nthreads=8, sorted_ids=allow)
    assert_same_results(Dg, Ig, Do, Io)
    assert set(Ig[0][Ig[0] >= 0]) == set(allow[reached[allow - 1]])  # every reachable allowed label (labels are row + 1)
    assert (Ig[:, 3:] == -1).all()
    check_f64(oracle, L2, xb, labels, xq, Dg, Ig)


def test_flooded_walk_is_not_truncated(oracle):
    """Regression: the heap form once capped its candidate heap at 65,536 entries and, past the cap, ended the walk early
    and returned OK with a truncated answer.  Each query here lets through only the 4 labels farthest from it, so the walk
    floods the graph; the measured open set exceeds that old cap, and the answer must still be those 4 labels."""
    n, d = 200000, 16
    ix, h, xb, labels = adopted(oracle, L2, n, d, M=16, efc=40, seed=1)
    blob = ix.get_trained_state()
    rng = np.random.default_rng(2)
    xq = rng.random((4, d)).astype(np.float32)
    X = xb.astype(np.float64)
    peak, reached = flooded_walk(blob, xq[0])
    print(f"n={n}: peak open set of a flooded walk {peak}")
    assert peak > 65536, f"the flooded walk peaks at {peak} open nodes: raise n to reach the regime this test is for"
    for qi in range(len(xq)):
        far = np.sort(labels[np.argsort(((X - xq[qi].astype(np.float64)) ** 2).sum(1))[-4:]])
        Dg, Ig = ix.search(xq[qi:qi + 1], 10, efsearch=32, sorted_ids=far)
        Do, Io, _, _ = h.search(xq[qi:qi + 1], 10, ef=32, sorted_ids=far)
        assert_same_results(Dg, Ig, Do, Io)
        assert (Ig[0, 4:] == -1).all()
        if qi == 0:
            assert set(Ig[0][Ig[0] >= 0]) == set(far[reached[far - 1]])
        check_f64(oracle, L2, xb, labels, xq[qi:qi + 1], Dg, Ig)
    # more queries than one launch's candidate pool holds: the queries run in chunks, each chunk equal to the oracle
    per_launch = HNSW_CAND_POOL_BYTES // ((n + 1) * 8)
    xm = rng.random((per_launch + 5, d)).astype(np.float32)
    allow = np.sort(rng.choice(labels, 4, replace=False))
    Dg, Ig = ix.search(xm, 4, efsearch=16, sorted_ids=allow)
    assert ix.stats()[0] == 2 and ix.stats()[6] == len(xm)
    Do, Io, _, _ = h.search(xm, 4, ef=16, nthreads=16, sorted_ids=allow)
    assert_same_results(Dg, Ig, Do, Io)


@pytest.mark.parametrize("metric", [L2, IP])
def test_exact_ties(oracle, metric):
    """Duplicated rows under different labels tie exactly.  DESIGN §6: the merged-array form may break such ties in another
    order than std::priority_queue, so the checks are order (distance, label), the multiset of distances, and the ids
    wherever a distance is not tied."""
    rng = np.random.default_rng(21)
    base = rng.random((800, 16)).astype(np.float32)
    xb = np.concatenate([base, base[:400], base[:200]])
    ix, h, _, labels = pair(oracle, metric, len(xb), 16, M=12, efc=64, data=xb)
    xq = np.concatenate([base[:10], rng.random((10, 16)).astype(np.float32)])
    _, inv, cnt = np.unique(xb, axis=0, return_inverse=True, return_counts=True)
    tied = labels[cnt[inv.ravel()] > 1]  # a tie group may straddle the k-th slot: one member on each side
    for kw in ({}, {"id_range": (1100, 3000)}):
        Dg, Ig = ix.search(xq, 12, efsearch=64, **kw)
        Do, Io, _, _ = h.search(xq, 12, ef=64, nthreads=8, **kw)
        check_f64(oracle, metric, xb, labels, xq, Dg, Ig)
        for qi in range(len(xq)):
            assert np.array_equal(np.sort(Dg[qi]).view(np.uint32), np.sort(Do[qi]).view(np.uint32))
            single = ~np.isin(Io[qi], tied)
            assert np.array_equal(Ig[qi][single], Io[qi][single])
