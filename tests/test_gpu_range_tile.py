"""Range search on the tensor-core tile scan (tc_range_search): Flat and IVF-Flat, L2 / IP / cosine, on the FP16 mirror
(IVF-Flat, d % 8 == 0) and on TF32 rows (Flat, and IVF-Flat with d % 8 == 4).

The tile pass only selects candidates: its capture threshold is the radius widened by the certificate bound, and every
captured row is re-scored by the exact kernel.  So every answer must equal the same call with exact_only (the exact scan
with the same threshold) in ids, distance bits and counts, and the restated expectation of test_gpu_exact_edges
(range_expect: the FP32 values of quad_distance's order, strict threshold, (key, id) order).  The profiling counters say
which path served the batch: stats[1] = queries of the tile pass, stats[2] = queries it handed to the exact scan."""
import numpy as np
import pytest

import b200vs
from b200vs import COSINE, FLAT, IP, IVF_FLAT, L2
from gpu_util import require_gpu
from test_gpu_exact_edges import boundary_radius, cand_mask, prep, radius_for, range_expect, raw_fp32

pytestmark = pytest.mark.gpu
NLIST = 32


@pytest.fixture(autouse=True)
def _gpu():
    require_gpu()


def _rows(rng, n, d):
    return rng.standard_normal((n, d)).astype(np.float32)


class Case:
    """A Flat or IVF-Flat index whose rows include exact duplicates (ties resolve by id), with the stored rows for the
    restated expectation (every list probed when nprobe = NLIST)."""

    def __init__(self, o, kind, metric, d, n=12000, dup=300, seed=0):
        rng = np.random.default_rng(seed)
        self.o, self.kind, self.metric, self.d = o, kind, metric, d
        xb = _rows(rng, n, d)
        xb = np.concatenate([xb, xb[:dup]])
        self.all_ids = rng.permutation(np.arange(1, n + dup + 1, dtype=np.int64))
        if kind == FLAT:
            self.ix = b200vs.Index(FLAT, metric, d)
        else:
            self.ix = b200vs.Index(IVF_FLAT, metric, d, nlist=NLIST)
            cent = prep(o, metric, xb[rng.choice(n, NLIST, replace=False)])
            self.ix.set_trained_state(b200vs.ivf_state_blob(cent, metric))
        self.ix.add(xb, self.all_ids)
        self.ix.coalescing(0)
        self.ix.set_profiling(True)
        self.refresh()

    def refresh(self):
        _, self.X, _, self.ids = self.ix.export_lists(1 if self.kind == FLAT else NLIST)

    def kw(self, nprobe):
        return {} if self.kind == FLAT else dict(nprobe=nprobe)

    def range(self, xq, radius, mr, route, nprobe=NLIST, **kw):
        """range_search == exact_only, bit for bit; the tile pass served it iff route == 'tile'; returns (D, I, C)."""
        D, I, C = self.ix.range_search(xq, radius, mr, **self.kw(nprobe), **kw)
        st = self.stats = self.ix.stats()
        if route == "tile":
            assert st[1] == len(xq), f"expected the tile pass, stats {st}"
        else:
            assert st[1] == 0, f"expected the exact scan, stats {st}"
        De, Ie, Ce = self.ix.range_search(xq, radius, mr, exact_only=True, **self.kw(nprobe), **kw)
        assert self.ix.stats()[1] == 0
        assert np.array_equal(C, Ce), "counts differ from the exact scan"
        assert np.array_equal(I, Ie), "ids differ from the exact scan"
        assert np.array_equal(D.view(np.uint32), De.view(np.uint32)), "distance bits differ from the exact scan"
        return D, I, C

    def expect(self, D, I, C, xq, radius, mr, queries, cand=None):
        Q = prep(self.o, self.metric, xq)
        for qi in queries:
            want_i, want_d, _ = range_expect(self.X, self.ids, Q[qi], self.metric, radius, mr, cand)
            assert C[qi] == len(want_i), f"query {qi}: {C[qi]} hits, expected {len(want_i)}"
            assert np.array_equal(I[qi, :C[qi]], want_i) and (I[qi, C[qi]:] == -1).all()
            assert np.array_equal(D[qi, :C[qi]].view(np.uint32), want_d.view(np.uint32))
            assert (D[qi, C[qi]:] == 0).all()


CASES = [(FLAT, 32), (FLAT, 36), (IVF_FLAT, 64), (IVF_FLAT, 36)]


@pytest.mark.parametrize("kind,d", CASES)
@pytest.mark.parametrize("metric", [L2, IP, COSINE])
def test_tile_range_equals_exact(oracle, metric, kind, d):
    c = Case(oracle, kind, metric, d, seed=11 + d + metric)
    rng = np.random.default_rng(5 + metric)
    xq = _rows(rng, 300, d)
    Q = prep(oracle, metric, xq)
    radius = radius_for(raw_fp32(c.X, Q[0], metric), metric, 100)
    some = list(range(6)) + [150, 299]
    # more than one 128-query group per list, and a single group
    for nq in (300, 16):
        D, I, C = c.range(xq[:nq], radius, 1024, "tile")
        c.expect(D, I, C, xq[:nq], radius, 1024, some[:6] if nq == 16 else some)
    # the probe-limited IVF search (candidates = the probed lists) against the exact scan alone
    if kind == IVF_FLAT:
        c.range(xq, radius, 1024, "tile", nprobe=6)
    # max_results 1 / 128 / 1024 / 4096 with more hits than kept: ties among the duplicated rows resolve by id
    wide = radius_for(raw_fp32(c.X, Q[0], metric), metric, 1500)
    for mr in (1, 128, 1024, 4096):
        D, I, C = c.range(xq[:32], wide, mr, "tile")
        c.expect(D, I, C, xq[:32], wide, mr, range(4))
    # the duplicated rows are hits of their own query: two rows per distance, id order
    dq = c.X[:32].copy() if metric == L2 else prep(oracle, metric, c.X[:32].copy())
    rd = radius_for(raw_fp32(c.X, prep(oracle, metric, dq)[0], metric), metric, 40)
    D, I, C = c.range(dq, rd, 64, "tile")
    c.expect(D, I, C, dq, rd, 64, range(8))
    # zero hits
    top = max(raw_fp32(c.X, Q[qi], metric).max() for qi in range(16))
    none = 0.0 if metric == L2 else float(np.float32(1) - top - np.float32(0.01))
    D, I, C = c.range(xq[:16], none, 64, "tile")
    assert (C == 0).all() and (I == -1).all() and (D == 0).all()
    # rows on the radius and a few ulps either side of it
    raw = raw_fp32(c.X, Q[0], metric)
    j, r = boundary_radius(raw, metric)
    for step in (-3, -1, 0, 1, 3):
        rr = float(np.float32(r))
        for _ in range(abs(step)):
            rr = float(np.nextafter(np.float32(rr), np.float32(np.inf if step > 0 else -np.inf)))
        D, I, C = c.range(xq[:16], rr, 256, "tile")
        c.expect(D, I, C, xq[:16], rr, 256, range(2))
        if step == 0:
            assert c.ids[j] not in I[0, :C[0]], "the row on the boundary must be excluded"
    # filters: id range, sorted ids, negated
    sub = np.sort(rng.choice(c.ids, 3000, replace=False))
    for filt in (dict(id_range=(2000, 9000)), dict(sorted_ids=sub), dict(sorted_ids=sub, negate=True)):
        D, I, C = c.range(xq[:64], radius, 512, "tile", **filt)
        c.expect(D, I, C, xq[:64], radius, 512, range(4), cand=cand_mask(c.ids, **filt))
    # tombstones
    c.ix.delete(c.all_ids[:2500])
    c.refresh()
    D, I, C = c.range(xq[:64], radius, 1024, "tile")
    c.expect(D, I, C, xq[:64], radius, 1024, range(4))
    # below 16 queries and exact_only: the exact scan
    c.range(xq[:15], radius, 1024, "exact")


@pytest.mark.parametrize("kind,d", [(FLAT, 32), (IVF_FLAT, 64)])
@pytest.mark.parametrize("metric", [L2, IP])
def test_capture_overflow_reruns_exactly(oracle, metric, kind, d):
    """Every row is a hit: more captured rows than the capture buffer holds (16384 a query), so every query is handed to
    the exact scan, and the answer is still the exact one."""
    c = Case(oracle, kind, metric, d, n=20000, dup=0, seed=3)
    xq = _rows(np.random.default_rng(8), 40, d)
    D, I, C = c.range(xq, 1e30, 256, "tile")
    st = c.stats
    assert st[2] == len(xq), f"every query must be re-run, stats {st}"
    assert (C == 256).all()
    c.expect(D, I, C, xq, 1e30, 256, range(3))


def test_untrained_ivf_has_no_hits():
    ix = b200vs.Index(IVF_FLAT, L2, 64, nlist=NLIST)
    D, I, C = ix.range_search(_rows(np.random.default_rng(1), 32, 64), 1e9, 16)
    assert (C == 0).all() and (I == -1).all() and (D == 0).all()


@pytest.mark.parametrize("metric", [L2, IP])
def test_norms_out_of_range_take_the_exact_scan(oracle, metric):
    """Rows whose norms leave the range the certificate bound covers (tc_norms_in_range): the exact scan serves the batch."""
    rng = np.random.default_rng(4)
    d = 32
    scale = np.float32(2.0 ** 63) if metric == L2 else np.float32(np.finfo(np.float32).max / 4)
    ix = b200vs.Index(FLAT, metric, d)
    xb = _rows(rng, 3000, d) * scale
    xb[:, 1:] = 0 if metric == IP else xb[:, 1:]
    ix.add(xb, np.arange(1, 3001, dtype=np.int64))
    ix.set_profiling(True)
    xq = _rows(rng, 20, d)
    D, I, C = ix.range_search(xq, 1e38 if metric == L2 else 0.5, 64)
    assert ix.stats()[1] == 0, "the tile pass must not serve rows outside the certified range"
    De, Ie, Ce = ix.range_search(xq, 1e38 if metric == L2 else 0.5, 64, exact_only=True)
    assert np.array_equal(C, Ce) and np.array_equal(I, Ie) and np.array_equal(D.view(np.uint32), De.view(np.uint32))
