"""Exactness across the whole FP32 range: tiny, huge and mixed-magnitude data against float64 and the oracle.

The tile scan is exact because its certificate holds: |approx - exact| <= eps(q) for every (query, row), eps = tc_eps()
(DESIGN.md 4.2).  A purely relative eps holds only while the arithmetic stays normal: subnormal rounding errs by an
absolute amount, the FP16 mirror's scale product hs * qs can underflow to 0 or overflow, and ||x||^2 or ||q||^2 can
overflow while the exact distances sum(q_i - x_i)^2 stay finite.  These tests walk a ladder of power-of-two scales
through each of those regimes, on both sides of each boundary, and check

  a) the certificate's premise against float64, in all five tile arithmetics (eps = +inf is allowed: the query is then
     re-run on the exact scan, and only then may an approximate score be non-finite);
  b) every float search path end to end: ids and distance bits equal the oracle's and the exact scan's;
  c) the route: ordinary data never leaves the tile scan, overflowing data always ends on the exact scan;
  d) cosine normalisation of rows whose squared norm underflows or overflows, bit for bit against the oracle.

Data are U[0.5, 1) ("u") or standard normal ("n": signs matter for IP), rows and queries scaled independently by 2^m.
The boundaries quoted below are for U[0.5, 1) at the end-to-end dimension D = 64: the largest coordinate lies in
[2^(m-1), 2^m), so the FP16 scales are hs = qs = 2^(m-15) and ||x||^2 ~ 37 * 2^(2m)."""
import numpy as np
import pytest

import b200vs
import oracle_lib
from b200vs import COSINE, FLAT, HNSW, IP, IVF_FLAT, IVF_PQ, L2
from gpu_util import require_gpu
from test_gpu_tc_bound import exact_scores

pytestmark = pytest.mark.gpu

N, D, NQ, K, NLIST, NPROBE, PQ_M = 4000, 64, 32, 10, 64, 8, 8

# name -> (query exponent, row exponent)
RUNGS = {
    "sub": (-130, -130),    # coordinates are FP32 subnormals (< 2^-126); every product and norm underflows to 0
    "prod-": (-66, -66),    # products q_i x_i in [2^-134, 2^-132): subnormal (below m = -63)
    "prod+": (-63, -63),    # products in [2^-128, 2^-126): on the subnormal / normal boundary
    "fp16-": (-60, -60),    # FP16 hs * qs = 2^-150: rounds to 0, every FP16 dot becomes 0
    "fp16+": (-59, -59),    # hs * qs = 2^-148: subnormal, still an exact power of two
    "m-20": (-20, -20),     # control: everything normal
    "m0": (0, 0),           # control
    "m20": (20, 20),        # control
    "norm-": (60, 60),      # ||x||^2 ~ 2^125: finite
    "norm+": (63, 63),      # ||x||^2 ~ 2^131: overflows; L2 distances of close pairs (~2^127) stay finite
    "inf": (66, 66),        # every L2 distance and inner product overflows
    "q-tiny": (-100, 40),   # asymmetric: products ~2^-60 normal, ||q||^2 ~2^-195 underflows to 0
    "x-tiny": (40, -100),
    "mixed": (None, None),  # rows and queries each at their own scale, 2^-60 .. 2^60
}
CONTROLS = {"m-20": -20, "m0": 0, "m20": 20}
METRICS = {L2: "L2", IP: "IP", COSINE: "cos"}


@pytest.fixture(autouse=True)
def _gpu():
    require_gpu()


def draw(rng, data, shape):
    return (0.5 + 0.5 * rng.random(shape) if data == "u" else rng.standard_normal(shape)).astype(np.float32)


def scale(x, m, rng):
    """x * 2^m (rounded to FP32 once, where it lands below the normal range); m = None: a random 2^-60 .. 2^60 per row."""
    if m is None:
        e = rng.integers(-60, 61, size=(x.shape[0], 1))
        return np.ldexp(x, e).astype(np.float32)
    return np.ldexp(x, m).astype(np.float32)


def dataset(rung, data, n, nq, d, seed):
    rng = np.random.default_rng(seed)
    mq, mx = RUNGS[rung]
    unit_b, unit_q = draw(rng, data, (n, d)), draw(rng, data, (nq, d))
    xb, xq = scale(unit_b, mx, rng), scale(unit_q, mq, rng)
    xq[1] = xb[7]  # a query on a stored row: distance 0, the exact top-1 whatever the scale
    return unit_b, xb, xq


def same(tag, got, want, id_mask=None):
    """Ids and distance bits equal.  A NaN (inf - inf inside an overflowing distance) matches any NaN: the CPU's default
    NaN is negative, CUDA's positive.  id_mask: where ids must match (default everywhere)."""
    Dg, Ig = got
    Dw, Iw = want
    bad = np.argwhere((Ig != Iw) & (True if id_mask is None else id_mask))
    assert bad.size == 0, f"{tag}: ids differ at {bad[:4].tolist()}: {Ig[tuple(bad[0])]} vs {Iw[tuple(bad[0])]}"
    bad = np.argwhere((Dg.view(np.uint32) != Dw.view(np.uint32)) & ~(np.isnan(Dg) & np.isnan(Dw)))
    assert bad.size == 0, f"{tag}: distance bits differ at {bad[:4].tolist()}: {Dg[tuple(bad[0])]!r} vs {Dw[tuple(bad[0])]!r}"


def nan_rows(D):
    """Queries whose oracle result holds a NaN distance (an inner product that overflowed to +inf and -inf): the
    oracle's heaps order NaN arbitrarily, so there is no reference order to compare with (DESIGN.md 6)."""
    return np.isnan(D).any(axis=1)[:, None]


def same_as_oracle(tag, got, want, id_mask=True):
    """As same(), except that ids tied at an infinite distance may come in another order (the exact scan orders such
    ties by id, the oracle's heaps do not for -inf), and queries with a NaN oracle distance are not compared."""
    keep = ~nan_rows(want[0])
    Dg = np.where(keep, got[0], np.float32(0))
    Dw = np.where(keep, want[0], np.float32(0))
    same(tag, (Dg, got[1]), (Dw, want[1]), id_mask=np.isfinite(want[0]) & keep & id_mask)


def same_as_oracle_hnsw(tag, got, want):
    """HNSW: where a query's top-k distances repeat, the beam may walk ties in another order (DESIGN.md 6), so only
    distances are compared for that query.  Tiny IP data makes every distance 1 - ip = 1.0, and so on."""
    distinct = np.array([len(np.unique(r.view(np.uint32))) == r.size for r in want[0]])
    same_as_oracle(tag, got, want, id_mask=distinct[:, None])


def stored(oracle, metric, x):
    return oracle.normalize_faiss(x) if metric == COSINE else x


# ---------------------------------------------------------------------------------------------------------------------
# a) the premise of the certificate, against float64
# ---------------------------------------------------------------------------------------------------------------------
ARITHS = {"tf32": dict(), "split": dict(split=True), "fp16": dict(half=True), "tf32-sample": dict(sample=True),
          "fp16-sample": dict(half=True, sample=True)}
SPAN, SAMPLE = 2048, 32  # TC_SPAN, TC_SAMPLE: the first 32 rows of every 2048-row span are sampled


@pytest.mark.parametrize("rung", list(RUNGS))
@pytest.mark.parametrize("data", ["u", "n"])
@pytest.mark.parametrize("d", [32, 64, 768])
def test_tc_premise_holds_or_eps_is_inf(oracle, d, data, rung):
    n, nq = 512, 16
    _, xb, xq = dataset(rung, data, n, nq, d, seed=d * 31 + len(rung) + (data == "n"))
    sampled = np.zeros(n, bool)
    sampled[[r for s in range(0, n, SPAN) for r in range(s, min(s + SAMPLE, n))]] = True
    for metric in (L2, IP, COSINE):
        ix = b200vs.Index(FLAT, metric, d)
        ix.add(xb, np.arange(n, dtype=np.int64))
        s64, rerr = exact_scores(oracle, metric, stored(oracle, metric, xb), stored(oracle, metric, xq))
        for name, kw in ARITHS.items():
            approx, eps = ix.tc_scores(xq, **kw)
            tag = f"{rung}/{data} d={d} {METRICS[metric]} {name}"
            assert not np.isnan(eps).any() and np.all(eps >= 0), f"{tag}: eps {eps}"
            cols = sampled if kw.get("sample") else np.ones(n, bool)
            if kw.get("sample"):
                assert np.isnan(approx[:, ~cols]).all()
            a = approx[:, cols].astype(np.float64)
            inf_q = np.isinf(eps)
            assert np.isfinite(a[~inf_q]).all(), f"{tag}: non-finite approximate score under a finite eps"
            lhs = np.abs(a - s64[:, cols]) + rerr[:, cols]
            bad = np.argwhere((lhs > eps[:, None].astype(np.float64)) & ~inf_q[:, None])
            assert bad.size == 0, (f"{tag}: bound violated at (q, row) {bad[0].tolist()}: |err| {lhs[tuple(bad[0])]:.6g} "
                                   f"> eps {eps[bad[0][0]]:.6g} (approx {a[tuple(bad[0])]!r}, s64 {s64[:, cols][tuple(bad[0])]!r})")
        ix.close()


# ---------------------------------------------------------------------------------------------------------------------
# b) + c) every float search path, end to end
# ---------------------------------------------------------------------------------------------------------------------
def route(rung, metric, data):
    """What the tile scan must do with the query batch:
      'serve'   take every query and certify it (re-run none);
      'exact'   leave every query to the exact scan: decline the batch, or take it and re-run every query (eps = +inf
                once L2's (||q|| + max ||x||)^2 or IP's ||q|| max ||x|| passes 2^125);
      'decline' not take the batch at all: max ||x||^2 > 2^125 (L2) or max ||x|| = inf (IP) leaves no query a finite eps.
    Cosine rows and queries are normalised first, so only the controls say anything about its route."""
    if rung in CONTROLS:
        return "serve" if data == "u" else None
    if metric == COSINE:
        return None
    if rung in ("norm+", "inf"):
        return "decline"  # max ||x||^2 >= 2^130 at these scales (L2); ||x||^2 overflows to inf (IP)
    if rung == "norm-":
        return "exact"  # ||x||^2 ~ 2^124 .. 2^126: on either side of the L2 limit depending on d and the draw
    if rung == "mixed":
        return "any"  # rows up to 2^60: the L2 table may sit just past the limit
    return None  # underflow rungs: the tile scan takes the batch; exact by the certificate or by the re-run


def check_route(ix, rung, metric, data, nq, serve=True):
    """serve = False: lists of ~60 rows are mostly sampled, so the certificate legitimately fails for some queries at any
    scale; test_tile_scan_serves_ordinary_scales checks IVF-Flat's route on long lists instead."""
    st = ix.stats()
    r = route(rung, metric, data)
    if r == "decline":
        assert st[1] == 0, f"{rung}: the tile scan took {st[1]} queries although no eps can be finite"
    elif r == "exact":
        assert st[1] == 0 or st[2] == st[1] == nq, f"{rung}: tile scan took {st[1]}, re-ran {st[2]} of {nq} (eps = +inf)"
    elif r != "any":
        assert st[1] == nq, f"{rung}: the tile scan served {st[1]} of {nq} queries"
        if r == "serve" and serve:
            assert st[2] == 0, f"{rung}: {st[2]} queries re-run on ordinary data"


@pytest.mark.parametrize("rung", list(RUNGS))
@pytest.mark.parametrize("metric", [L2, IP, COSINE], ids=["L2", "IP", "cos"])
@pytest.mark.parametrize("data", ["u", "n"])
def test_flat_paths(oracle, data, metric, rung):
    _, xb, xq = dataset(rung, data, N, NQ, D, seed=101 + metric + len(rung))
    ids = np.arange(N, dtype=np.int64) * 3 + 5
    ix = b200vs.Index(FLAT, metric, D)
    ix.add(xb, ids)
    ix.set_profiling(True)
    want = oracle.flat_search(metric, stored(oracle, metric, xb), ids, xq, K, nthreads=8)
    ex = ix.search(xq, K, exact_only=True)
    same_as_oracle(f"{rung} exact vs oracle", ex, want)
    same(f"{rung} tile", ix.search(xq, K), ex)
    check_route(ix, rung, metric, data, NQ)
    same(f"{rung} flat_small", ix.search(xq[:4], K), (ex[0][:4], ex[1][:4]))
    assert ix.stats()[1] == 0
    ix.close()


def ivf_state(oracle, metric, unit_b, mx):
    """Centroids trained on the unscaled rows, then scaled like them (k-means itself is not under test here)."""
    cent = oracle.kmeans(metric, stored(oracle, metric, unit_b), NLIST, niter=4)
    return cent if metric == COSINE or mx is None else np.ldexp(cent, mx).astype(np.float32)


@pytest.mark.parametrize("rung", list(RUNGS))
@pytest.mark.parametrize("metric", [L2, IP, COSINE], ids=["L2", "IP", "cos"])
@pytest.mark.parametrize("d", [64, 36], ids=["fp16", "tf32"])
def test_ivf_flat_paths(oracle, d, metric, rung):
    data = "n" if metric == IP else "u"
    unit_b, xb, xq = dataset(rung, data, N, NQ, d, seed=202 + d + metric + len(rung))
    cent = ivf_state(oracle, metric, unit_b, RUNGS[rung][1])
    ids = np.arange(N, dtype=np.int64) + 1
    ix = b200vs.Index(IVF_FLAT, metric, d, nlist=NLIST)
    ix.set_trained_state(b200vs.ivf_state_blob(cent, metric))
    ix.add(xb, ids)
    ix.set_profiling(True)
    off, lx, _, lids = ix.export_lists(NLIST)
    want = oracle.ivfflat_search(metric, cent, off, lx, lids, xq, K, NPROBE, nthreads=8)
    ex = ix.search(xq, K, nprobe=NPROBE, exact_only=True)
    same_as_oracle(f"{rung} exact vs oracle", ex, want)
    same(f"{rung} tile", ix.search(xq, K, nprobe=NPROBE), ex)
    check_route(ix, rung, metric, data, NQ, serve=False)
    ix.close()


@pytest.mark.parametrize("rung", list(RUNGS))
@pytest.mark.parametrize("metric", [L2, IP], ids=["L2", "IP"])
def test_coarse_pass_ranks_centroids_like_the_oracle(oracle, metric, rung):
    """The split-arithmetic dense pass + certified re-score at the 1024 x 768 shape of the sharded coarse tests."""
    import torch
    nlist, d, nq, nprobe = 1024, 768, 64, 32
    _, cent, xq = dataset(rung, "u" if metric == L2 else "n", nlist, nq, d, seed=303 + metric + len(rung))
    ix = b200vs.Index(IVF_FLAT, metric, d, nlist=nlist)
    ix.set_trained_state(b200vs.ivf_state_blob(cent, metric))
    q = torch.from_numpy(xq).cuda()
    sc = torch.empty((nq, nprobe), dtype=torch.float32, device="cuda")
    pl = torch.empty((nq, nprobe), dtype=torch.int64, device="cuda")
    ix.coarse_device(nq, q.data_ptr(), nprobe, 0, nlist, sc.data_ptr(), pl.data_ptr())
    torch.cuda.synchronize()
    cd, ci = oracle.flat_search(metric, cent, np.arange(nlist, dtype=np.int64), xq, nprobe, nthreads=8)
    got = pl.cpu().numpy()
    bad = np.argwhere((got != ci) & np.isfinite(cd))  # ties at an infinite score: see same_as_oracle
    assert bad.size == 0, f"{rung}: probe differs at {bad[:4].tolist()}: {got[tuple(bad[0])]} vs {ci[tuple(bad[0])]}"
    if metric == L2:  # the coarse score is the L2 distance itself
        assert np.array_equal(sc.cpu().numpy().view(np.uint32), cd.view(np.uint32)), f"{rung}: coarse scores differ"
    ix.close()


@pytest.mark.parametrize("rung", list(RUNGS))
@pytest.mark.parametrize("metric", [L2, IP, COSINE], ids=["L2", "IP", "cos"])
def test_ivf_pq_and_hnsw(oracle, metric, rung):
    data = "n" if metric == IP else "u"
    unit_b, xb, xq = dataset(rung, data, N, NQ, D, seed=404 + metric + len(rung))
    mx = RUNGS[rung][1]
    ids = np.arange(N, dtype=np.int64) + 1
    st = stored(oracle, metric, unit_b)
    cent = oracle.kmeans(metric, st, NLIST, niter=4)
    cb = oracle.pq_train(st - cent[oracle.assign(metric, st, cent)], PQ_M, niter=4)
    if metric != COSINE and mx is not None:
        cent, cb = np.ldexp(cent, mx).astype(np.float32), np.ldexp(cb, mx).astype(np.float32)
    ix = b200vs.Index(IVF_PQ, metric, D, nlist=NLIST, pq_m=PQ_M, pq_nbits=8)
    ix.set_trained_state(b200vs.ivfpq_state_blob(cent, cb, metric))
    ix.add(xb, ids)
    off, _, codes, lids = ix.export_lists(NLIST, with_vectors=False, code_size=PQ_M)
    same_as_oracle(f"{rung} ivf-pq", ix.search(xq, K, nprobe=NPROBE),
         oracle.ivfpq_search(metric, cent, cb, off, codes, lids, xq, K, NPROBE, nthreads=8))
    ix.close()
    n = 1000
    h = oracle_lib.OracleHnsw(oracle, metric, D, n, 16, 100)
    h.add(xb[:n], ids[:n])
    hx = b200vs.Index(HNSW, metric, D, hnsw_m=16, hnsw_efc=100, max_elements=n)
    hx.add(xb[:n], ids[:n])
    Do, Io, _, _ = h.search(xq, K, ef=64, nthreads=8)
    same_as_oracle_hnsw(f"{rung} hnsw", hx.search(xq, K, efsearch=64), (Do, Io))
    hx.close()
    h.close()


def range_want(oracle, Dall, Iall, radius):
    """Per query: the (distance bits, id) pairs strictly inside the radius, sorted."""
    return [sorted((int(dv), int(i)) for dv, i, f in zip(Dr.view(np.uint32), Ir, Dr) if i >= 0 and f < radius)
            for Dr, Ir in zip(Dall, Iall)]


def range_got(D, I, C):
    return [sorted((int(dv), int(i)) for dv, i in zip(D[q, :C[q]].view(np.uint32), I[q, :C[q]])) for q in range(len(C))]


@pytest.mark.parametrize("rung", list(RUNGS))
def test_range_and_bruteforce_scans(oracle, rung):
    """L2 range search (Flat, IVF-Flat, the streaming range scan) and the streaming top-k scan; the radius is the
    median 10-th neighbour distance, so it scales with the data."""
    unit_b, xb, xq = dataset(rung, "u", N, NQ, D, seed=505 + len(rung))
    ids = np.arange(N, dtype=np.int64) + 1
    Dall, Iall = oracle.flat_search(L2, xb, ids, xq, N, nthreads=8)
    radius = float(np.float32(np.median(Dall[:, K - 1])))
    if not np.isfinite(radius) or radius == 0.0:
        radius = float(np.finfo(np.float32).max)
    want = range_want(oracle, Dall, Iall, radius)
    fl = b200vs.Index(FLAT, L2, D)
    fl.add(xb, ids)
    assert range_got(*fl.range_search(xq, radius, max_results=N)) == want, f"{rung}: Flat range search"
    rs = b200vs.BruteForceRangeScan(L2, D, xq, radius, max_results=N)
    for a in range(0, N, 2048):
        rs.push(xb[a:a + 2048], ids[a:a + 2048])
    assert range_got(*rs.finish()) == want, f"{rung}: streaming range scan"
    bs = b200vs.BruteForceScan(L2, D, xq, K)
    for a in range(0, N, 2048):
        bs.push(xb[a:a + 2048], ids[a:a + 2048])
    same_as_oracle(f"{rung} streaming top-k scan", bs.finish(), (Dall[:, :K], Iall[:, :K]))
    fl.close()
    cent = ivf_state(oracle, L2, unit_b, RUNGS[rung][1])
    iv = b200vs.Index(IVF_FLAT, L2, D, nlist=NLIST)
    iv.set_trained_state(b200vs.ivf_state_blob(cent, L2))
    iv.add(xb, ids)
    off, lx, _, lids = iv.export_lists(NLIST)
    Dv, Iv = oracle.ivfflat_search(L2, cent, off, lx, lids, xq, N, NPROBE, nthreads=8)
    assert range_got(*iv.range_search(xq, radius, max_results=N, nprobe=NPROBE)) == range_want(oracle, Dv, Iv, radius), \
        f"{rung}: IVF-Flat range search"
    iv.close()


# ---------------------------------------------------------------------------------------------------------------------
# c) the guard stays out of the way of ordinary data
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("m", [-40, -20, 0, 20, 40])
@pytest.mark.parametrize("kind", [FLAT, IVF_FLAT], ids=["flat", "ivf"])
@pytest.mark.parametrize("metric", [L2, IP], ids=["L2", "IP"])
def test_tile_scan_serves_ordinary_scales(oracle, metric, kind, m):
    """Uniform data at ordinary scales: the tile scan certifies every query.  IVF-Flat uses 16 lists of ~2500 rows, so
    that the threshold sample (32 rows of every 2048) is a small part of each list, as in a real deployment."""
    n = N if kind == FLAT else 40000
    rng = np.random.default_rng(606 + m)
    unit_b, unit_q = draw(rng, "u", (n, D)), draw(rng, "u", (NQ, D))
    xb, xq = np.ldexp(unit_b, m).astype(np.float32), np.ldexp(unit_q, m).astype(np.float32)
    ids = np.arange(n, dtype=np.int64)
    if kind == FLAT:
        ix = b200vs.Index(FLAT, metric, D)
        kw = {}
    else:
        cent = np.ldexp(oracle.kmeans(metric, unit_b, 16, niter=4), m).astype(np.float32)
        ix = b200vs.Index(IVF_FLAT, metric, D, nlist=16)
        ix.set_trained_state(b200vs.ivf_state_blob(cent, metric))
        kw = dict(nprobe=4)
    ix.add(xb, ids)
    ix.set_profiling(True)
    got = ix.search(xq, K, **kw)
    st = ix.stats()
    assert st[1] == NQ and st[2] == 0, f"2^{m}: served {st[1]}, re-ran {st[2]} of {NQ}"
    same(f"2^{m}", got, ix.search(xq, K, exact_only=True, **kw))
    ix.close()


# ---------------------------------------------------------------------------------------------------------------------
# d) cosine normalisation of rows whose squared norm underflows or overflows
# ---------------------------------------------------------------------------------------------------------------------
def extreme_rows(rng, n, d):
    """Rows at 2^-80 (||x||^2 underflows to 0), 2^-72 (||x||^2 subnormal), 2^-60, 1, 2^60 (||x||^2 near 2^126) and
    2^70 (||x||^2 overflows), each as U[0.5, 1) and normal draws."""
    exps = np.array([-80, -72, -60, 0, 60, 70])
    e = exps[np.arange(n) % len(exps)][:, None]
    x = np.where(np.arange(n)[:, None] % 2 == 0, draw(rng, "u", (n, d)), draw(rng, "n", (n, d)))
    return np.ldexp(x, e).astype(np.float32)


@pytest.mark.parametrize("d", [8, 64, 768])
def test_cosine_normalisation_of_extreme_rows(oracle, d):
    rng = np.random.default_rng(707 + d)
    left, right = extreme_rows(rng, 24, d), extreme_rows(rng, 36, d)
    for alg in (b200vs.ALGORITHM_FAISS, b200vs.ALGORITHM_HNSWLIB):
        want, wl, wr = oracle.calc_distance(alg, oracle_lib.COSINE, left, right)
        got, gl, gr = b200vs.calc_distance(alg, COSINE, left, right, return_normalized=True)
        for name, g, w in (("distances", got, want), ("left", gl, wl), ("right", gr, wr)):
            bad = np.argwhere(g.view(np.uint32) != w.view(np.uint32))
            assert bad.size == 0, f"alg {alg} d={d} {name} differ at {bad[:4].tolist()}: {g[tuple(bad[0])]!r} vs {w[tuple(bad[0])]!r}"
    n, nq = 600, 20
    xb, xq = extreme_rows(rng, n, d), extreme_rows(rng, nq, d)
    ids = np.arange(n, dtype=np.int64) + 1
    fl = b200vs.Index(FLAT, COSINE, d)
    fl.add(xb, ids)
    want = oracle.flat_search(COSINE, oracle.normalize_faiss(xb), ids, xq, K, nthreads=8)
    same_as_oracle(f"d={d} Flat cosine (faiss normalisation)", fl.search(xq, K), want)
    same_as_oracle(f"d={d} Flat cosine, exact scan", fl.search(xq, K, exact_only=True), want)
    fl.close()
    h = oracle_lib.OracleHnsw(oracle, COSINE, d, n, 16, 100)
    h.add(xb, ids)
    hx = b200vs.Index(HNSW, COSINE, d, hnsw_m=16, hnsw_efc=100, max_elements=n)
    hx.add(xb, ids)
    Do, Io, _, _ = h.search(xq, K, ef=64, nthreads=8)
    same_as_oracle_hnsw(f"d={d} HNSW cosine (hnswlib normalisation)", hx.search(xq, K, efsearch=64), (Do, Io))
    hx.close()
    h.close()
