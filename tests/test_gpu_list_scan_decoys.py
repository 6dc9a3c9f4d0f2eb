"""The tile scan's certificate (DESIGN.md 4.2) on decoys, for every list-scan arithmetic and metric and for both branches
of the sample threshold.

A result is exact because every approximate score lies within eps of its exact score, the capture threshold T is wide
enough, and the finish kernel certifies A_k + 2 eps <= T (A_k = the k-th captured score), re-running every query that
fails on the exact scan.  A decoy is a pair of rows: R, whose exact score is just better than D's, and D, whose
approximate score is far better than R's.

* Top-k decoys on IVF-Flat in each list-scan arithmetic: the FP16 mirror (d % 8 == 0: IP, cosine) and the TF32 list
  form (d = 132, no mirror: L2, IP, cosine).  R must be the k-th neighbour, and a batch of the decoy query alone must be
  certified; the device's own share of the window (Flat tc_scores in the same arithmetic) is asserted too.
* Sample placement: the threshold pass samples the first TC_SAMPLE = 32 rows of every TC_SPAN = 2048-row span of a
  list, in stored (insertion) order.  With D sampled and R not, tc_tau_with_margin takes each of its branches:
  (a) T = tau (at least TAU_SAFE = 3 sampled scores below tau - 2 eps): R is not captured, so only the certificate keeps
      the result exact, and the query must be re-run;
  (b) T = tau + 2 eps (only D sampled, k = 1): R is captured and the query certified;
  (c) T = tau again, because the predicted captures under tau + 2 eps would overflow tc_cand_cap(k): re-run, exact.
  The premises (which sampled scores lie where) are read from the device's sample pass (Flat tc_scores(sample=True)).

Every search is compared with exact_only (ids and distance bits) and with the oracle; stats()[2] counts the queries
the tile pass handed to the exact scan."""
import numpy as np
import pytest

import b200vs
import fp16_emu as H
import tf32_emu as E
from b200vs import COSINE, FLAT, IP, IVF_FLAT, L2
from gpu_util import assert_same_results, require_gpu
from test_gpu_ivf_flat_half import arena_bytes
from test_gpu_range_edges import decoy_centroids, tc_cand_cap
from test_gpu_tc_adversarial import run_both

pytestmark = pytest.mark.gpu

SPAN, SAMPLE, TAU_SAFE = 2048, 32, 3  # TC_SPAN, TC_SAMPLE, TAU_SAFE (csrc/tc_scan.cu)
NAMES = {L2: "L2", IP: "IP", COSINE: "cos"}


@pytest.fixture(autouse=True)
def _gpu():
    require_gpu()


# arithmetic -> (d, half, {metric: generator}, floor of the pair's share of the 2 eps window).  The FP16 and TF32 L2
# pairs use more than half of the window, so a kernel whose window were half as wide returns D; the TF32 IP and cosine
# pairs reach only about 0.45 and 0.37 (row truncation lowers |D| too, so D's side gains from the query's rounding
# alone), and their floor is that emulated share.
ARITH = {
    "fp16": (128, True, {L2: H.decoy_l2, IP: H.decoy_ip, COSINE: H.decoy_cos}, {L2: 0.5, IP: 0.5, COSINE: 0.5}),
    "tf32list": (132, False, {L2: E.decoy_l2, IP: E.decoy_ip, COSINE: E.decoy_cos}, {L2: 0.5, IP: 0.4, COSINE: 0.35}),
}


def ivf(metric, rows, ids, half):
    """IVF-Flat with decoy_centroids: the pair rows land in list 0 behind the filler rows."""
    d = rows.shape[1]
    ix = b200vs.Index(IVF_FLAT, metric, d, nlist=4)
    ix.set_trained_state(b200vs.ivf_state_blob(decoy_centroids(d), metric))
    ix.add(rows, ids)
    assert arena_bytes(ix, d, 4, half) > 0, "the index keeps the FP16 mirror exactly when d % 8 == 0"
    return ix


def device_share(rows, q, r, dd, metric, half):
    """(R's tile score - D's) / (2 eps) from the device's own list-scan arithmetic, on a Flat view of the same rows."""
    fl = b200vs.Index(FLAT, metric, rows.shape[1])
    fl.add(rows, np.arange(rows.shape[0], dtype=np.int64))
    S, Eps = fl.tc_scores(np.repeat(q, 16, axis=0), half=half)
    fl.close()
    return float((np.float64(S[0, r]) - np.float64(S[0, dd])) / (2 * np.float64(Eps[0])))


# ---- top-k decoys ------------------------------------------------------------------------------------------------------
TOPK = [("fp16", IP), ("fp16", COSINE), ("tf32list", L2), ("tf32list", IP), ("tf32list", COSINE)]


@pytest.mark.parametrize("k", [1, 10])
@pytest.mark.parametrize("arith,metric", TOPK, ids=[f"{a}-{NAMES[m]}" for a, m in TOPK])
def test_topk_decoys(oracle, arith, metric, k):
    """32 queries, each with its own pair; index p holds pair p among filler rows and is searched with the whole batch:
    query p returns R as its k-th neighbour, and a batch of 16 copies of it stays on the tile path."""
    d, half, gens, floors = ARITH[arith]
    floor, npair = floors[metric], 32
    pairs = [gens[metric](np.random.default_rng(3000 * k + 100 * metric + p), d, k, nfill=1500) for p in range(npair)]
    xq = np.concatenate([p[1] for p in pairs])
    cent = decoy_centroids(d)
    for p in range(0, npair, 4):
        rows, q, r, dd = pairs[p]
        ids = np.arange(rows.shape[0], dtype=np.int64) * 7 + 3
        ix = ivf(metric, rows, ids, half)
        off, lx, _, lids = ix.export_lists(4)
        if metric == COSINE:  # unit vectors: the cosine normalisation leaves the pair and the query bit for bit
            for row in (r, dd):
                at = np.nonzero(lids == ids[row])[0][0]
                assert np.array_equal(lx[at].view(np.uint32), rows[row].view(np.uint32)), "a pair row was renormalised"
            assert np.array_equal(oracle.normalize_faiss(q).view(np.uint32), q.view(np.uint32)), "the query was renormalised"
        share = device_share(rows, q, r, dd, metric, half)
        print(f"[{arith}-{NAMES[metric]} k={k}] pair {p}: device share {share:.3f}")
        assert share > floor, f"pair {p}: on the device the decoy uses {share:.3f} of the 2 eps window"
        D, I, st = run_both(ix, xq, k, nprobe=4)
        assert st[1] == npair, st
        assert I[p, k - 1] == ids[r], f"pair {p}: the decoy displaced R (got id {I[p, k - 1]}, R {ids[r]}, D {ids[dd]})"
        _, Ic, stc = run_both(ix, np.repeat(q, 16, axis=0), k, nprobe=4)
        assert stc[1] == 16 and stc[2] == 0, f"pair {p}: the decoy query fell back to the exact scan: stats {stc}"
        assert np.all(Ic[:, k - 1] == ids[r])
        Do, Io = oracle.ivfflat_search(metric, cent, off, lx, lids, xq, k, 4, nthreads=8)
        assert_same_results(D, I, Do, Io)
        ix.close()


# ---- sample placement ------------------------------------------------------------------------------------------------
# (index kind, arithmetic): Flat scans TF32 rows as one list (the dense form), IVF-Flat its FP16 mirror or, at d = 132,
# the TF32 list form
PLACE = [(FLAT, "tf32"), (IVF_FLAT, "fp16"), (IVF_FLAT, "tf32list")]


def place_rows(gen, d, k, n, placed, seed):
    """n rows in stored order: {position: role} with role 'D', 'R' or 'C<m>' (the m-th closer row of the generator's
    k), filler rows everywhere else.  The filler rows are made non-negative on the axes decoy_centroids uses, so every
    row lands in list 0.  Returns (rows, query, position of R, position of D)."""
    src, q, r, dd = gen(np.random.default_rng(seed), d, k, nfill=n)
    fill = src[:n].copy()
    fill[:, d // 2:d // 2 + 3] = np.abs(fill[:, d // 2:d // 2 + 3])
    role = {"R": src[r], "D": src[dd], **{f"C{m}": src[n + m] for m in range(k - 1)}}
    rows = np.empty((n, d), np.float32)
    it = iter(fill)
    for i in range(n):
        rows[i] = role[placed[i]] if i in placed else next(it)
    pos = {v: i for i, v in placed.items()}
    return rows, q, pos.get("R"), pos["D"]


def sampled_scores(rows, q, metric, half):
    """The device's sample-pass scores of the decoy query (NaN off the sample) and its eps, on a Flat view of the rows."""
    fl = b200vs.Index(FLAT, metric, rows.shape[1])
    fl.add(rows, np.arange(rows.shape[0], dtype=np.int64))
    S, Eps = fl.tc_scores(np.repeat(q, 16, axis=0), half=half, sample=True)
    fl.close()
    return S[0].astype(np.float64), float(Eps[0])


def search_placed(oracle, kind, metric, rows, q, k, half):
    """16 copies of the decoy query on the tile path, on exact_only and on the oracle.  Returns (I, ids, stats)."""
    n, d = rows.shape
    ids = np.arange(n, dtype=np.int64) * 5 + 11
    xq = np.repeat(q, 16, axis=0)
    if kind == FLAT:
        ix = b200vs.Index(FLAT, metric, d)
        ix.add(rows, ids)
        kw = {}
    else:
        ix = ivf(metric, rows, ids, half)
        kw = dict(nprobe=4)
    off, lx, _, lids = ix.export_lists(1 if kind == FLAT else 4)
    assert off[1] - off[0] == n and np.array_equal(lids[:n], ids), "list 0 must hold every row in insertion order"
    assert np.array_equal(lx[:n].view(np.uint32), rows.view(np.uint32))
    D, I, st = run_both(ix, xq, k, **kw)
    print(f"\n[placement {'flat' if kind == FLAT else 'ivf'} {NAMES[metric]} k={k}] stats {st}")
    if kind == FLAT:
        Do, Io = oracle.flat_search(metric, rows, ids, xq, k, nthreads=8)
    else:
        Do, Io = oracle.ivfflat_search(metric, decoy_centroids(d), off, lx, lids, xq, k, 4, nthreads=8)
    assert_same_results(D, I, Do, Io)
    ix.close()
    return I, ids, st


def place_setup(kind, arith, metric):
    d, half, gens, floor = ARITH["tf32list" if arith == "tf32" else arith]
    if kind == FLAT:
        d = 128
    return d, half, gens[metric], floor[metric]


@pytest.mark.parametrize("metric", [L2, IP], ids=["L2", "IP"])
@pytest.mark.parametrize("kind,arith", PLACE, ids=["flat-tf32", "ivf-fp16", "ivf-tf32list"])
def test_sampled_decoy_with_safe_threshold(oracle, kind, arith, metric):
    """(a) k = 4: D sampled at position 3 behind 3 closer rows, R unsampled at 40 in the same span: tau is D's score, at
    least TAU_SAFE sampled scores lie below tau - 2 eps, so T = tau and R is not captured.  Only the certificate
    (A_k + 2 eps <= T fails) keeps the result exact: every copy is re-run, and R is the k-th neighbour.  A finish that
    trusted the sampling argument returns D."""
    k = 4
    d, half, gen, _ = place_setup(kind, arith, metric)
    # the generator's closer rows 1..3 of 4 (the first is too near R for the TF32 IP window)
    placed = {**{m: f"C{m + 1}" for m in range(k - 1)}, k - 1: "D", 40: "R"}
    rows, q, r, dd = place_rows(gen, d, k + 1, 1500, placed, 51 + metric)
    S, eps = sampled_scores(rows, q, metric, half)
    fin = np.sort(S[np.isfinite(S)])
    tau = fin[k - 1]
    assert S[dd] == tau and np.isnan(S[r]), "premise: tau is D's sampled score, R is not sampled"
    assert np.sum(S <= tau - 2.01 * eps) >= TAU_SAFE, "premise: the T = tau branch"
    I, ids, st = search_placed(oracle, kind, metric, rows, q, k, half)
    assert np.all(I[:, k - 1] == ids[r]), f"R must be the {k}-th neighbour (got {I[0]}, R {ids[r]}, D {ids[dd]})"
    assert st[1] == 16 and st[2] == 16, f"every copy must be re-run on the exact scan: stats {st}"


@pytest.mark.parametrize("metric", [L2, IP], ids=["L2", "IP"])
@pytest.mark.parametrize("kind,arith", PLACE, ids=["flat-tf32", "ivf-fp16", "ivf-tf32list"])
def test_sampled_decoy_with_margin(oracle, kind, arith, metric):
    """(b) k = 1, D the only sampled row near the query (position 5), R unsampled at 40: no sampled score lies below
    tau - 2 eps, so T = tau + 2 eps captures R and the query is certified.  Where the pair uses more than half of the
    window, a margin of eps instead of 2 eps would miss R and re-run the query."""
    d, half, gen, floor = place_setup(kind, arith, metric)
    rows, q, r, dd = place_rows(gen, d, 1, 1500, {5: "D", 40: "R"}, 61 + metric)
    S, eps = sampled_scores(rows, q, metric, half)
    tau = np.nanmin(S)
    assert S[dd] == tau and np.isnan(S[r]), "premise: tau is D's sampled score, R is not sampled"
    assert np.sum(S <= tau + 2.01 * eps) == 1, "premise: the margin branch (only D near tau)"
    assert device_share(rows, q, r, dd, metric, half) > floor
    I, ids, st = search_placed(oracle, kind, metric, rows, q, 1, half)
    assert np.all(I[:, 0] == ids[r])
    assert st[1] == 16 and st[2] == 0, f"R must be captured under tau + 2 eps and the query certified: stats {st}"


@pytest.mark.parametrize("metric", [L2, IP], ids=["L2", "IP"])
@pytest.mark.parametrize("kind,arith", PLACE, ids=["flat-tf32", "ivf-fp16", "ivf-tf32list"])
def test_sampled_ties_overflow_the_prediction(oracle, kind, arith, metric):
    """(c) k = 1, a copy of D on every sampled row of three spans (96 scores equal to tau) and R unsampled at 100: no
    sampled score lies below tau - 2 eps, and (96 + 4 sqrt 96) * 64 predicted captures exceed tc_cand_cap(1), so
    T = tau.  R is not captured, the certificate fails, and the re-run returns R."""
    d, half, gen, _ = place_setup(kind, arith, metric)
    n = 2 * SPAN + SAMPLE + 200
    placed = {s + i: "D" for s in range(0, n, SPAN) for i in range(SAMPLE)}
    placed[100] = "R"
    rows, q, r, dd = place_rows(gen, d, 1, n, placed, 71 + metric)
    S, eps = sampled_scores(rows, q, metric, half)
    tau = np.nanmin(S)
    cs = int(np.sum(S <= tau + 2 * eps))
    assert cs == 3 * SAMPLE and np.sum(S <= tau - 2 * eps) == 0 and np.isnan(S[r]), "premise: 96 sampled ties at tau"
    assert (cs + 4 * np.sqrt(cs)) * (SPAN // SAMPLE) > tc_cand_cap(1), "premise: the predicted captures overflow"
    I, ids, st = search_placed(oracle, kind, metric, rows, q, 1, half)
    assert np.all(I[:, 0] == ids[r])
    assert st[1] == 16 and st[2] == 16, f"every copy must be re-run on the exact scan: stats {st}"
