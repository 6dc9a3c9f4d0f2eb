"""A numpy model of the candidate-pass exactness argument (DESIGN.md §4.2, §10-2) under adversarial score errors.

The tile scan only SELECTS rows with approximate scores a = e + noise, |noise| <= eps (e = the exact FP32 score); the
returned top-k must equal the exact scan's.  This file checks the selection rules themselves, independent of any kernel:

  single rank      tau = k-th smallest SAMPLED approximate score; capture a <= T; window a <= A_k + 2 eps (A_k = k-th
                   smallest captured); certified iff no overflow and A_k + 2 eps <= T.  T = tau, or T = tau + 2 eps
                   (the margin branch of tc_tau_with_margin: always certified).
  coarse set mode  rows with a <= A_k - 2 eps are certainly in the exact top-k, rows with a > A_k + 2 eps certainly not.
  list-sharded     every rank captures under the MIN over ranks of tau; a query is certified when ANY rank certifies
                   (that rank's A_k bounds the global one from above); each rank returns the exact top-k of its own
                   window and the merged result is the exact global top-k.  (Round-2 design; the shipped multi-GPU path
                   uses per-rank thresholds, which is the single-rank rule applied per shard.)

Uncertified queries take the exact scan in the engine, so the property to test is: certified => identical to exact.
"""
import numpy as np
import pytest


def exact_topk(e, ids, k):
    order = np.lexsort((ids, e))  # (score, id) ascending: the engine's tie rule
    return ids[order[:k]]


def noisy(rng, e, eps, adversarial, pivot=None):
    """Approximate scores.  Adversarial: rows at or below the pivot (the exact k-th best score) look worse by up to
    eps, rows above it look better by up to eps — the worst case for any threshold / window rule."""
    if adversarial:
        return e + np.where(e <= pivot, eps, -eps) * rng.choice([1.0, 0.97, 0.5], size=e.shape)
    return e + rng.uniform(-eps, eps, size=e.shape)


def kth(e, k):
    return np.sort(e)[k - 1]


def rank_select(a, e, ids, k, eps, T):
    """One rank: capture under T, window, exact re-score.  Returns (local exact top-k ids, certified, captured)."""
    cap = a <= T
    n = int(cap.sum())
    if n >= k:
        a_k = np.sort(a[cap])[k - 1]
        win = cap & (a <= a_k + 2 * eps)
        certified = bool(a_k + 2 * eps <= T)
    else:
        win = cap
        certified = False
    return exact_topk(e[win], ids[win], k), certified, n


@pytest.mark.parametrize("adversarial", [False, True])
@pytest.mark.parametrize("margin", [False, True])
def test_single_rank_rule(adversarial, margin):
    rng = np.random.default_rng(1 + 2 * adversarial + margin)
    checked = certified_n = 0
    for trial in range(400):
        n, k = int(rng.integers(200, 3000)), int(rng.integers(1, 20))
        eps = float(rng.choice([1e-3, 0.02, 0.2]))
        e = np.round(rng.normal(10, 1, n), 2 if trial % 3 == 0 else 6)  # rounding creates exact ties
        ids = rng.permutation(n).astype(np.int64)
        a = noisy(rng, e, eps, adversarial, kth(e, k))
        step = int(rng.choice([4, 16, 32])) if not margin else int(rng.choice([1, 2, 4]))
        sample = a[::step]
        if sample.size < k:
            continue
        tau = np.sort(sample)[k - 1]
        T = tau + 2 * eps if margin else tau
        got, certified, _ = rank_select(a, e, ids, k, eps, T)
        if margin:
            assert certified, "tau + 2 eps certifies by construction"
        if certified:
            certified_n += 1
            assert np.array_equal(got, exact_topk(e, ids, k))
        checked += 1
    assert checked > 300 and certified_n > 50


def test_coarse_set_mode_rule():
    """Probe tables are sets: sure rows (a <= A_k - 2 eps) + the best of the uncertain band == the exact top-k set."""
    rng = np.random.default_rng(5)
    for trial in range(400):
        n, k = int(rng.integers(64, 2000)), int(rng.integers(1, 48))
        if k > n:
            continue
        eps = float(rng.choice([1e-4, 0.01, 0.1]))
        e = rng.normal(0, 1, n)
        ids = np.arange(n, dtype=np.int64)
        a = noisy(rng, e, eps, trial % 2 == 0, kth(e, k))
        a_k = np.sort(a)[k - 1]
        if int((a <= a_k).sum()) != k:  # ties at the k-th approximate score: the kernel re-scores the full window instead
            continue
        sure = a <= a_k - 2 * eps
        band = (~sure) & (a <= a_k + 2 * eps)
        need = k - int(sure.sum())
        assert 0 < need <= int(band.sum())
        fill = exact_topk(e[band], ids[band], need)
        got = set(ids[sure].tolist()) | set(fill.tolist())
        assert got == set(exact_topk(e, ids, k).tolist())


@pytest.mark.parametrize("adversarial", [False, True])
def test_sharded_min_threshold_rule(adversarial):
    rng = np.random.default_rng(11 + adversarial)
    certified_n = 0
    for trial in range(300):
        world, k = int(rng.choice([2, 4, 8])), int(rng.integers(1, 16))
        eps = float(rng.choice([1e-3, 0.05]))
        sizes = rng.integers(20, 1500, world)
        e_all, ids_all, parts = [], [], []
        next_id = 0
        for r in range(world):
            e_all.append(rng.normal(10 + 0.3 * rng.standard_normal(), 1, sizes[r]))  # shards differ: some hold no global top-k row
            ids_all.append(np.arange(next_id, next_id + sizes[r], dtype=np.int64))
            next_id += sizes[r]
        pivot = kth(np.concatenate(e_all), k)  # the global k-th best exact score
        for e, ids in zip(e_all, ids_all):
            parts.append((e, ids, noisy(rng, e, eps, adversarial, pivot)))
        taus = []
        for e, ids, a in parts:
            s = a[::8]
            taus.append(np.sort(s)[k - 1] if s.size >= k else np.inf)
        T = min(taus)
        if not np.isfinite(T):
            continue
        outs, certs = [], []
        for e, ids, a in parts:
            got, cert, _ = rank_select(a, e, ids, k, eps, T)
            outs.append(got)
            certs.append(cert)
        if not any(certs):
            continue  # engine: exact re-run on every rank
        certified_n += 1
        e_cat, id_cat = np.concatenate(e_all), np.concatenate(ids_all)
        cand = np.concatenate(outs)
        merged = exact_topk(e_cat[cand], id_cat[cand], k)  # ids are positions here, so e_cat[cand] is the candidate's exact score
        assert np.array_equal(merged, exact_topk(e_cat, id_cat, k))
    assert certified_n > 100


def test_model_has_teeth_window_of_one_eps_is_not_enough():
    """Negative control: with a window of A_k + eps (instead of 2 eps) adversarial errors DO lose exact top-k rows, so
    the checks above would catch a kernel-side rule that is too tight."""
    rng = np.random.default_rng(3)
    misses = 0
    for trial in range(300):
        n, k, eps = 2000, 10, 0.2
        e = rng.normal(10, 1, n)
        ids = np.arange(n, dtype=np.int64)
        a = noisy(rng, e, eps, True, kth(e, k))
        a_k = np.sort(a)[k - 1]
        win = a <= a_k + eps
        if not np.array_equal(exact_topk(e[win], ids[win], k), exact_topk(e, ids, k)):
            misses += 1
    assert misses > 0


def test_capture_threshold_rule_failure_rate_and_cost():
    """tc_tau_with_margin (csrc/tc_scan.cu): T = tau when at least 3 sampled scores lie below tau - 2 eps, else T = tau + 2 eps.
    Monte Carlo on the headline shape (31 250 probed rows per query, 1 / 64 sampled, k = 10, 2 eps = 0.32 sigma of the score
    distribution): the rule must (a) almost never leave a query uncertified (A_k + 2 eps > T), while round 1's T = tau alone
    fails a few times per thousand queries, and (b) capture far fewer rows than the unconditional margin."""
    rng = np.random.default_rng(5)
    n, k, ratio, two_eps, trials = 31250, 10, 64, 0.32, 3000
    fail_rule = fail_tau = 0
    cap_rule = cap_tau = cap_margin = 0
    for _ in range(trials):
        a = rng.standard_normal(n)
        s = a[::ratio]  # the sampled rows (any fixed subset of iid rows)
        tau = np.partition(s, k - 1)[k - 1]
        a_k = np.partition(a, k - 1)[k - 1]
        c_lo = int((s <= tau - two_eps).sum())
        T = tau if c_lo >= 3 else tau + two_eps
        fail_rule += a_k + two_eps > T
        fail_tau += a_k + two_eps > tau
        cap_rule += int((a <= T).sum())
        cap_tau += int((a <= tau).sum())
        cap_margin += int((a <= tau + two_eps).sum())
    assert fail_rule / trials <= 1e-3, fail_rule
    assert fail_rule <= fail_tau
    assert cap_rule < 0.75 * cap_margin  # the conditional rule is much cheaper than "always add 2 eps"
    assert cap_rule < 2.2 * cap_tau       # ... and costs at most about twice the captures of the tightest threshold
