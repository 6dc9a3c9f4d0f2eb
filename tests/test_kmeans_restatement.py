"""The training restatement (tests/kmeans_restate.py) checked on the CPU, before it is used to pin the GPU training.

On integer-valued data every sum is exact both in float32 and in 64-bit fixed point, so the restatement must equal the
oracle's faiss::Clustering restatement (float sums in point order) bit for bit: that pins the random streams, the
subsample, the initialisation, the mean's roundings and split_clusters.  On float data the fixed-point sums differ from
faiss's float sums, so there the restated update is held to the float64 mean within the fixed-point quantum."""
import numpy as np
import pytest

import kmeans_restate as kr
from oracle_lib import IP, L2


def int_rows(rng, n, d):
    return rng.integers(-8, 9, (n, d)).astype(np.float32)


def test_mt19937_stream():
    # std::mt19937 [rand.predef]: the 10000th output of a default-constructed generator (seed 5489) is 4123659995
    assert int(kr.mt19937(5489).random_raw(10000)[-1]) == 4123659995
    assert kr.mt19937(1234).random_raw(2).tolist() == [822569775, 2137449171]


def test_rand_perm_is_a_permutation():
    for m in (1, 2, 7, 1000):
        p = kr.rand_perm(m, 1234)
        assert np.array_equal(np.sort(p), np.arange(m))
    assert not np.array_equal(kr.rand_perm(1000, 1234), kr.rand_perm(1000, 1235))


def test_fixed_point_scale():
    assert kr.fixed_point_scale(8.0, 4096) == 2.0 ** (61 - 15)  # 8 * 4096 = 2^15
    assert kr.fixed_point_scale(9.0, 4096) == 2.0 ** (61 - 15)  # ilogb rounds down
    assert kr.fixed_point_scale(0.0, 10) == 1.0 and kr.fixed_point_scale(np.inf, 10) == 1.0
    assert kr.fixed_point_scale(1e-30, 100) == 2.0 ** (61 - np.frexp(1e-30 * 100)[1] + 1)


CASES = {  # n, d, k, seed
    "plain": (3000, 16, 20, 1),
    "subsample": (6000, 8, 16, 2),  # 6000 > 16 * 256
    "n_eq_k": (32, 8, 32, 3),
}


@pytest.mark.parametrize("metric", [L2, IP])
@pytest.mark.parametrize("case", sorted(CASES))
def test_integer_data_equals_oracle_kmeans(oracle, metric, case):
    n, d, k, seed = CASES[case]
    x = int_rows(np.random.default_rng(seed), n, d)
    got = kr.kmeans(oracle, metric, x, k)
    want = oracle.kmeans(metric, x, k, nthreads=8)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))


@pytest.mark.parametrize("metric", [L2, IP])
def test_integer_data_empty_clusters_equal_oracle_kmeans(oracle, metric):
    """Few distinct rows: the initial centroids repeat rows, labels tie, clusters go empty and split_clusters runs."""
    rng = np.random.default_rng(5)
    x = int_rows(rng, 6, 12)[rng.integers(0, 6, 2000)]
    empty = []
    got = kr.kmeans(oracle, metric, x, 24, empty_per_iter=empty)
    assert sum(e > 0 for e in empty) >= 3, empty
    want = oracle.kmeans(metric, x, 24, nthreads=8)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))


@pytest.mark.parametrize("nbits,M,n", [(1, 4, 1000), (4, 4, 5000), (8, 2, 70000)])
def test_integer_data_equals_oracle_pq_train(oracle, nbits, M, n):
    """Sub-quantisers (25 iterations, L2, one k-means per sub-space); each n exceeds 256 * 2^nbits: subsampled."""
    x = int_rows(np.random.default_rng(nbits), n, 8)
    got = kr.pq_train(oracle, x, M, nbits)
    want = oracle.pq_train(x, M, nbits=nbits, nthreads=8)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))


def heterogeneous_rows(rng, n, d):
    """Columns near 1e4 next to columns near 1e-6, mixed signs."""
    col = np.where(np.arange(d) % 3 == 0, 1e4, np.where(np.arange(d) % 3 == 1, 1e-6, 1.0))
    return (rng.standard_normal((n, d)) * col).astype(np.float32)


@pytest.mark.parametrize("data", ["normal", "heterogeneous"])
@pytest.mark.parametrize("metric", [L2, IP])
def test_lloyd_update_within_fixed_point_bound(oracle, data, metric):
    """One restated update from given centroids: every coordinate is within 0.5 / scale + 2 ulp32 of the float64 mean of
    its rows (the fixed-point quantum is absolute, amax * m * 2^-61 at most, the same for every coordinate)."""
    rng = np.random.default_rng(17)
    n, d, k = 20000, 24, 40
    x = rng.standard_normal((n, d)).astype(np.float32) if data == "normal" else heterogeneous_rows(rng, n, d)
    cent = x[rng.choice(n, k, replace=False)].copy()
    labels = oracle.assign(metric, x, cent, nthreads=8).astype(np.int64)
    scale = kr.fixed_point_scale(np.abs(x).max(), n)
    got, counts = kr.lloyd_update(x, labels, cent, scale)
    sums = np.zeros((k, d), np.float64)
    np.add.at(sums, labels, x.astype(np.float64))
    live = counts > 0
    mean = sums[live] / counts[live, None].astype(np.float64)
    err = np.abs(got[live].astype(np.float64) - mean)
    bound = 0.5 / scale + 2 * np.spacing(np.abs(got[live]))
    assert (err <= bound).all(), float((err / bound).max())
    assert np.array_equal(got[~live], cent[~live])
