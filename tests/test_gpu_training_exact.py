"""GPU training pinned to the bit: every trained state (`get_trained_state()`) equals the blob that the numpy restatement
of the training rule (tests/kmeans_restate.py) predicts, byte for byte.  Covers IVF-Flat at shapes that reach every
assignment branch of kmeans_gpu (tensor-core coarse pass, exact scan, chunk tail, subsample, copy, one centroid),
adversarial data, the composed IVF-PQ training at nbits 1-8 and the binary IVF training.  With integer-valued data (and
for any binary data, whose +-1 rows have integer sums) the engine must also equal the oracle's faiss::Clustering
restatement, which checks it independently of tests/kmeans_restate.py."""
import numpy as np
import pytest

import b200vs
import binary_oracle as bo
import kmeans_restate as kr
from b200vs import BINARY_IVF_FLAT, FLAT, HAMMING, IVF_FLAT, IVF_PQ
from gpu_util import require_gpu
from oracle_lib import COSINE, IP, L2

pytestmark = pytest.mark.gpu

METRICS = {"l2": L2, "ip": IP, "cosine": COSINE}


@pytest.fixture(autouse=True)
def _gpu():
    require_gpu()


def assert_blob_equal(got, want, header, sections):
    """Byte equality of two trained-state blobs; on a mismatch name the first differing entry.  sections: the arrays after
    the `header` bytes, as (name, shape, dtype)."""
    got, want = np.asarray(got, np.uint8), np.asarray(want, np.uint8)
    assert got.size == want.size, f"blob sizes differ: engine {got.size} B, restated {want.size} B"
    diff = np.flatnonzero(got != want)
    if diff.size == 0:
        return
    pos = int(diff[0])
    assert pos >= header, f"headers differ: engine {got[:header].view(np.int64)}, restated {want[:header].view(np.int64)}"
    pos -= header
    base = header
    for name, shape, dt in sections:
        isz = np.dtype(dt).itemsize
        nbytes = int(np.prod(shape)) * isz
        if pos < nbytes:
            g = got[base:base + nbytes].view(dt).reshape(shape)
            w = want[base:base + nbytes].view(dt).reshape(shape)
            idx = np.unravel_index(pos // isz, shape)
            pytest.fail(f"first difference at {name}{list(map(int, idx))}: engine {g[idx].item()!r}, restated "
                        f"{w[idx].item()!r} ({int((g != w).sum())} of {g.size} values differ)")
        pos -= nbytes
        base += nbytes


def assert_ivf_blob_equal(got, want, k, d):
    assert_blob_equal(got, want, 32, [("centroid", (k, d), np.float32)])


def assert_pq_blob_equal(got, want, nlist, d, M, nbits):
    assert_blob_equal(got, want, 48, [("centroid", (nlist, d), np.float32),
                                      ("codebook", (M, 1 << nbits, d // M), np.float32)])


def assert_binary_blob_equal(got, want, k, dim):
    assert_blob_equal(got, want, 32, [("centroid byte", (k, dim // 8), np.uint8)])


def clustered(rng, n, d, centers=50, noise=0.5):
    c = rng.standard_normal((centers, d)) * 2
    return (c[rng.integers(0, centers, n)] + noise * rng.standard_normal((n, d))).astype(np.float32)


def engine_ivf_flat(metric, x, nlist):
    ix = b200vs.Index(IVF_FLAT, metric, x.shape[1], nlist=nlist)
    ix.train(x)
    blob = ix.get_trained_state()
    ix.close()
    return blob


def check_ivf_flat(oracle, metric, x, nlist):
    k = 1 if x.shape[0] < nlist else nlist
    got = engine_ivf_flat(metric, x, nlist)
    assert_ivf_blob_equal(got, kr.train_ivf_flat(oracle, metric, x, nlist), k, x.shape[1])
    return got


# n, d, nlist: the branch of kmeans_gpu each shape reaches
IVF_FLAT_SHAPES = {
    "tc_d96": (12000, 96, 64),          # tensor-core coarse pass (d % 4 == 0, d >= 32, >= 64 centroids)
    "scan_d30": (5000, 30, 32),         # d % 4 != 0: exact scan
    "scan_d16": (5000, 16, 32),         # d < 32: exact scan
    "chunk_tail": (32773, 32, 200),     # one 32768-row TC chunk + a 5-row tail (< 16 rows) through the exact scan
    "subsample": (20000, 32, 64),       # n > 256 * nlist: the first 16384 rows of perm(n, 1234)
    "n_eq_nlist": (64, 32, 64),         # the sample is copied
    "n_lt_nlist": (40, 32, 64),         # one centroid
}


@pytest.mark.parametrize("metric", sorted(METRICS))
@pytest.mark.parametrize("shape", list(IVF_FLAT_SHAPES))
def test_ivf_flat_equals_restatement(oracle, shape, metric):
    n, d, nlist = IVF_FLAT_SHAPES[shape]
    x = clustered(np.random.default_rng(n + d), n, d)
    check_ivf_flat(oracle, METRICS[metric], x, nlist)


def adversarial(kind, rng, n, d):
    if kind == "few_distinct":  # 5 distinct rows: duplicated initial centroids, tied labels, empty clusters
        return rng.standard_normal((5, d)).astype(np.float32)[rng.integers(0, 5, n)]
    x = clustered(rng, n, d)
    if kind == "scale_1e17":  # about the largest scale at which these rows' squared distances stay finite (at 1e30
        # every one is +inf, and no nearest centroid is defined)
        return (x * np.float32(1e17)).astype(np.float32)
    if kind == "scale_1e-30":  # products underflow: distances and inner products tie at or near zero
        return (x * np.float32(1e-30)).astype(np.float32)
    if kind == "mixed_signs":  # every row next to its negation
        return np.concatenate([x[:n // 2], -x[:n // 2]])
    if kind == "constant_column":
        x[:, 3] = np.float32(7.25)
        x[:, 10] = np.float32(-3.0)
        return x
    if kind == "heterogeneous":  # columns near 1e4 next to columns near 1e-6
        col = np.where(np.arange(d) % 3 == 0, 1e4, np.where(np.arange(d) % 3 == 1, 1e-6, 1.0))
        return (x * col).astype(np.float32)
    raise ValueError(kind)


@pytest.mark.parametrize("metric", ["l2", "ip"])
@pytest.mark.parametrize("d", [32, 30])
@pytest.mark.parametrize("kind", ["few_distinct", "scale_1e17", "scale_1e-30", "mixed_signs", "constant_column",
                                  "heterogeneous"])
def test_ivf_flat_adversarial_equals_restatement(oracle, kind, d, metric):
    """d = 32 labels through the tensor-core pass, d = 30 through the exact scan."""
    x = adversarial(kind, np.random.default_rng(7), 8000, d)
    check_ivf_flat(oracle, METRICS[metric], x, 64)


def test_ivf_flat_few_distinct_rows_split_clusters(oracle):
    """The few-distinct-rows data really leaves clusters empty, so split_clusters shapes the pinned state."""
    x = adversarial("few_distinct", np.random.default_rng(7), 8000, 32)
    empty = []
    kr.kmeans(oracle, L2, x, 64, empty_per_iter=empty)
    assert min(empty) > 0, empty


@pytest.mark.parametrize("metric", ["l2", "ip"])
@pytest.mark.parametrize("d", [32, 30])
def test_ivf_flat_integer_data_equals_oracle_kmeans(oracle, metric, d):
    """Integer-valued rows: exact sums on both sides, so the engine equals faiss::Clustering restated with float sums."""
    rng = np.random.default_rng(23)
    x = rng.integers(-8, 9, (12000, d)).astype(np.float32)
    got = check_ivf_flat(oracle, METRICS[metric], x, 64)
    want = b200vs.ivf_state_blob(oracle.kmeans(METRICS[metric], x, 64, nthreads=8), METRICS[metric])
    assert_ivf_blob_equal(got, want, 64, d)


def engine_ivf_pq(metric, x, nlist, M, nbits):
    ix = b200vs.Index(IVF_PQ, metric, x.shape[1], nlist=nlist, pq_m=M, pq_nbits=nbits)
    ix.train(x)
    blob, sub = ix.get_trained_state(), ix.sub_type()
    ix.close()
    return blob, sub


# n, d, nlist, M, nbits
IVF_PQ_CASES = {
    "nbits8": (70000, 32, 16, 8, 8),        # n > 256 * ksub: the PQ subsample (and the coarse one)
    "nbits4_dsub2": (5000, 32, 16, 16, 4),
    "nbits4_dsub1": (5000, 32, 16, 32, 4),
    "nbits1": (3000, 32, 8, 8, 1),
    "nbits7": (40000, 32, 16, 8, 7),
    "threshold": (4096, 32, 16, 8, 4),      # exactly max(256 * nlist, 256 * ksub): IVF-PQ, neither sample subsampled
}


@pytest.mark.parametrize("case,metric", [("nbits8", "l2"), ("nbits8", "ip"), ("nbits8", "cosine"), ("nbits4_dsub2", "l2"),
                                         ("nbits4_dsub2", "ip"), ("nbits4_dsub1", "l2"), ("nbits1", "l2"),
                                         ("nbits7", "cosine"), ("threshold", "l2"), ("threshold", "cosine")])
def test_ivf_pq_equals_restatement(oracle, case, metric):
    n, d, nlist, M, nbits = IVF_PQ_CASES[case]
    x = clustered(np.random.default_rng(n + M + nbits), n, d)
    got, sub = engine_ivf_pq(METRICS[metric], x, nlist, M, nbits)
    assert sub == IVF_PQ
    assert_pq_blob_equal(got, kr.train_ivf_pq(oracle, METRICS[metric], x, nlist, M, nbits), nlist, d, M, nbits)


def test_ivf_pq_below_threshold_is_flat(oracle):
    """One row fewer than the threshold: an inner Flat index, no trained state on either side."""
    n, d, nlist, M, nbits = IVF_PQ_CASES["threshold"]
    x = clustered(np.random.default_rng(1), n - 1, d)
    got, sub = engine_ivf_pq(L2, x, nlist, M, nbits)
    assert sub == FLAT and got.size == 0
    assert kr.train_ivf_pq(oracle, L2, x, nlist, M, nbits).size == 0


def engine_binary(x, dim, nlist):
    ix = b200vs.Index(BINARY_IVF_FLAT, HAMMING, dim, nlist=nlist)
    ix.train(x)
    blob = ix.get_trained_state()
    ix.close()
    return blob


# n, dim, nlist, data
BINARY_CASES = {
    "dim8": (3000, 8, 16, "random"),
    "dim64": (3000, 64, 16, "random"),
    "dim256": (3000, 256, 16, "random"),
    "dim1000": (3000, 1000, 16, "random"),
    "subsample": (5000, 64, 8, "random"),      # n > 256 * nlist
    "n_eq_nlist": (16, 64, 16, "random"),
    "n_lt_nlist": (10, 64, 16, "random"),
    "tie_heavy": (20000, 128, 32, "tie_heavy"),
}


@pytest.mark.parametrize("case", list(BINARY_CASES))
def test_binary_ivf_equals_restatement_and_oracle(oracle, case):
    n, dim, nlist, data = BINARY_CASES[case]
    rng = np.random.default_rng(n + dim)
    nb = dim // 8
    x = rng.integers(0, 256, (n, nb), dtype=np.uint8) if data == "random" else bo.tie_heavy(rng, n, nb, patterns=64, flips=10)
    k = 1 if n < nlist else nlist
    got = engine_binary(x, dim, nlist)
    assert_binary_blob_equal(got, kr.train_binary(oracle, x, dim, nlist), k, dim)
    # +-1 rows have integer sums: the engine also equals faiss::Clustering restated with float sums
    assert_binary_blob_equal(got, b200vs.binary_ivf_state_blob(bo.kmeans(oracle, x, dim, k)), k, dim)
