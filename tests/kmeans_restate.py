"""Training restated in numpy, to the bit: what `kmeans_gpu` (csrc/ivf_common.h) and the three training routines that call
it (IvfFlatIndex::train, IvfPqIndex::train, the binary IVF train) compute, so their trained state can be predicted on the
CPU.  Labels come from `oracle.assign` (the engine's certified tensor-core pass and its exact scan both equal it); the
rest is exact integer / IEEE arithmetic:

  - random streams: std::mt19937 (numpy's legacy RandomState seeds and steps the same generator);
  - subsample: the first k * max_pts rows of rand_perm(n, seed); initial centroids: the first k rows of
    rand_perm(m, seed + 1); m == k copies the sample;
  - sums: every value times scale = 2^(61 - ilogb(amax * m)), rounded half-even to int64, summed exactly;
  - mean: (float)((double)sum / scale) * (1.0f / (float)count); empty clusters keep their row until split;
  - faiss split_clusters with a fresh mt19937(1234) every iteration.

TEST INFRASTRUCTURE: imported only from tests/."""
import numpy as np

import b200vs
import binary_oracle as bo
from oracle_lib import COSINE, L2

SEED = 1234
MAX_PTS = 256
SPLIT_EPS = np.float32(1 / 1024.)


def mt19937(seed):
    """The std::mt19937(seed) generator; .random_raw(n) yields its next n outputs as uint64."""
    return np.random.RandomState(seed)._bit_generator


def rand_perm(m, seed):
    """kmeans_rand_perm / faiss rand_perm: i2 = i + mt() % (m - i), then swap, for i = 0 .. m - 2."""
    perm = list(range(m))
    if m > 1:
        raw = mt19937(seed).random_raw(m - 1)
        i = np.arange(m - 1, dtype=np.uint64)
        for a, b in enumerate((i + raw % (np.uint64(m) - i)).tolist()):
            perm[a], perm[b] = perm[b], perm[a]
    return np.array(perm, dtype=np.int64)


def fixed_point_scale(amax, m):
    """2^(61 - ilogb(amax * m)) (1.0 when amax is 0 or not finite): a sum of m values of magnitude <= amax stays < 2^62."""
    amax = float(np.float32(amax))
    if not (amax > 0 and np.isfinite(amax)):
        return 1.0
    return float(np.ldexp(1.0, 61 - (int(np.frexp(amax * float(m))[1]) - 1)))


def lloyd_update(x, labels, cent, scale):
    """One centroid update: fixed-point sums of each cluster's rows, then the two-rounding mean.  Returns the new
    centroids (empty clusters keep their row of `cent`) and the float32 counts split_clusters starts from."""
    k = cent.shape[0]
    labels = np.asarray(labels, np.int64)
    counts = np.bincount(labels, minlength=k)
    q = np.rint(np.asarray(x, np.float32).astype(np.float64) * scale).astype(np.int64)
    order = np.argsort(labels, kind="stable")
    nz = np.flatnonzero(counts)
    starts = np.concatenate([[0], np.cumsum(counts)[:-1]])
    sums = np.add.reduceat(q[order], starts[nz], axis=0)  # exact int64 (|sum| < 2^62)
    out = cent.copy()
    inv = np.float32(1) / counts[nz].astype(np.float32)
    out[nz] = (sums.astype(np.float64) / scale).astype(np.float32) * inv[:, None]
    return out, counts.astype(np.float32)


def split_clusters(cent, hassign, m):
    """faiss split_clusters: every empty cluster copies a big one chosen with probability (count - 1) / (m - k), the
    copies drift apart by (1 +- 2^-10) on alternating coordinates, and the count is halved between them."""
    k, d = cent.shape
    rng = mt19937(SEED)
    raw, used = rng.random_raw(1024), 0
    one, denom, top = np.float32(1), np.float32(m - k), np.float32(4294967295)
    up = np.where(np.arange(d) % 2 == 0, one + SPLIT_EPS, one - SPLIT_EPS).astype(np.float32)
    down = np.where(np.arange(d) % 2 == 0, one - SPLIT_EPS, one + SPLIT_EPS).astype(np.float32)
    for ci in range(k):
        if hassign[ci] != 0:
            continue
        cj = 0
        while True:
            if used == raw.size:
                raw, used = rng.random_raw(1024), 0
            p = np.float32(hassign[cj] - one) / denom
            r = np.float32(raw[used]) / top
            used += 1
            if r < p:
                break
            cj = (cj + 1) % k
        cent[ci] = cent[cj] * up
        cent[cj] = cent[cj] * down
        hassign[ci] = hassign[cj] / np.float32(2)
        hassign[cj] = hassign[cj] - hassign[ci]
    return cent


def kmeans(oracle, metric, x, k, niter=10, max_pts=MAX_PTS, seed=SEED, nthreads=8, empty_per_iter=None):
    """kmeans_gpu: [k, d] float32 centroids of the RAW rows x (cosine rows are normalised after the subsample).
    empty_per_iter: a list that receives the number of empty clusters of every iteration."""
    x = np.ascontiguousarray(x, np.float32)
    n = x.shape[0]
    if n > k * max_pts:
        x = x[rand_perm(n, seed)[:k * max_pts]]
    m = x.shape[0]
    if metric == COSINE:
        x = oracle.normalize_faiss(x)
    if m == k:
        return x.copy()
    cent = x[rand_perm(m, seed + 1)[:k]].copy()
    scale = fixed_point_scale(np.abs(x).max(), m)
    for _ in range(niter):
        labels = oracle.assign(metric, x, cent, nthreads=nthreads)
        cent, hassign = lloyd_update(x, labels, cent, scale)
        if empty_per_iter is not None:
            empty_per_iter.append(int((hassign == 0).sum()))
        cent = split_clusters(cent, hassign, m)
    return cent


def pq_train(oracle, x, M, nbits, niter=25, nthreads=8):
    """[M, 2^nbits, d / M] codebooks: one L2 k-means per sub-space of x."""
    x = np.ascontiguousarray(x, np.float32)
    dsub = x.shape[1] // M
    return np.stack([kmeans(oracle, L2, x[:, j * dsub:(j + 1) * dsub], 1 << nbits, niter=niter, nthreads=nthreads)
                     for j in range(M)])


def train_ivf_flat(oracle, metric, x, nlist, nthreads=8):
    """IvfFlatIndex::train: the trained-state blob.  Fewer rows than nlist train one centroid."""
    k = 1 if x.shape[0] < nlist else nlist
    return b200vs.ivf_state_blob(kmeans(oracle, metric, x, k, nthreads=nthreads), metric)


def train_ivf_pq(oracle, metric, x, nlist, M, nbits, nthreads=8):
    """IvfPqIndex::train: the trained-state blob, empty when the index falls back to an inner Flat index (fewer than
    max(256 * nlist, 256 * 2^nbits) rows)."""
    x = np.ascontiguousarray(x, np.float32)
    n, ksub = x.shape[0], 1 << nbits
    if n < max(256 * nlist, 256 * ksub):
        return np.zeros(0, np.uint8)
    cent = kmeans(oracle, metric, x, nlist, nthreads=nthreads)
    m = min(n, 256 * ksub)
    sub = x[rand_perm(n, SEED)[:m]] if m < n else x.copy()
    if metric == COSINE:
        sub = oracle.normalize_faiss(sub)
    res = sub - cent[oracle.assign(metric, sub, cent, nthreads=nthreads)]
    return b200vs.ivfpq_state_blob(cent, pq_train(oracle, res, M, nbits, nthreads=nthreads), metric)


def train_binary(oracle, x, dim, nlist, nthreads=8):
    """Binary IVF train: subsample the packed rows, expand to +-1 (LSB first), L2 k-means, bit set where > 0."""
    x = np.ascontiguousarray(x, np.uint8)
    n = x.shape[0]
    k = 1 if n < nlist else nlist
    if n > k * MAX_PTS:
        x = x[rand_perm(n, SEED)[:k * MAX_PTS]]
    return b200vs.binary_ivf_state_blob(bo.real_to_binary(kmeans(oracle, L2, bo.binary_to_real(x, dim), k, nthreads=nthreads)))
