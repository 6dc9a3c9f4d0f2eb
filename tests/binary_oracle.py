"""CPU oracle of the binary indexes (Binary Flat / Binary IVF-Flat): a numpy restatement of faiss IndexBinaryFlat,
IndexBinaryIVF and IndexBinaryIVF::train as the engine serves them (DESIGN.md §6, binary tie rules).

Hamming distances are exact integers, so the restatement needs no evaluation order: popcount of XOR over the packed bytes.
Orders:
  - results by (distance, id);
  - probes by (distance, list id), which decides WHICH lists are probed when distances tie at the nprobe boundary;
  - add-time assignment: the nearest centroid, ties to the smaller list id.
Range search: IndexBinary::range_search takes an int radius (the float is truncated toward zero) and keeps dis < radius.
Upstream faiss does not pin these tie rules or the strict comparison (unpinned, like the other faiss internals of DESIGN §2).
Training: binary_to_real (bit i = byte i >> 3, bit i & 7, LSB first -> 2b - 1), the oracle's L2 k-means, real_to_binary
(bit set where the coordinate is > 0)."""
import numpy as np

import oracle_lib


def hamming(xq, xb):
    """int64 [nq, n] Hamming distances between packed uint8 rows."""
    xq, xb = np.ascontiguousarray(xq, np.uint8), np.ascontiguousarray(xb, np.uint8)
    out = np.zeros((xq.shape[0], xb.shape[0]), np.int64)
    for i in range(xq.shape[0]):
        out[i] = np.bitwise_count(xb ^ xq[i]).sum(axis=1, dtype=np.int64)
    return out


def _allowed(ids, id_range=None, sorted_ids=None, negate=False):
    ok = ids >= 0
    if id_range is not None:
        ok &= (ids >= id_range[0]) & (ids < id_range[1])
    if sorted_ids is not None:
        inside = np.isin(ids, np.asarray(sorted_ids, np.int64))
        ok &= ~inside if negate else inside
    return ok


def _select(dist, ids, k):
    """Top k of one query by (distance, id); -1 / 0 padded."""
    order = np.lexsort((ids, dist))[:k]
    D = np.zeros(k, np.float32)
    I = np.full(k, -1, np.int64)
    D[:order.size] = dist[order]
    I[:order.size] = ids[order]
    return D, I


def flat_search(xb, ids, xq, k, **filt):
    ids = np.asarray(ids, np.int64)
    ok = _allowed(ids, **filt)
    dist = hamming(xq, xb)
    out = [_select(dist[i][ok], ids[ok], k) for i in range(dist.shape[0])]
    return np.stack([o[0] for o in out]), np.stack([o[1] for o in out])


def probes(centroids, xq, nprobe):
    """[nq, nprobe] list ids: the nprobe nearest centroids by (distance, list id)."""
    dist = hamming(xq, centroids)
    lists = np.arange(centroids.shape[0], dtype=np.int64)
    return np.stack([np.lexsort((lists, d))[:nprobe] for d in dist])


def assign(x, centroids):
    """Nearest centroid of every row, ties to the smaller list id."""
    return np.argmin(hamming(x, centroids), axis=1)


def ivf_search(centroids, list_off, xb, ids, xq, k, nprobe, **filt):
    """xb / ids in list-major order with list l owning rows [list_off[l], list_off[l + 1])."""
    ids = np.asarray(ids, np.int64)
    nprobe = min(nprobe, centroids.shape[0])
    P = probes(centroids, xq, nprobe)
    ok = _allowed(ids, **filt)
    D = np.zeros((xq.shape[0], k), np.float32)
    I = np.full((xq.shape[0], k), -1, np.int64)
    for i in range(xq.shape[0]):
        rows = np.concatenate([np.arange(list_off[l], list_off[l + 1]) for l in P[i]]).astype(np.int64)
        rows = rows[ok[rows]]
        D[i], I[i] = _select(hamming(xq[i:i + 1], xb[rows])[0], ids[rows], k)
    return D, I


def range_search(xb, ids, xq, radius, max_results, candidates=None, **filt):
    """(D, I, C) with hits dis < int(radius), the closest max_results by (distance, id).  candidates: per-query row index
    arrays (IVF: the rows of the probed lists), default every row."""
    ids = np.asarray(ids, np.int64)
    r = int(radius)  # truncation toward zero, like the float -> int conversion in the plugin
    ok = _allowed(ids, **filt)
    nq = xq.shape[0]
    D = np.zeros((nq, max_results), np.float32)
    I = np.full((nq, max_results), -1, np.int64)
    C = np.zeros(nq, np.int32)
    for i in range(nq):
        rows = np.arange(xb.shape[0]) if candidates is None else np.asarray(candidates[i], np.int64)
        rows = rows[ok[rows]]
        d = hamming(xq[i:i + 1], xb[rows])[0]
        hit = d < r
        D[i], I[i] = _select(d[hit], ids[rows][hit], max_results)
        C[i] = min(int(hit.sum()), max_results)
    return D, I, C


def binary_to_real(x, dim):
    bits = np.unpackbits(np.ascontiguousarray(x, np.uint8), axis=1, bitorder="little")[:, :dim]
    return bits.astype(np.float32) * 2 - 1


def real_to_binary(c):
    return np.packbits(c > 0, axis=1, bitorder="little")


def kmeans(oracle, x, dim, k):
    """faiss IndexBinaryIVF::train restated: binary_to_real, L2 k-means (niter 10, seed 1234, <= 256 rows per centroid),
    real_to_binary."""
    return real_to_binary(oracle.kmeans(oracle_lib.L2, binary_to_real(x, dim), k))


def tie_heavy(rng, n, nb, patterns=4, flips=2):
    """Rows drawn from a few patterns with a few flipped bits each: the k-th distance falls inside a block of ties."""
    base = rng.integers(0, 256, (patterns, nb), dtype=np.uint8)
    x = base[rng.integers(0, patterns, n)].copy()
    for _ in range(flips):
        bit = rng.integers(0, nb * 8, n)
        x[np.arange(n), bit >> 3] ^= (1 << (bit & 7)).astype(np.uint8)
    return x
