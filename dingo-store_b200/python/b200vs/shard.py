"""Host-side logic of the list-sharded multi-GPU search (SURVEY.md §8e): which rank owns which inverted list,
how rows travel to their owner at build time, and the merge rule of the per-shard top-k (the CUDA merge kernel
b200vs_merge_topk_device implements the same rule on the device; the numpy form here is what the CPU `gloo`
tests check the collective plumbing against).  Mirrors VectorIndexWrapper::MergeSearchResults
(src/vector/vector_index.cc:1056-1108): ascending distance, then smaller id, truncate to k."""
import numpy as np


def list_owner(list_ids, nlist_per_rank):
    """Contiguous blocks of lists per rank (equivalently: Raft regions -> GPUs)."""
    return np.asarray(list_ids, dtype=np.int64) // int(nlist_per_rank)


def split_rows_by_owner(list_ids, nlist_per_rank, world):
    """Returns (order, counts): rows sorted by owner rank (stable) and rows per rank — the all_to_all send plan."""
    owner = list_owner(list_ids, nlist_per_rank)
    order = np.argsort(owner, kind="stable")
    counts = np.bincount(owner, minlength=world).astype(np.int64)
    return order, counts


def row_owner(ids, world):
    """Owner rank of each id of a row-sharded FLAT / HNSW index: splitmix64's finalizer of the id read as a uint64, mod world
    (the rule b200vs_row_owner and the device routing apply)."""
    z = np.asarray(ids, dtype=np.int64).view(np.uint64).copy()
    with np.errstate(over="ignore"):
        z ^= z >> np.uint64(30)
        z *= np.uint64(0xbf58476d1ce4e5b9)
        z ^= z >> np.uint64(27)
        z *= np.uint64(0x94d049bb133111eb)
        z ^= z >> np.uint64(31)
    return (z % np.uint64(world)).astype(np.int32)


def merge_topk(parts_dist, parts_ids, k):
    """parts_*: [nparts, nq, k] API-semantics distances ascending, id -1 padded -> merged [nq, k]."""
    parts_dist = np.asarray(parts_dist, dtype=np.float32)
    parts_ids = np.asarray(parts_ids, dtype=np.int64)
    nparts, nq, kk = parts_dist.shape
    d = np.transpose(parts_dist, (1, 0, 2)).reshape(nq, nparts * kk)
    i = np.transpose(parts_ids, (1, 0, 2)).reshape(nq, nparts * kk)
    out_d = np.zeros((nq, k), np.float32)
    out_i = np.full((nq, k), -1, np.int64)
    for q in range(nq):
        valid = i[q] >= 0
        dv, iv = d[q][valid], i[q][valid]
        order = np.lexsort((iv, dv))[:k]
        out_d[q, :len(order)] = dv[order]
        out_i[q, :len(order)] = iv[order]
    return out_d, out_i
