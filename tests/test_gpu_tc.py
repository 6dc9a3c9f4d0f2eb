"""The tensor-core candidate pass (TMA + wgmma tile scan, tc_scan.cu) must return EXACTLY what the exact
FP32 scan returns (and therefore what the oracle returns): ids and distance bit patterns.  Large cases compare the
two CUDA paths with each other (size-independent property); small cases also go through the oracle."""
import numpy as np
import pytest

import b200vs
from b200vs import COSINE, FLAT, IP, IVF_FLAT, L2
from gpu_util import assert_same_results, require_gpu

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _gpu():
    require_gpu()


def tc_vs_exact(ix, xq, k, **kw):
    D1, I1 = ix.search(xq, k, **kw)
    st = ix.stats()
    D2, I2 = ix.search(xq, k, exact_only=True, **kw)
    assert st[1] == xq.shape[0], f"tensor-core pass was not used: stats {st}"
    assert ix.stats()[1] == 0
    assert_same_results(D1, I1, D2, I2)
    return D1, I1


@pytest.mark.parametrize("metric", [L2, IP, COSINE])
@pytest.mark.parametrize("n,d,nq,k", [(3000, 64, 16, 5), (20000, 128, 64, 10), (50000, 768, 100, 10), (9000, 96, 33, 100),
                                      (6000, 36, 17, 1)])
def test_flat_tc_equals_exact_and_oracle(oracle, metric, n, d, nq, k):
    rng = np.random.default_rng(n + d + k)
    xb = rng.random((n, d)).astype(np.float32)
    xq = rng.random((nq, d)).astype(np.float32)
    ids = np.arange(n, dtype=np.int64) * 3 + 5
    ix = b200vs.Index(FLAT, metric, d)
    ix.add(xb, ids)
    D, I = tc_vs_exact(ix, xq, k)
    if n <= 20000:
        stored = oracle.normalize_faiss(xb) if metric == COSINE else xb
        Do, Io = oracle.flat_search(metric, stored, ids, xq, k, nthreads=8)
        assert_same_results(D, I, Do, Io)


@pytest.mark.parametrize("metric", [L2, IP, COSINE])
@pytest.mark.parametrize("n,d,nlist,nprobe,nq,k", [(20000, 128, 64, 8, 64, 10), (60000, 768, 64, 8, 128, 10),
                                                   (30000, 256, 128, 128, 40, 20), (8000, 64, 16, 3, 200, 3)])
def test_ivfflat_tc_equals_exact(oracle, metric, n, d, nlist, nprobe, nq, k):
    rng = np.random.default_rng(n + d + nlist)
    xb = rng.random((n, d)).astype(np.float32)
    ids = np.arange(1, n + 1, dtype=np.int64)
    ix = b200vs.Index(IVF_FLAT, metric, d, nlist=nlist)
    ix.train(xb)
    for a in range(0, n, 7000):
        ix.add(xb[a:a + 7000], ids[a:a + 7000])
    xq = rng.random((nq, d)).astype(np.float32)
    D, I = tc_vs_exact(ix, xq, k, nprobe=nprobe)
    if n <= 30000:
        cent = ix.get_trained_state()[32:].view(np.float32).reshape(nlist, d)
        off, lx, _, lids = ix.export_lists(nlist)
        Do, Io = oracle.ivfflat_search(metric, cent, off, lx, lids, xq, k, nprobe, nthreads=8)
        assert_same_results(D, I, Do, Io)


def test_tc_with_filters_deletes_and_clustered_data(oracle):
    rng = np.random.default_rng(5)
    n, d, nlist = 40000, 128, 32
    centers = rng.random((200, d)).astype(np.float32)
    xb = (centers[rng.integers(0, 200, n)] + 0.02 * rng.standard_normal((n, d))).astype(np.float32)  # tight clusters: small gaps
    ids = np.arange(1, n + 1, dtype=np.int64)
    ix = b200vs.Index(IVF_FLAT, L2, d, nlist=nlist)
    ix.train(xb)
    ix.add(xb, ids)
    ix.delete(ids[::7])
    xq = (xb[rng.integers(0, n, 96)] + 0.01 * rng.standard_normal((96, d))).astype(np.float32)
    allow = np.sort(rng.choice(ids, 5000, replace=False))
    for kw in (dict(), dict(id_range=(1000, 30000)), dict(sorted_ids=allow), dict(sorted_ids=allow, negate=True)):
        tc_vs_exact(ix, xq, 10, nprobe=8, **kw)
    fl = b200vs.Index(FLAT, IP, d)
    fl.add(xb, ids)
    fl.delete(ids[5::11])
    for kw in (dict(), dict(id_range=(1000, 30000)), dict(sorted_ids=allow)):
        tc_vs_exact(fl, xq, 10, **kw)


def test_tc_duplicates_and_ties():
    # many exact duplicates: the window select must keep every tied row and order ties by id.  With 400 copies more rows
    # tie at the k-th score than the hybrid finish kernel holds, so the streaming finish kernel takes those queries.
    rng = np.random.default_rng(6)
    for nbase, copies in ((50, 40), (8, 400)):
        base = rng.random((nbase, 64)).astype(np.float32)
        xb = np.repeat(base, copies, axis=0)
        ids = rng.permutation(np.arange(1, xb.shape[0] + 1)).astype(np.int64)
        ix = b200vs.Index(FLAT, L2, 64)
        ix.add(xb, ids)
        xq = np.tile(base, (32 // nbase + 1, 1))[:32] + 0.001
        D, I = tc_vs_exact(ix, xq, 10)
        for row in I:
            assert list(row) == sorted(row)  # all 10 are the same duplicated vector -> ascending ids


def test_headline_shape_small(oracle):
    # the benchmark's shape at 1/10 scale: IVF-Flat L2 d=768, nprobe 32 of 128 lists, batch 256, top-10
    rng = np.random.default_rng(7)
    n, d, nlist = 100_000, 768, 128
    xb = rng.random((n, d), dtype=np.float32)
    ids = np.arange(1, n + 1, dtype=np.int64)
    ix = b200vs.Index(IVF_FLAT, L2, d, nlist=nlist)
    ix.train(xb[:32768])
    for a in range(0, n, 32768):
        ix.add(xb[a:a + 32768], ids[a:a + 32768])
    xq = rng.random((256, d), dtype=np.float32)
    D, I = tc_vs_exact(ix, xq, 10, nprobe=32)
    ix.set_profiling(True)
    ix.search(xq, 10, nprobe=32)
    st = ix.stats()
    ix.set_profiling(False)
    assert st[2] <= 2, f"too many queries fell back to the exact scan: {st}"
    cent = ix.get_trained_state()[32:].view(np.float32).reshape(nlist, d)
    off, lx, _, lids = ix.export_lists(nlist)
    Do, Io = oracle.ivfflat_search(L2, cent, off, lx, lids, xq[:64], 10, 32, nthreads=16)
    assert_same_results(D[:64], I[:64], Do, Io)


def test_sharded_rank_shape(oracle):
    """What one rank of a list-sharded deployment holds: all centroids, rows for a quarter of the lists only.  Identical
    to the exact scan and the oracle."""
    rng = np.random.default_rng(17)
    n, d, nlist, own = 120_000, 256, 128, 32
    xb = rng.random((n, d), dtype=np.float32)
    ids = np.arange(1, n + 1, dtype=np.int64)
    ix = b200vs.Index(IVF_FLAT, L2, d, nlist=nlist)
    ix.train(xb[:32768])
    cent = ix.get_trained_state()[32:].view(np.float32).reshape(nlist, d)
    asg = oracle.assign(L2, xb, cent, nthreads=16)
    keep = asg < own  # this "rank" owns lists [0, own)
    for a in range(0, n, 32768):
        m = keep[a:a + 32768]
        if m.any():
            ix.add(xb[a:a + 32768][m], ids[a:a + 32768][m])
    xq = rng.random((512, d), dtype=np.float32)
    off, lx, _, lids = ix.export_lists(nlist)
    assert off[own] == off[nlist]  # the other lists are empty here
    Do, Io = oracle.ivfflat_search(L2, cent, off, lx, lids, xq[:64], 10, 32, nthreads=16)
    D, I = tc_vs_exact(ix, xq, 10, nprobe=32)
    ix.set_profiling(True)
    ix.search(xq, 10, nprobe=32)
    st = ix.stats()
    ix.set_profiling(False)
    assert st[1] == 512
    assert_same_results(D[:64], I[:64], Do, Io)
