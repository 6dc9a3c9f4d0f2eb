"""Tiny batches: the reference's own execution shape is ONE query per pool task (src/vector/vector_index.cc:54, :244-271).
  * flat_small_kernel: single-launch exact Flat search for nq < 16 (csrc/flat_small.cu) — bit-exact vs the oracle, ties included;
  * request coalescing: concurrent nq = 1 callers of b200vs_search share batches (csrc/api.cu)."""
import threading

import numpy as np
import pytest

import b200vs
import oracle_lib
from gpu_util import assert_same_results, require_gpu

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("metric,om", [(b200vs.L2, oracle_lib.L2), (b200vs.IP, oracle_lib.IP), (b200vs.COSINE, oracle_lib.COSINE)])
@pytest.mark.parametrize("n,d,k", [(100_000, 128, 10), (5000, 96, 1), (33_333, 100, 32), (20_000, 7, 10),
                                   (4096, 2048, 64)])
def test_flat_small_batches_match_oracle(oracle, metric, om, n, d, k):
    require_gpu()
    rng = np.random.default_rng(n + d)
    xb = rng.random((n, d)).astype(np.float32)
    ids = rng.permutation(np.arange(1, n + 1, dtype=np.int64))  # id order != row order: ties must follow ids
    ix = b200vs.Index(b200vs.FLAT, metric, d)
    for a in range(0, n, 32768):
        ix.add(xb[a:a + 32768], ids[a:a + 32768])
    xn = oracle.normalize_faiss(xb) if metric == b200vs.COSINE else xb
    for nq in (1, 2, 5, 15):
        xq = rng.random((nq, d)).astype(np.float32)
        qn = oracle.normalize_faiss(xq) if metric == b200vs.COSINE else xq
        D, I = ix.search(xq, k)
        Do, Io = oracle.flat_search(om, xn, ids, qn, k, nthreads=4)
        assert_same_results(D, I, Do, Io)
        De, Ie = ix.search(xq, k, exact_only=True)  # the general path
        assert_same_results(D, I, De, Ie)
    # filters and tombstones ride along
    xq = rng.random((3, d)).astype(np.float32)
    qn = oracle.normalize_faiss(xq) if metric == b200vs.COSINE else xq
    ix.delete(ids[:n // 3])
    D, I = ix.search(xq, k, id_range=(10, n // 2))
    Do, Io = oracle.flat_search(om, xn[n // 3:], ids[n // 3:], qn, k, nthreads=4, id_range=(10, n // 2))
    assert_same_results(D, I, Do, Io)


def test_flat_small_mass_duplicates(oracle):
    """Thousands of identical rows: the k-th key is shared by more rows than any rank-sort buffer holds; ids decide."""
    require_gpu()
    n, d, k = 20000, 64, 10
    rng = np.random.default_rng(1)
    xb = np.repeat(rng.random((4, d)).astype(np.float32), n // 4, axis=0)
    ids = rng.permutation(np.arange(1, n + 1, dtype=np.int64))
    ix = b200vs.Index(b200vs.FLAT, b200vs.L2, d)
    ix.add(xb, ids)
    xq = xb[[0, n // 2, n - 1]] + 0.001
    D, I = ix.search(xq, k)
    Do, Io = oracle.flat_search(oracle_lib.L2, xb, ids, xq, k, nthreads=2)
    assert_same_results(D, I, Do, Io)


@pytest.mark.parametrize("itype", ["flat", "ivf"])
def test_concurrent_single_query_callers_are_coalesced(oracle, itype):
    """16 caller threads x nq = 1 (the reference's search pool): every caller gets exactly the answer of a lone call, and
    the library ran fewer batches than it served requests."""
    require_gpu()
    n, d, k, nlist = 60000, 128, 10, 64
    rng = np.random.default_rng(3)
    xb = rng.random((n, d)).astype(np.float32)
    ids = np.arange(1, n + 1, dtype=np.int64)
    if itype == "flat":
        ix = b200vs.Index(b200vs.FLAT, b200vs.L2, d)
    else:
        ix = b200vs.Index(b200vs.IVF_FLAT, b200vs.L2, d, nlist=nlist)
        ix.set_trained_state(b200vs.ivf_state_blob(oracle.kmeans(oracle_lib.L2, xb[:nlist * 64], nlist, nthreads=8), b200vs.L2))
    ix.add(xb, ids)
    nthreads, per = 16, 24
    xq = rng.random((nthreads * per, d)).astype(np.float32)
    kw = {} if itype == "flat" else {"nprobe": 8}
    ix.coalescing(0)
    Dw, Iw = np.zeros((xq.shape[0], k), np.float32), np.zeros((xq.shape[0], k), np.int64)
    for i in range(xq.shape[0]):  # lone calls, coalescing off
        Dw[i], Iw[i] = (a[0] for a in ix.search(xq[i:i + 1], k, **kw))
    ix.coalescing(1)
    b0, r0 = ix.coalescing()
    Dg, Ig = np.zeros_like(Dw), np.zeros_like(Iw)
    errs = []

    def worker(t):
        try:
            for j in range(per):
                i = t * per + j
                D, I = ix.search(xq[i:i + 1], k, **kw)
                Dg[i], Ig[i] = D[0], I[0]
        except Exception as e:  # noqa: BLE001
            errs.append(e)
    ths = [threading.Thread(target=worker, args=(t,)) for t in range(nthreads)]
    for t in ths:
        t.start()
    for t in ths:
        t.join()
    assert not errs, errs
    assert_same_results(Dg, Ig, Dw, Iw)
    b1, r1 = ix.coalescing()
    assert r1 - r0 == nthreads * per
    assert b1 - b0 < r1 - r0, "concurrent callers were never merged into a shared batch"
    # a request with its own k / filter does not poison the others
    D, I = ix.search(xq[:3], 4, id_range=(1, 1000), **kw)
    assert I.shape == (3, 4) and (I[I >= 0] < 1000).all()
