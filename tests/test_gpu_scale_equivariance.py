"""Scaling every row and query by a power of two scales every exact FP32 operation exactly, as long as nothing leaves the
normal range.  Data drawn from [0.5, 1) and scaled by 2^+-20 keeps every difference, square and sum normal, so each
search path must return the same ids with L2 distances scaled by exactly 2^+-40 and cosine distances bit-identical.  IP
distances are reported as 1 - ip, which absorbs small ip values, so IP compares two large scales (2^12 and 2^20): there
1 - ip = -ip exactly.  A path that hides an absolute constant (a fixed epsilon, a clamp, a threshold) fails here; no
oracle is needed."""
import numpy as np
import pytest

import b200vs
from b200vs import COSINE, FLAT, HNSW, IP, IVF_FLAT, IVF_PQ, L2
from gpu_util import require_gpu

pytestmark = pytest.mark.gpu

N, D, NQ, K, NLIST, PQ_M = 4000, 64, 32, 10, 64, 8


@pytest.fixture(autouse=True)
def _gpu():
    require_gpu()


def scales(metric):
    """(base scale, other scales): distances at scale s equal those at the base scale times (s / base)^2."""
    return (2.0 ** 12, [2.0 ** 20]) if metric == IP else (1.0, [2.0 ** 20, 2.0 ** -20])


def searches(kind, metric, xb, xq, state):
    """{path name: (D, I)} of every search path of one index type, on data already scaled."""
    ids = np.arange(N, dtype=np.int64) + 1
    out = {}
    if kind == FLAT:
        ix = b200vs.Index(FLAT, metric, D)
        ix.add(xb, ids)
        out["tile"] = ix.search(xq, K)
        assert ix.stats()[1] == NQ
        out["flat_small"] = ix.search(xq[:4], K)
        assert ix.stats()[1] == 0
        out["exact"] = ix.search(xq, K, exact_only=True)
    elif kind == IVF_FLAT:
        ix = b200vs.Index(IVF_FLAT, metric, D, nlist=NLIST)
        ix.set_trained_state(b200vs.ivf_state_blob(state[0], metric))
        ix.add(xb, ids)
        out["tile"] = ix.search(xq, K, nprobe=8)
        assert ix.stats()[1] == NQ
        out["exact"] = ix.search(xq, K, nprobe=8, exact_only=True)
    elif kind == IVF_PQ:
        ix = b200vs.Index(IVF_PQ, metric, D, nlist=NLIST, pq_m=PQ_M, pq_nbits=8)
        ix.set_trained_state(b200vs.ivfpq_state_blob(state[0], state[1], metric))
        ix.add(xb, ids)
        out["pq"] = ix.search(xq, K, nprobe=8)
    else:
        ix = b200vs.Index(HNSW, metric, D, hnsw_m=16, hnsw_efc=100, max_elements=N)
        ix.add(xb, ids)
        out["hnsw"] = ix.search(xq, K, efsearch=64)
    ix.close()
    return out


@pytest.mark.parametrize("metric", [L2, IP, COSINE])
@pytest.mark.parametrize("kind", [FLAT, IVF_FLAT, IVF_PQ, HNSW])
def test_power_of_two_scaling(oracle, kind, metric):
    rng = np.random.default_rng(kind * 10 + metric)
    xb = (0.5 + 0.5 * rng.random((N, D))).astype(np.float32)
    xq = (0.5 + 0.5 * rng.random((NQ, D))).astype(np.float32)
    stored = oracle.normalize_faiss(xb) if metric == COSINE else xb
    state = None
    if kind in (IVF_FLAT, IVF_PQ):
        cent = oracle.kmeans(metric, stored, NLIST, niter=4)
        cb = oracle.pq_train(stored - cent[oracle.assign(metric, stored, cent)], PQ_M, niter=4) if kind == IVF_PQ else None
        state = (cent, cb)

    def scaled(s):
        f = np.float32(s)
        st = None
        if state is not None:  # cosine rows are normalised inside, so its trained state does not scale
            c = state[0] if metric == COSINE else state[0] * f
            cb = None if state[1] is None else (state[1] if metric == COSINE else state[1] * f)
            st = (c, cb)
        return searches(kind, metric, xb * f, xq * f, st)

    base, others = scales(metric)
    want = scaled(base)
    for s in others:
        got = scaled(s)
        for path, (Dw, Iw) in want.items():
            Dg, Ig = got[path]
            assert np.array_equal(Ig, Iw), f"{path}: ids differ at scale {s}"
            if metric == COSINE:
                assert np.array_equal(Dg.view(np.uint32), Dw.view(np.uint32)), f"{path}: cosine distances differ at scale {s}"
            else:
                f = np.float32((s / base) ** 2)
                assert np.array_equal(Dg.view(np.uint32), (Dw * f).view(np.uint32)), f"{path}: distances not scaled exactly at {s}"
