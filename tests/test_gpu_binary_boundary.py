"""The binary indexes at the boundary users call: the Hamming distance matrix (b200vs_calc_distance_binary) against the
binary oracle, and request coalescing of concurrent b200vs_search_binary callers on Binary Flat and Binary IVF-Flat."""
import threading

import numpy as np
import pytest

import b200vs
import binary_oracle as bo
from b200vs import BINARY_FLAT, BINARY_IVF_FLAT, HAMMING
from gpu_util import assert_same_results, require_gpu

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _gpu():
    require_gpu()


@pytest.mark.parametrize("nbytes", [1, 3, 8, 32, 100, 4096])
@pytest.mark.parametrize("nl,nr", [(1, 1), (257, 129), (0, 5), (5, 0)])
def test_calc_distance_binary_matches_oracle(nbytes, nl, nr):
    rng = np.random.default_rng(nbytes * 1000 + nl + nr)
    left = rng.integers(0, 256, (nl, nbytes), dtype=np.uint8)
    right = rng.integers(0, 256, (nr, nbytes), dtype=np.uint8)
    if nl and nr:
        right[0] = left[-1]  # a zero distance
    got = b200vs.calc_distance_binary(left, right)
    assert got.shape == (nl, nr) and got.dtype == np.float32
    assert np.array_equal(got, bo.hamming(left, right).astype(np.float32))


@pytest.mark.parametrize("nbytes", [3, 32, 4096])
def test_calc_distance_binary_tie_heavy(nbytes):
    rng = np.random.default_rng(nbytes)
    left = bo.tie_heavy(rng, 64, nbytes)
    right = bo.tie_heavy(rng, 96, nbytes)
    got = b200vs.calc_distance_binary(left, right)
    want = bo.hamming(left, right)
    assert np.array_equal(got, want.astype(np.float32))
    assert np.unique(want).size < want.size // 10  # many equal distances
    full = np.full((2, nbytes), 0xFF, np.uint8)
    assert np.array_equal(b200vs.calc_distance_binary(full, np.zeros((1, nbytes), np.uint8)), np.full((2, 1), nbytes * 8, np.float32))


def test_calc_distance_binary_refusals():
    L = b200vs.lib()
    u = np.zeros((2, 4), np.uint8)
    out = np.zeros((2, 2), np.float32)
    ill = b200vs.EILLEGAL_PARAMETERS
    for nbytes in (0, -1, 4097):  # checked first, even for an empty matrix
        assert L.b200vs_calc_distance_binary(0, nbytes, 2, u.ctypes.data, 2, u.ctypes.data, out.ctypes.data) == ill
        assert L.b200vs_calc_distance_binary(0, nbytes, 0, None, 0, None, None) == ill
    assert L.b200vs_calc_distance_binary(0, 4, 0, None, 2, u.ctypes.data, None) == b200vs.OK  # nothing to compute
    assert L.b200vs_calc_distance_binary(0, 4, 2, u.ctypes.data, 0, None, None) == b200vs.OK
    assert L.b200vs_calc_distance_binary(0, 4, 2, None, 2, u.ctypes.data, out.ctypes.data) == ill
    assert L.b200vs_calc_distance_binary(0, 4, -1, u.ctypes.data, 2, u.ctypes.data, out.ctypes.data) == ill
    with pytest.raises(ValueError):
        b200vs.calc_distance_binary(u, np.zeros((2, 5), np.uint8))


def make_index(itype, rng, n, dim, nlist=64):
    xb = bo.tie_heavy(rng, n, dim // 8, patterns=256, flips=12)
    ids = np.arange(1, n + 1, dtype=np.int64)
    if itype == "flat":
        ix = b200vs.Index(BINARY_FLAT, HAMMING, dim)
    else:
        ix = b200vs.Index(BINARY_IVF_FLAT, HAMMING, dim, nlist=nlist)
        ix.set_trained_state(b200vs.binary_ivf_state_blob(xb[rng.choice(n, nlist, replace=False)]))
    ix.add(xb, ids)
    return ix, xb


def run_threads(nthreads, fn):
    errs = []

    def wrap(t):
        try:
            fn(t)
        except Exception as e:  # noqa: BLE001
            errs.append(e)
    ths = [threading.Thread(target=wrap, args=(t,)) for t in range(nthreads)]
    for t in ths:
        t.start()
    for t in ths:
        t.join()
    assert not errs, errs


def lone_calls(ix, xq, k, **kw):
    """Results of one call per query with coalescing off."""
    ix.coalescing(0)
    D = np.zeros((xq.shape[0], k), np.float32)
    I = np.zeros((xq.shape[0], k), np.int64)
    for i in range(xq.shape[0]):
        d, l = ix.search(xq[i:i + 1], k, **kw)
        D[i], I[i] = d[0], l[0]
    ix.coalescing(1)
    return D, I


@pytest.mark.parametrize("itype", ["flat", "ivf"])
def test_concurrent_single_query_callers_are_coalesced(itype):
    """16 caller threads x nq = 1 (the reference's search pool): every caller gets exactly the answer of a lone call, and
    the library ran fewer batches than it served requests."""
    rng = np.random.default_rng(21)
    ix, xb = make_index(itype, rng, 200000, 256)
    nthreads, per, k = 16, 32, 10
    xq = np.concatenate([xb[rng.integers(0, xb.shape[0], nthreads * per // 2)],
                         bo.tie_heavy(rng, nthreads * per // 2, 32, patterns=256, flips=40)])
    kw = {} if itype == "flat" else {"nprobe": 8}
    Dw, Iw = lone_calls(ix, xq, k, **kw)
    b0, r0 = ix.coalescing()
    Dg, Ig = np.zeros_like(Dw), np.zeros_like(Iw)

    def worker(t):
        for j in range(per):
            i = t * per + j
            D, I = ix.search(xq[i:i + 1], k, **kw)
            Dg[i], Ig[i] = D[0], I[0]
    run_threads(nthreads, worker)
    assert_same_results(Dg, Ig, Dw, Iw)
    b1, r1 = ix.coalescing()
    assert r1 - r0 == nthreads * per
    assert b1 - b0 < r1 - r0, "concurrent callers were never merged into a shared batch"


@pytest.mark.parametrize("itype", ["flat", "ivf"])
def test_calls_with_different_k_or_nprobe_are_not_merged(itype):
    """Concurrent callers with four different (k, nprobe) settings: each gets the answer of a lone call with its own
    settings, which differ from one setting to the next."""
    rng = np.random.default_rng(22)
    ix, xb = make_index(itype, rng, 100000, 128)
    settings = [(5, 1), (10, 1), (5, 16), (10, 16)] if itype == "ivf" else [(5, 0), (10, 0), (7, 0), (12, 0)]
    nthreads, per = 16, 16
    xq = bo.tie_heavy(rng, nthreads * per, 16, patterns=256, flips=30)
    want = {}
    for k, nprobe in settings:
        want[(k, nprobe)] = lone_calls(ix, xq, k, nprobe=nprobe)
    if itype == "ivf":  # the nprobe values give different answers, so a merge across them would show
        assert not np.array_equal(want[(10, 1)][1], want[(10, 16)][1])
    got = {s: (np.zeros_like(w[0]), np.zeros_like(w[1])) for s, w in want.items()}

    def worker(t):
        k, nprobe = settings[t % len(settings)]
        for j in range(per):
            i = t * per + j
            D, I = ix.search(xq[i:i + 1], k, nprobe=nprobe)
            got[(k, nprobe)][0][i], got[(k, nprobe)][1][i] = D[0], I[0]
    run_threads(nthreads, worker)
    for t in range(nthreads):
        s = settings[t % len(settings)]
        rows = slice(t * per, (t + 1) * per)
        assert_same_results(got[s][0][rows], got[s][1][rows], want[s][0][rows], want[s][1][rows])


@pytest.mark.parametrize("itype", ["flat", "ivf"])
def test_id_list_filtered_calls_bypass_the_queue(itype):
    rng = np.random.default_rng(23)
    ix, xb = make_index(itype, rng, 50000, 64)
    ids = np.arange(1, xb.shape[0] + 1, dtype=np.int64)
    allow = np.sort(rng.choice(ids, 5000, replace=False))
    nthreads, per, k = 8, 8, 10
    xq = xb[rng.integers(0, xb.shape[0], nthreads * per)]
    kw = {} if itype == "flat" else {"nprobe": 64}
    b0, r0 = ix.coalescing()
    Dg = np.zeros((xq.shape[0], k), np.float32)
    Ig = np.zeros((xq.shape[0], k), np.int64)

    def worker(t):
        for j in range(per):
            i = t * per + j
            D, I = ix.search(xq[i:i + 1], k, sorted_ids=allow, **kw)
            Dg[i], Ig[i] = D[0], I[0]
    run_threads(nthreads, worker)
    assert ix.coalescing() == (b0, r0)  # no filtered call went through the coalescer
    Do, Io = bo.flat_search(xb, ids, xq, k, sorted_ids=allow)  # nprobe = nlist: the IVF answer is the Flat answer
    assert_same_results(Dg, Ig, Do, Io)
