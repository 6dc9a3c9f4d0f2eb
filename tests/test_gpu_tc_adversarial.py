"""End-to-end parity of the tile path on data and shapes chosen to break it: decoys built to sit inside the finish
kernel's 2 eps window, forced certification failures, list lengths around every tile / box / chunk / span boundary, query
groups around 128 columns, wide k, large d and degenerate cosine data.  Every case compares the tile path with
exact_only=True (ids and distance bits) and, where the size allows, with the oracle, and asserts through stats() that
the route it means to exercise actually ran."""
import numpy as np
import pytest

import b200vs
import fp16_emu as H
import tf32_emu as E
from b200vs import COSINE, FLAT, IP, IVF_FLAT, L2
from gpu_util import assert_same_results, require_gpu

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _gpu():
    require_gpu()


def run_both(ix, xq, k, **kw):
    """Tile path (profiling on, so stats()[2] counts the re-run queries) and exact path: identical results.
    Returns (D, I, stats of the tile search)."""
    ix.set_profiling(True)
    D1, I1 = ix.search(xq, k, **kw)
    st = ix.stats()
    ix.set_profiling(False)
    D2, I2 = ix.search(xq, k, exact_only=True, **kw)
    assert ix.stats()[1] == 0
    assert_same_results(D1, I1, D2, I2)
    return D1, I1, st


def far_centroids(nlist, d, scale=1000.0):
    c = np.zeros((nlist, d), np.float32)
    for l in range(nlist):
        c[l, l % d] = scale * (1 + l // d)
    return c


# ---- decoys ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("k", [1, 10])
@pytest.mark.parametrize("metric", [L2, IP])
@pytest.mark.parametrize("index_type", [FLAT, IVF_FLAT])
def test_decoys(oracle, index_type, metric, k):
    """32 queries, each with its own (R, D) pair: D's exact distance lies just above R's, its approximate score far below.
    Index p holds pair p among filler rows; every index is searched with the whole batch and query p must return R as
    its k-th neighbour.  Each pair is built against the arithmetic that scans it: Flat scans TF32 rows (tf32_emu.decoy_*),
    IVF-Flat at d = 128 its FP16 mirror (fp16_emu.decoy_*).  The L2 and FP16 IP decoys use up more than half of the 2 eps
    window, so a kernel whose eps is half of what it claims returns D."""
    d, npair = 128, 32
    emu = E if index_type == FLAT else H
    gen = emu.decoy_l2 if metric == L2 else emu.decoy_ip
    pairs = [gen(np.random.default_rng(1000 * k + p), d, k, nfill=1500) for p in range(npair)]
    xq = np.concatenate([p[1] for p in pairs])
    for p in range(0, npair, 4):  # 8 of the 32 indexes: every query is still searched against 8 different indexes
        rows, _, r, dd = pairs[p]
        ids = np.arange(rows.shape[0], dtype=np.int64) * 7 + 3
        if index_type == FLAT:
            ix = b200vs.Index(FLAT, metric, d)
            kw = {}
        else:
            # centroid 0 = 0, the others far out on negative filler axes: every pair row (and, for L2, every row) lands
            # in list 0 behind filler rows, as in the Flat index.  The sample pass reads only the first rows of a list,
            # so it misses the pair rows; had it sampled R, the threshold rule would flag the query and re-run it exactly
            # (correct, but the window would not be tested).
            cent = np.zeros((4, d), np.float32)
            cent[1:, d // 2:d // 2 + 3] = -1000 * np.eye(3, dtype=np.float32)
            ix = b200vs.Index(IVF_FLAT, metric, d, nlist=4)
            ix.set_trained_state(b200vs.ivf_state_blob(cent, metric))
            kw = dict(nprobe=4)
        ix.add(rows, ids)
        D, I, st = run_both(ix, xq, k, **kw)
        assert st[1] == npair, st
        assert I[p, k - 1] == ids[r], f"pair {p}: the decoy displaced R (got id {I[p, k - 1]}, R {ids[r]}, D {ids[dd]})"
        # the decoy query itself is certified on the tile path (a batch of its copies: none is re-run exactly)
        _, Ic, stc = run_both(ix, np.repeat(xq[p:p + 1], 16, axis=0), k, **kw)
        assert stc[1] == 16 and stc[2] == 0, f"pair {p}: the decoy query fell back to the exact scan: stats {stc}"
        assert np.all(Ic[:, k - 1] == ids[r])
        if index_type == FLAT:
            Do, Io = oracle.flat_search(metric, rows, ids, xq, k, nthreads=8)
        else:
            cent = ix.get_trained_state()[32:].view(np.float32).reshape(4, d)
            off, lx, _, lids = ix.export_lists(4)
            Do, Io = oracle.ivfflat_search(metric, cent, off, lx, lids, xq, k, 4, nthreads=8)
        assert_same_results(D, I, Do, Io)
        ix.close()


# ---- forced fallback -------------------------------------------------------------------------------------------------
def test_capture_overflow_falls_back_for_every_query(oracle):
    """A large common offset: every row lies inside every query's window, n > the capture buffer (8192 for k <= 32), so
    every query overflows and is re-run on the exact scan."""
    rng = np.random.default_rng(11)
    n, d, nq = 20000, 64, 32
    xb = (1000 + 1e-3 * rng.random((n, d))).astype(np.float32)
    xq = (1000 + 1e-3 * rng.random((nq, d))).astype(np.float32)
    ids = np.arange(n, dtype=np.int64)
    ix = b200vs.Index(FLAT, L2, d)
    ix.add(xb, ids)
    D, I, st = run_both(ix, xq, 10)
    assert st[1] == nq and st[2] == nq, st
    Do, Io = oracle.flat_search(L2, xb, ids, xq, 10, nthreads=8)
    assert_same_results(D, I, Do, Io)


def test_mixed_batch_duplicates_fall_back_alone(oracle):
    """10 000 copies of one row plus random rows; half the queries sit on the duplicate, half are random.  The duplicate
    queries capture 10 000 tied rows each (more than the capture buffer, and more than a warp's hit staging holds, so the
    write-through runs) and are re-run exactly; the random queries stay certified.  Ties come back in ascending id order."""
    rng = np.random.default_rng(12)
    d, ndup, nrand = 64, 10000, 10000
    dup = np.full((1, d), 1.5, np.float32)
    xb = np.concatenate([np.repeat(dup, ndup, axis=0), rng.random((nrand, d), dtype=np.float32)])
    ids = rng.permutation(np.arange(5, 5 + xb.shape[0])).astype(np.int64)
    xq = np.concatenate([np.repeat(dup, 16, axis=0), rng.random((16, d), dtype=np.float32)])
    ix = b200vs.Index(FLAT, L2, d)
    ix.add(xb, ids)
    D, I, st = run_both(ix, xq, 10)
    assert st[1] == 32 and st[2] == 16, st
    dup_ids = np.sort(ids[:ndup])[:10]
    assert np.all(I[:16] == dup_ids[None, :]) and np.all(D[:16] == 0)
    Do, Io = oracle.flat_search(L2, xb, ids, xq, 10, nthreads=8)
    assert_same_results(D, I, Do, Io)


# ---- list-length edges -----------------------------------------------------------------------------------------------
LENGTHS = [0, 1, 31, 32, 33, 95, 96, 97, 127, 128, 129, 511, 512, 513, 2047, 2048, 2049, 2080, 4097]


def test_list_length_edges(oracle):
    """Hand-placed centroids fix every list's length exactly: around the 32-row boxes of a last tile, the 128-row tile,
    the 512-row chunk and the 2048-row sample span.  The longest list is added last, so it ends the arena.  Then a
    delete, and an add that outgrows (relocates) a list."""
    rng = np.random.default_rng(13)
    d, nlist = 64, len(LENGTHS)
    cent = far_centroids(nlist, d, 100.0)
    ix = b200vs.Index(IVF_FLAT, L2, d, nlist=nlist)
    ix.set_trained_state(b200vs.ivf_state_blob(cent, L2))
    next_id = [1]

    def rows_of(l, m):
        x = (cent[l] + rng.random((m, d))).astype(np.float32)
        i = np.arange(next_id[0], next_id[0] + m, dtype=np.int64)
        next_id[0] += m
        return x, i

    for l in np.argsort(LENGTHS, kind="stable"):
        if LENGTHS[l]:
            ix.add(*rows_of(l, LENGTHS[l]))
    qc = rng.integers(0, nlist, 96)
    xq = (cent[qc] + rng.random((96, d))).astype(np.float32)

    def check(expect_lengths):
        off, lx, _, lids = ix.export_lists(nlist)
        assert list(np.diff(off)) == expect_lengths
        for nprobe in (nlist, 3):
            D, I, st = run_both(ix, xq, 10, nprobe=nprobe)
            assert st[1] == 96, st
            Do, Io = oracle.ivfflat_search(L2, cent, off, lx, lids, xq, 10, nprobe, nthreads=8)
            assert_same_results(D, I, Do, Io)

    check(LENGTHS)
    _, lids = ix.export_list(LENGTHS.index(2049))
    ix.delete(lids[::3])
    lengths = list(LENGTHS)
    lengths[LENGTHS.index(2049)] -= len(lids[::3])
    check(lengths)
    grow = LENGTHS.index(32)
    ix.add(*rows_of(grow, 600))  # outgrows its slot: the list moves
    lengths[grow] += 600
    check(lengths)


@pytest.mark.parametrize("nq", [16, 127, 128, 129, 257])
def test_query_groups_of_one_list(nq):
    """Every query probes the same list: query groups of 128 columns, with a group of one query at 129 and 257."""
    rng = np.random.default_rng(nq)
    xb = rng.random((5000, 64), dtype=np.float32)
    ix = b200vs.Index(FLAT, L2, 64)
    ix.add(xb, np.arange(5000, dtype=np.int64))
    _, _, st = run_both(ix, rng.random((nq, 64), dtype=np.float32), 10)
    assert st[1] == nq


@pytest.mark.parametrize("k", [32, 33, 100, 128, 129])
def test_wide_k(oracle, k):
    """k up to 128 on the tile path with n >= 50 000, so the capture buffer size (which grows with k) matters; k = 129
    goes to the exact scan."""
    rng = np.random.default_rng(k)
    n, d = 50000, 32
    xb = rng.random((n, d), dtype=np.float32)
    ids = np.arange(n, dtype=np.int64)
    xq = rng.random((64, d), dtype=np.float32)
    ix = b200vs.Index(FLAT, IP, d)
    ix.add(xb, ids)
    D, I, st = run_both(ix, xq, k)
    assert st[1] == (64 if k <= 128 else 0), st
    Do, Io = oracle.flat_search(IP, xb, ids, xq[:8], k, nthreads=8)
    assert_same_results(D[:8], I[:8], Do, Io)


# ---- large d ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("d", [1536, 2048])
def test_large_d_ivf(d):
    rng = np.random.default_rng(d)
    xb = rng.standard_normal((20000, d)).astype(np.float32)
    ix = b200vs.Index(IVF_FLAT, L2, d, nlist=16)
    ix.set_trained_state(b200vs.ivf_state_blob(xb[:16], L2))
    ix.add(xb, np.arange(20000, dtype=np.int64))
    _, _, st = run_both(ix, rng.standard_normal((256, d)).astype(np.float32), 10, nprobe=4)
    assert st[1] == 256, st


def test_large_d_flat_and_coarse(oracle):
    rng = np.random.default_rng(4096)
    d = 4096
    xb = rng.random((8000, d), dtype=np.float32)
    ix = b200vs.Index(FLAT, IP, d)
    ix.add(xb, np.arange(8000, dtype=np.int64))
    _, _, st = run_both(ix, rng.random((64, d), dtype=np.float32), 10)
    assert st[1] == 64, st
    # 8192 centroids at d = 4096: the coarse pass's register select and streaming finish at their largest shape
    cent = rng.random((8192, d), dtype=np.float32)
    iv = b200vs.Index(IVF_FLAT, L2, d, nlist=8192)
    iv.set_trained_state(b200vs.ivf_state_blob(cent, L2))
    iv.add(xb, np.arange(8000, dtype=np.int64))
    xq = rng.random((64, d), dtype=np.float32)
    D, I, st = run_both(iv, xq, 10, nprobe=64)
    off, lx, _, lids = iv.export_lists(8192)
    Do, Io = oracle.ivfflat_search(L2, cent, off, lx, lids, xq[:16], 10, 64, nthreads=16)
    assert_same_results(D[:16], I[:16], Do, Io)


# ---- degenerate data -------------------------------------------------------------------------------------------------
def test_cosine_zero_rows_and_zero_query(oracle):
    rng = np.random.default_rng(21)
    n, d = 3000, 64
    xb = rng.random((n, d), dtype=np.float32)
    xb[::10] = 0
    ids = np.arange(n, dtype=np.int64)
    xq = rng.random((32, d), dtype=np.float32)
    xq[3] = 0
    ix = b200vs.Index(FLAT, COSINE, d)
    ix.add(xb, ids)
    Do, Io = oracle.flat_search(COSINE, oracle.normalize_faiss(xb), ids, xq, 10, nthreads=8)
    D, I, st = run_both(ix, xq, 10)
    assert st[1] == 32
    assert_same_results(D, I, Do, Io)
    Ds, Is = ix.search(xq[:4], 10)  # flat_small
    assert ix.stats()[1] == 0
    assert_same_results(Ds, Is, Do[:4], Io[:4])
