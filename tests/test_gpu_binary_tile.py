"""Binary Flat and Binary IVF-Flat batched search on the BMMA tile scan (binary_tile.cu): ids AND distances bit-equal to
tests/binary_oracle.py and to the same index searched with exact_only, and the path each call takes (stats[1] = queries
served by the tile scan, stats[2] = queries re-run on the exact scan, both with profiling on)."""
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


def big_ids(rng, n):
    return rng.choice(np.iinfo(np.int64).max - 1, size=n, replace=False).astype(np.int64)


def tile_eligible(nq, cand, k):
    """The dispatch rule of bt_eligible: cand = candidate rows per query (Flat: rows incl. tombstones; IVF: rows x
    nprobe / nlist)."""
    return nq >= 16 and k <= 128 and cand >= 256 * k and nq * cand >= 2 ** 23 * max(1.0, k / 32)


def search_checked(ix, xq, k, Do=None, Io=None, sub=None, tile=None, **kw):
    """Search with profiling on; equal to exact_only on every query and to the oracle (Do, Io) on the queries `sub`;
    stats[1] = nq when `tile`, 0 when not, either when None.  Returns (D, I, stats)."""
    nq = xq.shape[0]
    ix.set_profiling(True)
    D, I = ix.search(xq, k, **kw)
    st = ix.stats()
    ix.set_profiling(False)
    De, Ie = ix.search(xq, k, exact_only=True, **kw)
    assert np.array_equal(D, De) and np.array_equal(I, Ie)
    assert ix.stats()[1] == 0
    if Do is not None:
        sel = slice(None) if sub is None else sub
        assert_same_results(D[sel], I[sel], Do, Io)
    assert st[1] in (0, nq), st
    if tile is not None:
        assert st[1] == (nq if tile else 0), st
    if st[1] == 0:
        assert st[2] == 0
    return D, I, st


def check_flat(ix, xb, ids, xq, k, n_oracle=32, tile=None, **kw):
    filt = {key: kw[key] for key in ("id_range", "sorted_ids", "negate") if key in kw}
    sub = np.arange(0, xq.shape[0], max(1, xq.shape[0] // n_oracle))
    Do, Io = bo.flat_search(xb, ids, xq[sub], k, **filt)
    return search_checked(ix, xq, k, Do, Io, sub=sub, tile=tile, **kw)


@pytest.mark.parametrize("dim", [8, 24, 64, 256, 264, 1000, 4096, 32768])
@pytest.mark.parametrize("nq", [15, 16, 1024])
def test_flat_shapes_tile(dim, nq):
    rng = np.random.default_rng(dim + nq)
    n = 32768 if dim <= 1000 else 8192
    xb = rng.integers(0, 256, (n, dim // 8), dtype=np.uint8)
    xq = rng.integers(0, 256, (nq, dim // 8), dtype=np.uint8)
    ids = big_ids(rng, n)
    ix = b200vs.Index(BINARY_FLAT, HAMMING, dim)
    ix.add(xb, ids)
    for k in (1, 10, 128, 129):
        tile = tile_eligible(nq, n, k)
        _, _, st = check_flat(ix, xb, ids, xq, k, n_oracle=8 if dim == 32768 else 32, tile=tile)
        if tile and dim >= 64 and k <= 10:
            assert st[2] == 0  # uniform data: no query needs the exact scan
    assert tile_eligible(1024, n, 10) and not tile_eligible(16, n, 10)


@pytest.mark.parametrize("nq", [16, 1024, 4097])
def test_flat_batch_sizes(nq):
    rng = np.random.default_rng(nq)
    n, dim = 40000, 256
    xb = rng.integers(0, 256, (n, dim // 8), dtype=np.uint8)
    xq = rng.integers(0, 256, (nq, dim // 8), dtype=np.uint8)
    ids = big_ids(rng, n)
    ix = b200vs.Index(BINARY_FLAT, HAMMING, dim)
    ix.add(xb, ids)
    for k in (1, 10, 128):
        tile = tile_eligible(nq, n, k)
        _, _, st = check_flat(ix, xb, ids, xq, k, tile=tile)
        assert st[2] == 0
    assert tile_eligible(4097, n, 128)


@pytest.mark.parametrize("k", [1, 10, 32, 128])
def test_flat_tie_heavy_tile(k):
    rng = np.random.default_rng(k * 7)
    n, dim, nq = 65536, 64, 1024
    xb = bo.tie_heavy(rng, n, dim // 8)
    xq = bo.tie_heavy(rng, nq, dim // 8)
    ids = big_ids(rng, n)
    ix = b200vs.Index(BINARY_FLAT, HAMMING, dim)
    ix.add(xb, ids)
    Do, _, _ = check_flat(ix, xb, ids, xq, k, tile=tile_eligible(nq, n, k))
    if k >= 10:
        assert (np.diff(Do, axis=1) == 0).mean() > 0.5  # the rank cut falls inside blocks of equal distances


def test_identical_rows_overflow_the_capture():
    rng = np.random.default_rng(1)
    n, dim, nq = 20000, 128, 512
    row = rng.integers(0, 256, (1, dim // 8), dtype=np.uint8)
    xb = np.repeat(row, n, axis=0)
    ids = big_ids(rng, n)
    xq = rng.integers(0, 256, (nq, dim // 8), dtype=np.uint8)
    ix = b200vs.Index(BINARY_FLAT, HAMMING, dim)
    ix.add(xb, ids)
    _, _, st = check_flat(ix, xb, ids, xq, 10, tile=True)
    assert st[2] == nq  # every row ties: the capture overflows, the exact scan answers


def test_filters_and_writes_tile():
    rng = np.random.default_rng(4)
    n, dim, nq = 20000, 128, 512
    xb = bo.tie_heavy(rng, n, dim // 8, patterns=8, flips=3)
    ids = np.arange(n, dtype=np.int64) * 5 + 1
    xq = xb[rng.integers(0, n, nq)]
    ix = b200vs.Index(BINARY_FLAT, HAMMING, dim)
    ix.add(xb, ids)
    check_flat(ix, xb, ids, xq, 20, tile=True, id_range=(1000, 60000))
    allow = np.sort(rng.choice(ids, 3000, replace=False))
    check_flat(ix, xb, ids, xq, 20, tile=True, sorted_ids=allow)
    check_flat(ix, xb, ids, xq, 20, tile=True, sorted_ids=allow, negate=True)
    # a filter admitting fewer than k rows: no sampled threshold, every query re-runs exactly
    few = np.sort(ids[:5])
    _, _, st = check_flat(ix, xb, ids, xq, 20, tile=True, sorted_ids=few)
    assert st[2] == nq
    dead = ids[::7]
    assert ix.delete(dead) == dead.size
    keep = ~np.isin(ids, dead)
    check_flat(ix, xb[keep], ids[keep], xq, 20, tile=True)  # tombstones stay in the rows until compaction
    new_rows = rng.integers(0, 256, (300, dim // 8), dtype=np.uint8)
    up_ids = ids[keep][:300]
    ix.upsert(new_rows, up_ids)
    xb2, ids2 = xb[keep].copy(), ids[keep]
    xb2[:300] = new_rows
    check_flat(ix, xb2, ids2, xq, 20, tile=True)
    gone = ids2[: ids2.size * 2 // 3]
    ix.delete(gone)
    assert ix.get_deleted_count() == 0  # compaction
    live = ~np.isin(ids2, gone)
    check_flat(ix, xb2[live], ids2[live], xq, 20)


@pytest.mark.parametrize("lens", ["edges", "uniform"])
@pytest.mark.parametrize("dim", [64, 264])
def test_ivf_lists_tile(lens, dim):
    """Lists that are empty, of 1 row, of TC_CHUNK +- 1 rows and of 2 TC_SPAN + 1 rows; nprobe 1, 8 and nlist."""
    rng = np.random.default_rng(dim + len(lens))
    nb, nlist = dim // 8, 16
    cent = rng.integers(0, 256, (nlist, nb), dtype=np.uint8)
    if lens == "edges":
        sizes = [0, 1, 511, 512, 513, 4097, 0, 1, 300, 2, 511, 513, 1000, 3, 0, 64]
        parts = []
        for l, m in enumerate(sizes):  # rows equal to their centroid with one flipped bit land in that list
            x = np.repeat(cent[l:l + 1], m, axis=0)
            if m:
                flip = rng.integers(0, dim, m)
                x[np.arange(m), flip // 8] ^= (1 << (flip % 8)).astype(np.uint8)
            parts.append(x)
        xb = np.concatenate(parts)
    else:
        xb = rng.integers(0, 256, (12000, nb), dtype=np.uint8)
    ids = big_ids(rng, xb.shape[0])
    ix = b200vs.Index(BINARY_IVF_FLAT, HAMMING, dim, nlist=nlist)
    ix.set_trained_state(b200vs.binary_ivf_state_blob(cent))
    ix.add(xb, ids)
    off, _, codes, lids = ix.export_lists(nlist)
    n = xb.shape[0]
    xq = rng.integers(0, 256, (4096, nb), dtype=np.uint8)
    sub = np.arange(0, 4096, 128)
    seen_tile = False
    for nprobe in (1, 8, nlist):
        for nq, k in ((15, 10), (4096, 1), (4096, 10), (4096, 128), (16, 129)):
            Do, Io = bo.ivf_search(cent, off, codes, lids, xq[:nq][sub[sub < nq]], k, nprobe)
            _, _, st = search_checked(ix, xq[:nq], k, Do, Io, sub=sub[sub < nq], tile=tile_eligible(nq, n * nprobe / nlist, k), nprobe=nprobe)
            seen_tile |= st[1] > 0
    assert seen_tile
    # tombstones, upsert, compaction
    ix.delete(ids[::3])
    ix.upsert(rng.integers(0, 256, (200, nb), dtype=np.uint8), ids[1:600:3])
    off, _, codes, lids = ix.export_lists(nlist)
    Do, Io = bo.ivf_search(cent, off, codes, lids, xq[sub], 10, nlist)
    search_checked(ix, xq, 10, Do, Io, sub=sub, nprobe=nlist)
    allow = np.sort(rng.choice(lids, min(lids.size, 500), replace=False))
    Do, Io = bo.ivf_search(cent, off, codes, lids, xq[sub], 10, nlist, sorted_ids=allow, negate=True)
    search_checked(ix, xq, 10, Do, Io, sub=sub, nprobe=nlist, sorted_ids=allow, negate=True)


def test_ivf_tie_heavy_and_persistence(tmp_path):
    rng = np.random.default_rng(9)
    n, nlist, dim, nq = 30000, 64, 512, 4096
    xb = bo.tie_heavy(rng, n, dim // 8, patterns=32, flips=4)
    ids = big_ids(rng, n)
    ix = b200vs.Index(BINARY_IVF_FLAT, HAMMING, dim, nlist=nlist)
    ix.train(xb)
    ix.add(xb, ids)
    blob = ix.get_trained_state()
    xq = bo.tie_heavy(rng, nq, dim // 8, patterns=32, flips=6)
    D, I, st = search_checked(ix, xq, 10, nprobe=8)
    assert st[1] == nq
    path = str(tmp_path / "bivf.idx")
    ix.save(path)
    ix2 = b200vs.Index(BINARY_IVF_FLAT, HAMMING, dim, nlist=nlist)
    ix2.load(path)
    D2, I2, st2 = search_checked(ix2, xq, 10, nprobe=8)
    assert st2[1] == nq
    assert np.array_equal(D, D2) and np.array_equal(I, I2)
    assert np.array_equal(ix2.get_trained_state(), blob)


def test_device_pointer_and_coalesced_callers():
    import torch
    rng = np.random.default_rng(12)
    n, dim, k, nq = 300000, 64, 10, 512
    xb = rng.integers(0, 256, (n, dim // 8), dtype=np.uint8)
    ids = big_ids(rng, n)
    xq = rng.integers(0, 256, (nq, dim // 8), dtype=np.uint8)
    ix = b200vs.Index(BINARY_FLAT, HAMMING, dim)
    ix.add(xb, ids)
    De, Ie = ix.search(xq, k, exact_only=True)
    Do, Io = bo.flat_search(xb, ids, xq[:32], k)
    assert_same_results(De[:32], Ie[:32], Do, Io)
    dev = torch.device("cuda", 0)
    q = torch.from_numpy(xq).to(dev)
    od = torch.empty((nq, k), dtype=torch.float32, device=dev)
    oi = torch.empty((nq, k), dtype=torch.int64, device=dev)
    st = torch.cuda.Stream(device=dev)
    sp, keep = b200vs.make_search_params()
    ix.set_profiling(True)
    ix.search_device(nq, q.data_ptr(), k, od.data_ptr(), oi.data_ptr(), stream=st.cuda_stream, sp=sp)
    st.synchronize()
    assert ix.stats()[1] == nq
    ix.set_profiling(False)
    assert np.array_equal(od.cpu().numpy(), De) and np.array_equal(oi.cpu().numpy(), Ie)
    # 32 concurrent one-query callers, coalesced into batches (a batch of >= 28 of them takes the tile scan)
    res = [None] * 32
    barrier = threading.Barrier(32)

    def one(i):
        barrier.wait()
        res[i] = ix.search(xq[i:i + 1], k)

    ths = [threading.Thread(target=one, args=(i,)) for i in range(32)]
    for t in ths:
        t.start()
    for t in ths:
        t.join()
    for i in range(32):
        assert np.array_equal(res[i][0], De[i:i + 1]) and np.array_equal(res[i][1], Ie[i:i + 1])
