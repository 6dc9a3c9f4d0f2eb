"""Binary Flat and Binary IVF-Flat on the GPU against the binary oracle (tests/binary_oracle.py): ids AND distances
bit-equal on every search, plus the write path, persistence, the state blob, training and the refusals of mixed calls."""
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


def assert_rows_in_oracle_lists(off, list_ids, ids, lists):
    """Every list segment of the export holds exactly the ids the oracle assigns to that list."""
    for l in range(off.size - 1):
        assert np.array_equal(np.sort(list_ids[off[l]:off[l + 1]]), np.sort(ids[lists == l])), f"list {l}"


def check_flat(ix, xb, ids, xq, k, **kw):
    filt = {key: kw[key] for key in ("id_range", "sorted_ids", "negate") if key in kw}
    D, I = ix.search(xq, k, **kw)
    Do, Io = bo.flat_search(xb, ids, xq, k, **filt)
    assert_same_results(D, I, Do, Io)
    st = ix.stats()
    assert st[0] > 0 and st[1] == 0  # the exact Hamming scan served every query
    return D, I


@pytest.mark.parametrize("dim", [8, 24, 64, 256, 520, 1024, 32768])
@pytest.mark.parametrize("nq", [1, 15, 16])
def test_flat_shapes(dim, nq):
    rng = np.random.default_rng(dim + nq)
    n = 300 if dim == 32768 else 3000
    xb = rng.integers(0, 256, (n, dim // 8), dtype=np.uint8)
    xq = rng.integers(0, 256, (nq, dim // 8), dtype=np.uint8)
    ids = big_ids(rng, n)
    ix = b200vs.Index(BINARY_FLAT, HAMMING, dim)
    ix.add(xb, ids)
    assert ix.get_count() == n
    for k in (1, 10, 129):
        check_flat(ix, xb, ids, xq, k)


@pytest.mark.parametrize("k", [1, 10, 129, 1024, 4096, 8192])
@pytest.mark.parametrize("nq", [1, 16, 1024])
def test_flat_tie_heavy(k, nq):
    rng = np.random.default_rng(k * 7 + nq)
    n, dim = 6000, 64
    xb = bo.tie_heavy(rng, n, dim // 8)
    xq = bo.tie_heavy(rng, nq, dim // 8)
    ids = big_ids(rng, n)
    ix = b200vs.Index(BINARY_FLAT, HAMMING, dim)
    ix.add(xb, ids)
    if k >= 1024 and nq == 1024:
        xq = xq[:64]
    D, I = check_flat(ix, xb, ids, xq, k)
    if k >= 10:
        assert (np.diff(D, axis=1) == 0).mean() > 0.5  # the rank cut falls inside blocks of equal distances


def test_flat_train_is_a_no_op():
    rng = np.random.default_rng(11)
    xb = rng.integers(0, 256, (100, 8), dtype=np.uint8)
    ids = np.arange(100, dtype=np.int64)
    ix = b200vs.Index(BINARY_FLAT, HAMMING, 64)
    assert ix.is_trained()
    ix.train(xb)
    ix.add(xb, ids)
    ix.train(xb)
    assert ix.is_trained() and ix.get_count() == 100
    check_flat(ix, xb, ids, xb[:5], 10)
    with pytest.raises(b200vs.B200VSError) as e:
        b200vs._check(b200vs.lib().b200vs_train_binary(ix.h, 0, None))  # the same n / x checks as IVF
    assert e.value.code == b200vs.EILLEGAL_PARAMETERS


def test_flat_k_above_rows_pads_and_limits():
    rng = np.random.default_rng(3)
    xb = rng.integers(0, 256, (50, 4), dtype=np.uint8)
    ids = np.arange(50, dtype=np.int64)
    ix = b200vs.Index(BINARY_FLAT, HAMMING, 32)
    ix.add(xb, ids)
    D, I = check_flat(ix, xb, ids, xb[:3], 100)
    assert (I[:, 50:] == -1).all() and (D[:, 50:] == 0).all()
    D0, I0 = ix.search(xb[:2], 0)
    assert D0.shape == (2, 0)
    with pytest.raises(b200vs.B200VSError):
        ix.search(np.zeros((65536, 4), np.uint8), 1)
    with pytest.raises(b200vs.B200VSError):
        ix.search(xb[:1], 8193)


def test_flat_filters_and_writes():
    rng = np.random.default_rng(4)
    n, dim = 5000, 128
    xb = bo.tie_heavy(rng, n, dim // 8, patterns=8, flips=3)
    ids = np.arange(n, dtype=np.int64) * 5 + 1
    xq = xb[rng.integers(0, n, 20)]
    ix = b200vs.Index(BINARY_FLAT, HAMMING, dim)
    ix.add(xb, ids)
    check_flat(ix, xb, ids, xq, 20, id_range=(1000, 9000))
    allow = np.sort(rng.choice(ids, 700, replace=False))
    check_flat(ix, xb, ids, xq, 20, sorted_ids=allow)
    check_flat(ix, xb, ids, xq, 20, sorted_ids=allow, negate=True)
    # tombstones, then upsert of existing ids with new rows
    dead = ids[::7]
    assert ix.delete(dead) == dead.size
    assert ix.delete(np.array([3], np.int64)) == 0  # unknown ids are ignored, like the float Flat (flat.cc:171-203)
    keep = ~np.isin(ids, dead)
    check_flat(ix, xb[keep], ids[keep], xq, 20)
    new_rows = rng.integers(0, 256, (300, dim // 8), dtype=np.uint8)
    up_ids = ids[keep][:300]
    ix.upsert(new_rows, up_ids)
    xb2, ids2 = xb[keep].copy(), ids[keep]
    xb2[:300] = new_rows
    check_flat(ix, xb2, ids2, xq, 20)
    with pytest.raises(b200vs.B200VSError) as e:
        ix.add(new_rows[:2], np.array([9, 9], np.int64))
    assert e.value.code == b200vs.EVECTOR_ID_DUPLICATED
    # delete past half: compaction, results unchanged
    gone = ids2[: ids2.size * 2 // 3]
    ix.delete(gone)
    assert ix.get_deleted_count() == 0
    live = ~np.isin(ids2, gone)
    check_flat(ix, xb2[live], ids2[live], xq, 20)
    off, vec, codes, eids = ix.export_lists(1)
    assert vec is None and np.array_equal(np.sort(eids), np.sort(ids2[live]))
    order = np.argsort(ids2[live])
    assert np.array_equal(codes[np.argsort(eids)], xb2[live][order])


def test_flat_range_search():
    rng = np.random.default_rng(5)
    n, dim = 4000, 24
    xb = bo.tie_heavy(rng, n, dim // 8, patterns=3, flips=3)
    ids = big_ids(rng, n)
    xq = xb[:9]
    ix = b200vs.Index(BINARY_FLAT, HAMMING, dim)
    ix.add(xb, ids)
    for radius in (3.0, 2.5, 0.0, -1.0, float(dim + 1), 1e30):
        for mr in (1, 64, 4096):
            D, I, C = ix.range_search(xq, radius, mr)
            Do, Io, Co = bo.range_search(xb, ids, xq, radius, mr)
            assert np.array_equal(C, Co)
            assert_same_results(D, I, Do, Io)


@pytest.mark.parametrize("dim", [24, 256, 520])
def test_ivf_shared_state(dim):
    rng = np.random.default_rng(dim)
    n, nlist, nb = 8000, 64, dim // 8
    xb = bo.tie_heavy(rng, n, nb, patterns=32, flips=4)
    ids = big_ids(rng, n)
    cent = rng.integers(0, 256, (nlist, nb), dtype=np.uint8)
    cent[5] = cent[4]  # duplicate centroids: tied at the probe boundary, and list 5 stays empty at add time
    cent[9] = cent[4]
    ix = b200vs.Index(BINARY_IVF_FLAT, HAMMING, dim, nlist=nlist)
    ix.set_trained_state(b200vs.binary_ivf_state_blob(cent))
    ix.add(xb, ids)
    off, _, codes, lids = ix.export_lists(nlist)
    assert_rows_in_oracle_lists(off, lids, ids, bo.assign(xb, cent))  # nearest, ties to the smaller list
    assert off[6] == off[5] and off[10] == off[9]
    xq = np.concatenate([cent[4:5], bo.tie_heavy(rng, 40, nb, patterns=32, flips=6)])
    for nprobe in (1, 3, 80, 1000):
        for nq in (1, 15, 16, 41):
            D, I = ix.search(xq[:nq], 10, nprobe=nprobe)
            Do, Io = bo.ivf_search(cent, off, codes, lids, xq[:nq], 10, nprobe)
            assert_same_results(D, I, Do, Io)
    assert np.array_equal(ix.get_trained_state(), b200vs.binary_ivf_state_blob(cent))
    # range search over the probed lists only
    P = bo.probes(cent, xq, 8)
    cand = [np.concatenate([np.arange(off[l], off[l + 1]) for l in p]) for p in P]
    for radius in (3.0, 2.5, 0.0, -1.0, float(dim + 1)):
        D, I, C = ix.range_search(xq, radius, 64, nprobe=8)
        Do, Io, Co = bo.range_search(codes, lids, xq, radius, 64, candidates=cand)
        assert np.array_equal(C, Co)
        assert_same_results(D, I, Do, Io)


def test_ivf_writes_and_empty_lists():
    rng = np.random.default_rng(7)
    n, nlist, dim = 6000, 32, 64
    xb = rng.integers(0, 256, (n, 8), dtype=np.uint8)
    ids = np.arange(n, dtype=np.int64) + 100
    cent = rng.integers(0, 256, (nlist, 8), dtype=np.uint8)
    ix = b200vs.Index(BINARY_IVF_FLAT, HAMMING, dim, nlist=nlist)
    with pytest.raises(b200vs.B200VSError) as e:
        ix.add(xb[:1], ids[:1])
    assert e.value.code == b200vs.EVECTOR_NOT_TRAIN
    D, I = ix.search(xb[:4], 5)  # untrained: empty results
    assert (I == -1).all() and (D == 0).all()
    ix.set_trained_state(b200vs.binary_ivf_state_blob(cent))
    ix.add(xb, ids)
    a = bo.assign(xb, cent)
    full = np.bincount(a).argmax()
    gone = ids[a == full]  # a fully deleted list
    assert ix.delete(gone) == gone.size
    with pytest.raises(b200vs.B200VSError) as e:
        ix.delete(np.array([1], np.int64))
    assert e.value.code == b200vs.EVECTOR_INVALID
    ix.upsert(xb[:50][::-1].copy(), ids[a != full][:50])
    off, _, codes, lids = ix.export_lists(nlist)
    xq = xb[rng.integers(0, n, 30)]
    for nprobe in (1, 8, 32):
        D, I = ix.search(xq, 20, nprobe=nprobe)
        Do, Io = bo.ivf_search(cent, off, codes, lids, xq, 20, nprobe)
        assert_same_results(D, I, Do, Io)
        D, I = ix.search(xq, 20, nprobe=nprobe, id_range=(300, 4000))
        Do, Io = bo.ivf_search(cent, off, codes, lids, xq, 20, nprobe, id_range=(300, 4000))
        assert_same_results(D, I, Do, Io)
    # delete most rows: compaction keeps every answer
    ix.delete(ids[: n * 3 // 4])
    off, _, codes, lids = ix.export_lists(nlist)
    D, I = ix.search(xq, 20, nprobe=32)
    Do, Io = bo.ivf_search(cent, off, codes, lids, xq, 20, 32)
    assert_same_results(D, I, Do, Io)


def test_persistence_and_blob(tmp_path):
    rng = np.random.default_rng(8)
    dim, nlist = 40, 16
    xb = rng.integers(0, 256, (3000, dim // 8), dtype=np.uint8)
    ids = big_ids(rng, 3000)
    xq = xb[:20]
    cent = xb[100:100 + nlist]
    for t in (BINARY_FLAT, BINARY_IVF_FLAT):
        ix = b200vs.Index(t, HAMMING, dim, nlist=nlist)
        if t == BINARY_IVF_FLAT:
            ix.set_trained_state(b200vs.binary_ivf_state_blob(cent))
        ix.add(xb, ids)
        ix.delete(ids[:500])
        D, I = ix.search(xq, 10, nprobe=4)
        p = str(tmp_path / f"b{t}.idx")
        ix.save(p)
        ix2 = b200vs.Index(t, HAMMING, dim, nlist=nlist)
        ix2.load(p)
        D2, I2 = ix2.search(xq, 10, nprobe=4)
        assert_same_results(D2, I2, D, I)
        other = b200vs.Index(t, HAMMING, dim + 8, nlist=nlist)
        with pytest.raises(b200vs.B200VSError) as e:
            other.load(p)
        assert e.value.code == b200vs.EINTERNAL
    fl = b200vs.Index(b200vs.FLAT, b200vs.L2, dim)
    fl.add(rng.random((10, dim)).astype(np.float32), np.arange(10))
    fp = str(tmp_path / "float.idx")
    fl.save(fp)
    for t in (BINARY_FLAT, BINARY_IVF_FLAT):
        with pytest.raises(b200vs.B200VSError) as e:
            b200vs.Index(t, HAMMING, dim, nlist=nlist).load(fp)
        assert e.value.code == b200vs.EINTERNAL
    ix = b200vs.Index(BINARY_IVF_FLAT, HAMMING, dim + 8, nlist=nlist)
    with pytest.raises(b200vs.B200VSError) as e:
        ix.set_trained_state(b200vs.binary_ivf_state_blob(cent))  # blob of another width
    assert e.value.code == b200vs.EILLEGAL_PARAMETERS


def test_training():
    rng = np.random.default_rng(9)
    dim, nlist, n = 128, 32, 20000
    xb = bo.tie_heavy(rng, n, dim // 8, patterns=64, flips=10)
    ids = np.arange(n, dtype=np.int64)
    blobs = []
    for _ in range(2):
        ix = b200vs.Index(BINARY_IVF_FLAT, HAMMING, dim, nlist=nlist)
        ix.train(xb)
        assert ix.is_trained()
        blobs.append(ix.get_trained_state())
    assert np.array_equal(blobs[0], blobs[1])  # deterministic
    cent = blobs[0][32:].reshape(nlist, dim // 8)
    # +-1 rows have integer sums, so the engine's fixed-point k-means equals the oracle's float one exactly
    ocent = bo.kmeans(oracle_lib_load(), xb, dim, nlist)
    assert np.array_equal(cent, ocent)
    ix.add(xb, ids)
    off, _, codes, lids = ix.export_lists(nlist)
    assert_rows_in_oracle_lists(off, lids, ids, bo.assign(xb, cent))
    fl = b200vs.Index(BINARY_FLAT, HAMMING, dim)
    fl.train(xb[:10])  # Flat needs no training: a no-op
    fl.add(xb, ids)
    xq = xb[rng.integers(0, n, 64)]
    _, I = ix.search(xq, 10, nprobe=nlist)
    Df, If = fl.search(xq, 10)
    assert np.array_equal(I, If)
    # fewer rows than nlist: one list
    small = b200vs.Index(BINARY_IVF_FLAT, HAMMING, dim, nlist=nlist)
    small.train(xb[:10])
    assert small.get_trained_state()[8:16].view(np.int64)[0] == 1


def oracle_lib_load():
    import oracle_lib
    return oracle_lib.load()


def test_search_device_matches_host():
    import torch
    rng = np.random.default_rng(10)
    xb = rng.integers(0, 256, (2000, 16), dtype=np.uint8)
    ids = np.arange(2000, dtype=np.int64)
    ix = b200vs.Index(BINARY_FLAT, HAMMING, 128)
    ix.add(xb, ids)
    xq = xb[:32]
    D, I = ix.search(xq, 10)
    q = torch.from_numpy(xq).cuda()
    od = torch.zeros((32, 10), dtype=torch.float32, device="cuda")
    oi = torch.zeros((32, 10), dtype=torch.int64, device="cuda")
    ix.search_device(32, q.data_ptr(), 10, od.data_ptr(), oi.data_ptr())
    assert_same_results(od.cpu().numpy(), oi.cpu().numpy(), D, I)


def test_cross_calls_refused():
    L = b200vs.lib()
    bx = b200vs.Index(BINARY_FLAT, HAMMING, 64)
    fx = b200vs.Index(b200vs.FLAT, b200vs.L2, 64)
    f = np.zeros((2, 64), np.float32)
    u = np.zeros((2, 8), np.uint8)
    ids = np.arange(2, dtype=np.int64)
    D, I = np.zeros((2, 1), np.float32), np.zeros((2, 1), np.int64)
    C = np.zeros(2, np.int32)
    ill = b200vs.EILLEGAL_PARAMETERS
    assert L.b200vs_train(bx.h, 2, f.ctypes.data) == ill
    assert L.b200vs_add_with_ids(bx.h, 2, f.ctypes.data, ids.ctypes.data, 0) == ill
    assert L.b200vs_search(bx.h, 2, f.ctypes.data, 1, None, D.ctypes.data, I.ctypes.data) == ill
    assert L.b200vs_range_search(bx.h, 2, f.ctypes.data, 1.0, 1, None, D.ctypes.data, I.ctypes.data, C.ctypes.data) == ill
    assert L.b200vs_train_binary(fx.h, 2, u.ctypes.data) == ill
    assert L.b200vs_add_with_ids_binary(fx.h, 2, u.ctypes.data, ids.ctypes.data, 0) == ill
    assert L.b200vs_search_binary(fx.h, 2, u.ctypes.data, 1, None, D.ctypes.data, I.ctypes.data) == ill
    assert L.b200vs_range_search_binary(fx.h, 2, u.ctypes.data, 1.0, 1, None, D.ctypes.data, I.ctypes.data, C.ctypes.data) == ill
    bx.add(u, ids)
    out = np.zeros((2, 64), np.float32)
    found = np.zeros(2, np.uint8)
    assert L.b200vs_reconstruct(bx.h, 2, ids.ctypes.data, out.ctypes.data, found.ctypes.data) == b200vs.EVECTOR_NOT_SUPPORT
    assert L.b200vs_debug_tc_scores(bx.h, 2, f.ctypes.data, 0, out.ctypes.data, out.ctypes.data) == b200vs.EVECTOR_NOT_SUPPORT
    with pytest.raises(b200vs.B200VSError) as e:
        b200vs.BruteForceScan(HAMMING, 64, f, 1)
    assert e.value.code == b200vs.EVECTOR_NOT_SUPPORT
    bi = b200vs.Index(BINARY_IVF_FLAT, HAMMING, 64, nlist=2)
    with pytest.raises(b200vs.B200VSError) as e:
        b200vs.Shard(bi, 0, 1, None)
    assert e.value.code == b200vs.EVECTOR_NOT_SUPPORT
