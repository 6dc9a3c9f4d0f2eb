"""Row-sharded FLAT and HNSW through the b200vs_shard_* deployment, on one GPU.

At a world of one the sharded calls run the whole flow (device routing, status agreement, owner-side add, local search
keyed on the merge key, packed all-gather payload, merge) and must equal the plain index: FLAT bit for bit (ids,
distance bits, range counts) on every local path; HNSW graph byte-equal and searches equal.  A world of W is emulated with
W standalone indexes built from the rows b200vs.row_owner assigns to each rank: FLAT's merged device results equal one
index of all rows, HNSW's equal the numpy merge of the oracle's walks on each exported graph."""
import os
import subprocess
import sys
import threading

import numpy as np
import pytest

import b200vs
import oracle_lib
from b200vs import COSINE, FLAT, HNSW, IP, L2
from b200vs import shard as shard_py
from gpu_util import require_gpu

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
D = 64


@pytest.fixture(autouse=True)
def _gpu():
    require_gpu()


def _rows(n, seed, d=D):
    return np.random.default_rng(seed).standard_normal((n, d)).astype(np.float32)


def _ids(n, seed):
    """Distinct ids in scattered order (ids are non-negative: -1 marks an empty result slot and a tombstoned row)."""
    return np.random.default_rng(seed).choice(np.arange(10 * n), n, replace=False).astype(np.int64)


def _same(a, b):
    for x, y in zip(a, b):
        if x.dtype == np.float32:
            assert np.array_equal(x.view(np.uint32), y.view(np.uint32)), "distance bits differ"
        else:
            assert np.array_equal(x, y), "ids / counts differ"


def _export(ix):
    off, X, _, I = ix.export_lists(1)
    return off, X, I


def _flat_pair(metric, n=20000, seed=1):
    x, ids = _rows(n, seed), _ids(n, seed + 1)
    plain = b200vs.Index(FLAT, metric, D)
    plain.add(x, ids)
    ix = b200vs.Index(FLAT, metric, D)
    sh = b200vs.Shard(ix, 0, 1, None, lanes=3)
    sh.add(x, ids)
    return plain, ix, sh, x, ids


@pytest.mark.parametrize("metric", [L2, IP, COSINE])
def test_flat_world_of_one(oracle, metric):
    import torch
    plain, ix, sh, x, ids = _flat_pair(metric)
    plain.coalescing(0)
    for a, b in zip(_export(ix), _export(plain)):
        assert np.array_equal(a, b), "sharded host add differs from a plain add"
    # device add: byte-equal export as well
    ixd = b200vs.Index(FLAT, metric, D)
    shd = b200vs.Shard(ixd, 0, 1, None)
    xd, idd = torch.from_numpy(x).cuda(), torch.from_numpy(ids).cuda()
    torch.cuda.synchronize()
    shd.add_device(x.shape[0] // 2, xd.data_ptr(), idd.data_ptr())
    shd.add_device(x.shape[0] - x.shape[0] // 2, xd[x.shape[0] // 2:].data_ptr(), idd[x.shape[0] // 2:].data_ptr())
    for a, b in zip(_export(ixd), _export(plain)):
        assert np.array_equal(a, b), "sharded device add differs from a plain add"
    shd.close()
    # every local path: tile scan (nq >= 16), flat_small (nq < 16), exact scan (exact_only); k wide enough to leave the warp merge
    for nq, k, kw in ((200, 10, {}), (200, 300, {}), (5, 10, {}), (40, 10, dict(exact_only=True)), (1, 100, {})):
        xq = _rows(nq, 7 + nq)
        _same(sh.search(xq, k, **kw), plain.search(xq, k, **kw))
    xq = _rows(100, 9)
    # filters, with and without negation
    sel = np.sort(ids[::3])
    for filt in (dict(id_range=(20000, 120000)), dict(sorted_ids=sel), dict(sorted_ids=sel, negate=True)):
        _same(sh.search(xq, 10, **filt), plain.search(xq, 10, **filt))
    # oracle on the host call (cosine: the stored rows and the prepared queries are unit rows, scored as IP)
    _, X, I = _export(plain)
    qo = oracle.normalize_faiss(xq) if metric == COSINE else xq
    _same(sh.search(xq, 10), oracle.flat_search(IP if metric == COSINE else metric, X, I, qo, 10, nthreads=8))
    # device calls on two caller streams
    qd = torch.from_numpy(xq).cuda()
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    outs = []
    for st in (s1, s2, s1):
        od = torch.empty((100, 10), dtype=torch.float32, device="cuda")
        oi = torch.empty((100, 10), dtype=torch.int64, device="cuda")
        sh.search_device(100, qd.data_ptr(), 10, od.data_ptr(), oi.data_ptr(), stream=st.cuda_stream)
        outs.append((st, od, oi))
    torch.cuda.synchronize()
    want = plain.search(xq, 10)
    for _, od, oi in outs:
        _same((od.cpu().numpy(), oi.cpu().numpy()), want)
    # threaded callers (seq < 0: next in call order)
    res, errs = {}, []

    def worker(t):
        try:
            res[t] = sh.search(_rows(64, 100 + t), 10)
        except Exception as e:  # noqa: BLE001
            errs.append(e)
    th = [threading.Thread(target=worker, args=(t,)) for t in range(6)]
    for t in th:
        t.start()
    for t in th:
        t.join()
    assert not errs
    for t in range(6):
        _same(res[t], plain.search(_rows(64, 100 + t), 10))
    # range search: tile range scan and the exact scan
    q0 = qo[0]
    raw = ((X - q0) ** 2).sum(1) if metric == L2 else X @ q0
    t = np.sort(raw)[200] if metric == L2 else np.sort(raw)[::-1][200]
    radius = float(t) if metric == L2 else float(np.float32(1) - np.float32(t))
    for nq, mr in ((100, 512), (8, 64), (100, 4096)):
        _same(sh.range_search(xq[:nq], radius, mr), plain.range_search(xq[:nq], radius, mr))
    # tombstones from the collective delete; unknown ids are ignored with OK
    dead = ids[::5]
    assert sh.delete(np.concatenate([dead, np.array([10 ** 12], np.int64)])) == dead.size
    plain.delete(dead)
    _same(sh.search(xq, 10), plain.search(xq, 10))
    _same(sh.range_search(xq, radius, 512), plain.range_search(xq, radius, 512))
    assert sh.delete(np.array([10 ** 12], np.int64)) == 0
    sh.close()


def test_device_routing_over_many_tiles():
    """One add of more rows than one pass of the offsets scan covers (more than 1024 tiles of 256 rows), on host and device
    pointers: the stored rows, their order and ids equal a plain add's."""
    import torch
    n, d = 300_001, 16
    x, ids = _rows(n, 61, d), _ids(n, 62)
    plain = b200vs.Index(FLAT, L2, d)
    plain.add(x, ids)
    for device in (False, True):
        ix = b200vs.Index(FLAT, L2, d)
        sh = b200vs.Shard(ix, 0, 1, None)
        if device:
            xd, idd = torch.from_numpy(x).cuda(), torch.from_numpy(ids).cuda()
            torch.cuda.synchronize()
            sh.add_device(n, xd.data_ptr(), idd.data_ptr())
        else:
            sh.add(x, ids)
        for a, b in zip(_export(ix), _export(plain)):
            assert np.array_equal(a, b)
        sh.close()


def test_flat_ip_merge_key_keeps_the_single_index_order(oracle):
    """Two rows whose inner products differ but round to the same 1 - ip: the merge must keep the larger ip first, as the
    single index does, not order them by id."""
    q = np.zeros((1, D), np.float32)
    q[0, 0] = 1.0
    a = np.zeros((2, D), np.float32)
    a[0, 0] = np.float32(1e-9)          # ip 1e-9  -> 1 - ip rounds to 1
    a[1, 0] = np.float32(2e-9)          # ip 2e-9  -> 1 - ip rounds to 1
    filler = _rows(5000, 3) * np.float32(-1e-3)
    filler[:, 0] = -1.0
    x = np.concatenate([a, filler])
    ids = np.concatenate([np.array([5, 9], np.int64), np.arange(100, 5100, dtype=np.int64)])
    plain = b200vs.Index(FLAT, IP, D)
    plain.add(x, ids)
    ix = b200vs.Index(FLAT, IP, D)
    sh = b200vs.Shard(ix, 0, 1, None)
    sh.add(x, ids)
    for nq in (1, 20):  # flat_small and the tile scan
        Dp, Ip = plain.search(np.repeat(q, nq, 0), 2)
        assert (Ip[:, :2] == [9, 5]).all() and (Dp[:, :2] == 1.0).all()
        _same(sh.search(np.repeat(q, nq, 0), 2), (Dp, Ip))
    sh.close()


@pytest.mark.parametrize("W", [2, 4])
@pytest.mark.parametrize("metric", [L2, IP, COSINE])
def test_flat_row_slices_merge_to_the_unsharded_index(metric, W):
    import torch
    n = 16000
    x, ids = _rows(n, 11), _ids(n, 12)
    own = b200vs.row_owner(ids, W)
    assert np.array_equal(own, shard_py.row_owner(ids, W))
    full = b200vs.Index(FLAT, metric, D)
    full.add(x, ids)
    nq, k = 64, 20
    xq = _rows(nq, 13)
    qd = torch.from_numpy(xq).cuda()
    pd = torch.empty((W, nq, k), dtype=torch.float32, device="cuda")
    pi = torch.empty((W, nq, k), dtype=torch.int64, device="cuda")
    parts = []
    for r in range(W):
        p = b200vs.Index(FLAT, metric, D)
        p.add(x[own == r], ids[own == r])
        parts.append(p)
        torch.cuda.synchronize()
        p.search_device(nq, qd.data_ptr(), k, pd[r].data_ptr(), pi[r].data_ptr())
    od = torch.empty((nq, k), dtype=torch.float32, device="cuda")
    oi = torch.empty((nq, k), dtype=torch.int64, device="cuda")
    b200vs.merge_topk_device(0, W, nq, k, pd.data_ptr(), pi.data_ptr(), od.data_ptr(), oi.data_ptr())
    torch.cuda.synchronize()
    Df, If = full.search(xq, k)
    assert all(len(set(r)) == k for r in Df)  # tie-free data
    _same((od.cpu().numpy(), oi.cpu().numpy()), (Df, If))


def _hnsw(metric, n=3000, d=32, max_elements=None):
    return b200vs.Index(HNSW, metric, d, hnsw_m=16, hnsw_efc=100, max_elements=max_elements or 2 * n)


def sh_plain_search(x, ids, metric, xq):
    p = _hnsw(metric)
    p.add(x, ids)
    return p.search(xq, 10, efsearch=64)


@pytest.mark.parametrize("metric", [L2, IP, COSINE])
def test_hnsw_world_of_one(metric):
    n, d = 3000, 32
    x, ids = _rows(n, 21, d), _ids(n, 22)
    plain, ix = _hnsw(metric), _hnsw(metric)
    plain.add(x[:2000], ids[:2000])
    plain.add(x[2000:], ids[2000:])
    sh = b200vs.Shard(ix, 0, 1, None)
    sh.add(x[:2000], ids[:2000])
    sh.add(x[2000:], ids[2000:])
    assert np.array_equal(ix.get_trained_state(), plain.get_trained_state()), "graph differs from a plain add"
    bp, bi = _hnsw(metric), _hnsw(metric)
    bp.add_batched(x, ids, 64)
    shb = b200vs.Shard(bi, 0, 1, None)
    shb.hnsw_add_batched(x, ids, 64)
    assert np.array_equal(bi.get_trained_state(), bp.get_trained_state()), "graph differs from a plain batched add"
    xq = _rows(50, 23, d)
    for kw in (dict(efsearch=64), dict(efsearch=16), dict(efsearch=64, id_range=(3000, 20000)),
               dict(efsearch=64, sorted_ids=np.sort(ids[::2])), dict(efsearch=64, sorted_ids=np.sort(ids[::2]), negate=True)):
        _same(sh.search(xq, 10, **kw), plain.search(xq, 10, **kw))
        _same(shb.search(xq, 10, **kw), bp.search(xq, 10, **kw))
    sh.delete(ids[::7])
    plain.delete(ids[::7])
    _same(sh.search(xq, 10, efsearch=64), plain.search(xq, 10, efsearch=64))
    sh.close()
    # range search is refused before the first collective, and its sequence number is used up: the next batch runs
    g = _hnsw(metric)
    shg = b200vs.Shard(g, 0, 1, None)
    shg.add(x, ids)
    with pytest.raises(b200vs.B200VSError) as e:
        shg.range_search(xq, 1.0, 10, seq=0)
    assert e.value.code == b200vs.EVECTOR_NOT_SUPPORT
    _same(shg.search(xq, 10, seq=1, efsearch=64), sh_plain_search(x, ids, metric, xq))
    shg.close()
    shb.close()


@pytest.mark.parametrize("W", [2, 4])
@pytest.mark.parametrize("metric", [L2, COSINE])
def test_hnsw_row_slices_merge_like_the_oracle(oracle, metric, W):
    import torch
    n, d, k = 4000, 32, 10
    x, ids = _rows(n, 31, d), _ids(n, 32)
    own = b200vs.row_owner(ids, W)
    xq = _rows(40, 33, d)
    qd = torch.from_numpy(xq).cuda()
    pd = torch.empty((W, 40, k), dtype=torch.float32, device="cuda")
    pi = torch.empty((W, 40, k), dtype=torch.int64, device="cuda")
    od_, oi_ = [], []
    for r in range(W):
        g = _hnsw(metric, n, d)
        g.add(x[own == r], ids[own == r])
        torch.cuda.synchronize()
        sp, _keep = b200vs.make_search_params(efsearch=64)
        g.search_device(40, qd.data_ptr(), k, pd[r].data_ptr(), pi[r].data_ptr(), sp=sp)
        h = oracle_lib.OracleHnsw(oracle, metric, d, n, 16, 100)
        h.load(g.get_trained_state())
        Do, Io, _, _ = h.search(xq, k, ef=64, nthreads=8)
        od_.append(Do)
        oi_.append(Io)
    od = torch.empty((40, k), dtype=torch.float32, device="cuda")
    oi = torch.empty((40, k), dtype=torch.int64, device="cuda")
    b200vs.merge_topk_device(0, W, 40, k, pd.data_ptr(), pi.data_ptr(), od.data_ptr(), oi.data_ptr())
    torch.cuda.synchronize()
    _same((od.cpu().numpy(), oi.cpu().numpy()), shard_py.merge_topk(np.stack(od_), np.stack(oi_), k))


def test_status_agreement_and_refusals():
    x, ids = _rows(100, 41), np.arange(100, dtype=np.int64)
    fl = b200vs.Index(FLAT, L2, D)
    sh = b200vs.Shard(fl, 0, 1, None)
    sh.add(x, ids)
    before = _export(fl)
    with pytest.raises(b200vs.B200VSError) as e:
        sh.add(_rows(3, 42), np.array([500, 501, 500], np.int64))
    assert e.value.code == b200vs.EVECTOR_ID_DUPLICATED
    for a, b in zip(_export(fl), before):
        assert np.array_equal(a, b)
    # upsert of existing ids through the collective add replaces the rows, as a plain add does
    plain = b200vs.Index(FLAT, L2, D)
    plain.add(x, ids)
    y = _rows(10, 43)
    sh.add(y, ids[:10])
    plain.add(y, ids[:10])
    for a, b in zip(_export(fl), _export(plain)):
        assert np.array_equal(a, b)
    # the collectives a row-sharded index has no use for
    assert sh.train(x) is None
    for call in (lambda: sh.broadcast_state(0), lambda: sh.list_range(), lambda: sh.plan_commit()):
        with pytest.raises(b200vs.B200VSError) as e:
            call()
        assert e.value.code == b200vs.EVECTOR_NOT_SUPPORT
    import torch
    xd = torch.from_numpy(x).cuda()
    with pytest.raises(b200vs.B200VSError) as e:
        sh.plan_add_device(100, xd.data_ptr())
    assert e.value.code == b200vs.EVECTOR_NOT_SUPPORT
    assert sh.delete(np.array([10 ** 9, 10 ** 9 + 1], np.int64)) == 0
    sh.close()
    # HNSW over max_elements: refused, graph unchanged (host and batched builders)
    g = _hnsw(L2, 100, D, max_elements=120)
    shg = b200vs.Shard(g, 0, 1, None)
    shg.add(x, ids)
    st = g.get_trained_state()
    for call in (lambda: shg.add(_rows(30, 44), np.arange(1000, 1030)), lambda: shg.hnsw_add_batched(_rows(30, 44), np.arange(1000, 1030))):
        with pytest.raises(b200vs.B200VSError) as e:
            call()
        assert e.value.code == b200vs.EINTERNAL
        assert np.array_equal(g.get_trained_state(), st)
    with pytest.raises(b200vs.B200VSError) as e:
        b200vs.Shard(b200vs.Index(FLAT, L2, D), 0, 1, None).hnsw_add_batched(x, ids)
    assert e.value.code == b200vs.EILLEGAL_PARAMETERS
    shg.close()
    # a non-empty index cannot be wrapped
    with pytest.raises(b200vs.B200VSError) as e:
        b200vs.Shard(plain, 0, 1, None)
    assert e.value.code == b200vs.EVECTOR_NOT_SUPPORT


def test_hnsw_search_refusals_come_before_the_collectives():
    """efsearch outside [0, 1024] and a walk larger than the search kernel's shared memory are refused from the arguments, as
    b200vs_search refuses them, also on a rank whose graph is still empty; a refused efsearch does not become the sticky ef."""
    n, d = 3000, 32
    x, ids = _rows(n, 51, d), _ids(n, 52)
    plain, g = _hnsw(L2), _hnsw(L2)
    plain.add(x, ids)
    sh = b200vs.Shard(g, 0, 1, None)
    sh.add(x, ids)
    xq = _rows(40, 53, d)
    _same(sh.search(xq, 10, efsearch=64), plain.search(xq, 10, efsearch=64))
    for efs in (2000, -1):
        with pytest.raises(b200vs.B200VSError) as e:
            sh.search(xq, 10, efsearch=efs)
        assert e.value.code == b200vs.EILLEGAL_PARAMETERS
        with pytest.raises(b200vs.B200VSError) as e:
            plain.search(xq, 10, efsearch=efs)
        assert e.value.code == b200vs.EILLEGAL_PARAMETERS
    # efsearch 0 walks with the sticky ef, still 64 on both
    _same(sh.search(xq, 10), plain.search(xq, 10))
    _same(sh.search(xq, 10), plain.search(xq, 10, efsearch=64))
    # a walk beyond the kernel's shared memory: refused on a rank that holds rows and on one that holds none
    empty = b200vs.Shard(_hnsw(L2), 0, 1, None)
    for s_ in (sh, empty):
        with pytest.raises(b200vs.B200VSError) as e:
            s_.search(xq, 30000)
        assert e.value.code == b200vs.EILLEGAL_PARAMETERS
    _same(sh.search(xq, 10), plain.search(xq, 10, efsearch=64))
    empty.close()
    sh.close()


def test_batched_build_refusal_is_agreed_before_any_change():
    """The batched builder's shared-memory refusal depends on the rows a rank receives (min(batch, n)): it is part of the
    status agreement, so the call is refused before any graph changes."""
    g = b200vs.Index(HNSW, L2, 32, hnsw_m=16, hnsw_efc=5000, max_elements=20000)
    sh = b200vs.Shard(g, 0, 1, None)
    with pytest.raises(b200vs.B200VSError) as e:
        sh.hnsw_add_batched(_rows(9000, 54, 32), _ids(9000, 55), 8192)
    assert e.value.code == b200vs.EILLEGAL_PARAMETERS
    assert g.get_count() == 0
    sh.close()


def test_single_flat_index_still_refuses_device_adds():
    """The device-row add of a Flat owner is the shard's building block; b200vs_add_with_ids_device on FLAT is unchanged."""
    import torch
    fl = b200vs.Index(FLAT, L2, D)
    x = torch.zeros((4, D), device="cuda")
    i = torch.arange(4, dtype=torch.int64, device="cuda")
    torch.cuda.synchronize()
    with pytest.raises(b200vs.B200VSError) as e:
        fl.add_device(4, x.data_ptr(), i.data_ptr())
    assert e.value.code == b200vs.EVECTOR_NOT_SUPPORT
    assert fl.get_count() == 0


def test_two_ranks_match_a_plain_index():
    """torchrun --nproc-per-node 2 (tests/shard_worker_rows.py): each rank contributes different rows."""
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
           "--master-port", "29527", os.path.join(ROOT, "tests", "shard_worker_rows.py")]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert "SHARD_WORKER_ROWS OK" in r.stdout
