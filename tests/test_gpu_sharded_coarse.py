"""List-sharded coarse quantiser (b200vs_coarse_device + b200vs_search_probes_device).

A multi-GPU deployment replicates the centroids and shards the inverted lists (SURVEY §8e).  Each rank ranks only
its own slice of the centroid table, the per-rank top-nprobe are all-gathered and merged with the (distance, id)
rule, and every rank then scans the merged probes.  Here the slices are taken on ONE index, so the composition
must reproduce b200vs_search_device bit for bit, and the merged probe table must equal the oracle's.
"""
import numpy as np
import pytest

import b200vs
import oracle_lib
from gpu_util import require_gpu

pytestmark = pytest.mark.gpu


def _build(metric, n, d, nlist, seed):
    rng = np.random.default_rng(seed)
    xb = rng.random((n, d), dtype=np.float32)
    ids = np.arange(100, 100 + n, dtype=np.int64)
    ix = b200vs.Index(b200vs.IVF_FLAT, metric, d, nlist=nlist)
    ix.train(xb)
    ix.add(xb, ids)
    return ix, xb, ids


def _sharded(ix, torch, xq, k, nprobe, nlist, parts, sp=None, own_stream=True):
    """own_stream: everything is enqueued on one caller stream (the deployed shape).  Otherwise stream = NULL: the
    library runs each call on a stream of its own and returns when the results are complete."""
    nq = xq.shape[0]
    q = torch.from_numpy(xq).cuda()
    torch.cuda.synchronize()
    ts = torch.cuda.Stream() if own_stream else None
    st = ts.cuda_stream if own_stream else None
    per = nlist // parts
    gs = torch.empty((parts, nq, nprobe), dtype=torch.float32, device="cuda")
    gl = torch.empty((parts, nq, nprobe), dtype=torch.int64, device="cuda")
    for r in range(parts):
        ix.coarse_device(nq, q.data_ptr(), nprobe, r * per, (r + 1) * per, gs[r].data_ptr(), gl[r].data_ptr(), stream=st)
    ps = torch.empty((nq, nprobe), dtype=torch.float32, device="cuda")
    pl = torch.empty((nq, nprobe), dtype=torch.int64, device="cuda")
    b200vs.merge_topk_device(0, parts, nq, nprobe, gs.data_ptr(), gl.data_ptr(), ps.data_ptr(), pl.data_ptr(), st)
    if not own_stream:
        torch.cuda.synchronize()  # the merge ran on the legacy default stream
    od = torch.empty((nq, k), dtype=torch.float32, device="cuda")
    oi = torch.empty((nq, k), dtype=torch.int64, device="cuda")
    ix.search_probes_device(nq, q.data_ptr(), k, pl.data_ptr(), nprobe, od.data_ptr(), oi.data_ptr(), stream=st, sp=sp)
    torch.cuda.synchronize()
    return od.cpu().numpy(), oi.cpu().numpy(), ps.cpu().numpy(), pl.cpu().numpy()


@pytest.mark.parametrize("metric", [b200vs.L2, b200vs.IP])
@pytest.mark.parametrize("nq,parts", [(5, 2), (300, 4)])
def test_sharded_coarse_equals_plain_search(metric, nq, parts):
    require_gpu()
    import torch
    n, d, nlist, k, nprobe = 20000, 64, 64, 10, 8
    ix, xb, ids = _build(metric, n, d, nlist, 3)
    xq = np.random.default_rng(9).random((nq, d), dtype=np.float32)
    wd, wi = ix.search(xq, k, nprobe=nprobe)
    sp, _keep = b200vs.make_search_params(nprobe=nprobe)
    od, oi, ps, pl = _sharded(ix, torch, xq, k, nprobe, nlist, parts, sp=sp)
    assert np.array_equal(oi, wi)
    assert np.array_equal(od.view(np.uint32), wd.view(np.uint32))
    # merged probes == the oracle's coarse ranking over the full centroid table
    o = oracle_lib.load()
    cent = ix.get_trained_state()[32:].view(np.float32).reshape(nlist, d)
    om = oracle_lib.L2 if metric == b200vs.L2 else oracle_lib.IP
    cd, ci = o.flat_search(om, cent, np.arange(nlist, dtype=np.int64), xq, nprobe)
    assert np.array_equal(pl, ci)
    if metric == b200vs.L2:  # the merged score is the ranking score: the L2 distance itself (-ip for IP)
        assert np.array_equal(ps.view(np.uint32), cd.view(np.uint32))


def test_sharded_coarse_tile_path_large():
    """Shapes that take the TMA + wgmma coarse pass (1024 centroids, 768-d, 1024 queries)."""
    require_gpu()
    import torch
    n, d, nlist, k, nprobe = 60000, 768, 1024, 10, 32
    ix, xb, ids = _build(b200vs.L2, n, d, nlist, 5)
    xq = np.random.default_rng(11).random((1024, d), dtype=np.float32)
    wd, wi = ix.search(xq, k, nprobe=nprobe)
    sp, _keep = b200vs.make_search_params(nprobe=nprobe)
    for parts, own in ((2, True), (8, True), (4, False)):
        od, oi, ps, pl = _sharded(ix, torch, xq, k, nprobe, nlist, parts, sp=sp, own_stream=own)
        assert np.array_equal(oi, wi)
        assert np.array_equal(od.view(np.uint32), wd.view(np.uint32))


def test_coarse_split_by_queries_equals_plain_search():
    """The other split: each 'rank' ranks a slice of the batch against ALL centroids; concatenating the probe tables
    (what one all-gather does) and scanning them reproduces the plain search."""
    require_gpu()
    import torch
    n, d, nlist, k, nprobe, nq, parts = 60000, 768, 1024, 10, 32, 1024, 4
    ix, xb, ids = _build(b200vs.L2, n, d, nlist, 5)
    xq = np.random.default_rng(12).random((nq, d), dtype=np.float32)
    wd, wi = ix.search(xq, k, nprobe=nprobe)
    sp, _keep = b200vs.make_search_params(nprobe=nprobe)
    q = torch.from_numpy(xq).cuda()
    torch.cuda.synchronize()
    ts = torch.cuda.Stream()
    bq = nq // parts
    sc = torch.empty((nq, nprobe), dtype=torch.float32, device="cuda")
    pl = torch.empty((nq, nprobe), dtype=torch.int64, device="cuda")
    for r in range(parts):
        ix.coarse_device(bq, q[r * bq:].data_ptr(), nprobe, 0, nlist, sc[r * bq:].data_ptr(), pl[r * bq:].data_ptr(), stream=ts.cuda_stream)
    od = torch.empty((nq, k), dtype=torch.float32, device="cuda")
    oi = torch.empty((nq, k), dtype=torch.int64, device="cuda")
    ix.search_probes_device(nq, q.data_ptr(), k, pl.data_ptr(), nprobe, od.data_ptr(), oi.data_ptr(), stream=ts.cuda_stream, sp=sp)
    torch.cuda.synchronize()
    assert np.array_equal(oi.cpu().numpy(), wi)
    assert np.array_equal(od.cpu().numpy().view(np.uint32), wd.view(np.uint32))
    o = oracle_lib.load()
    cent = ix.get_trained_state()[32:].view(np.float32).reshape(nlist, d)
    cd, ci = o.flat_search(oracle_lib.L2, cent, np.arange(nlist, dtype=np.int64), xq[:64], nprobe)
    assert np.array_equal(pl.cpu().numpy()[:64], ci)
    assert np.array_equal(sc.cpu().numpy()[:64].view(np.uint32), cd.view(np.uint32))


@pytest.mark.parametrize("metric", [b200vs.L2, b200vs.IP])
@pytest.mark.parametrize("nlist,dups", [(2048, 0), (4096, 0), (8192, 0), (10000, 0), (2048, 600), (1024, 300)],
                         ids=["2048", "4096", "8192", "10000", "2048-dup600", "1024-dup300"])
def test_coarse_large_tables_match_oracle(metric, nlist, dups):
    """Every register-select width (8 / 16 / 32 keys per thread) and the generic path above 8192 centroids, on a
    trained state loaded from outside (random centroids, duplicates included so exact ties occur).  dups > 0 repeats one
    centroid that often, with a query on it: more rows tie at the k-th score than the re-score window holds (512 rows in
    the register select used at 2048 centroids, 256 in the small-table kernel used at 1024), so the next finish kernel
    takes that query."""
    require_gpu()
    import torch
    d, nq, nprobe = 64, 96, 48
    rng = np.random.default_rng(nlist)
    cent = rng.random((nlist, d), dtype=np.float32)
    cent[5] = cent[4]
    cent[nlist - 1] = cent[7]
    if dups:
        cent[8:8 + dups] = 1.0  # the nearest row for L2 and the largest inner product for IP
    ix = b200vs.Index(b200vs.IVF_FLAT, metric, d, nlist=nlist)
    ix.set_trained_state(b200vs.ivf_state_blob(cent, metric))
    xq = rng.random((nq, d), dtype=np.float32)
    xq[0] = cent[4]
    if dups:
        xq[1] = cent[8]
    q = torch.from_numpy(xq).cuda()
    sc = torch.empty((nq, nprobe), dtype=torch.float32, device="cuda")
    pl = torch.empty((nq, nprobe), dtype=torch.int64, device="cuda")
    ix.coarse_device(nq, q.data_ptr(), nprobe, 0, nlist, sc.data_ptr(), pl.data_ptr())
    o = oracle_lib.load()
    om = oracle_lib.L2 if metric == b200vs.L2 else oracle_lib.IP
    cd, ci = o.flat_search(om, cent, np.arange(nlist, dtype=np.int64), xq, nprobe)
    assert np.array_equal(pl.cpu().numpy(), ci)
    if metric == b200vs.L2:
        assert np.array_equal(sc.cpu().numpy().view(np.uint32), cd.view(np.uint32))
    # the probe-table flavour (set mode) must select the same SET of lists
    xb = rng.random((4000, d), dtype=np.float32)
    ix.add(xb, np.arange(4000, dtype=np.int64))
    wd, wi = ix.search(xq, 10, nprobe=nprobe)
    od = torch.empty((nq, 10), dtype=torch.float32, device="cuda")
    oi = torch.empty((nq, 10), dtype=torch.int64, device="cuda")
    sp, _keep = b200vs.make_search_params(nprobe=nprobe)
    ix.search_probes_device(nq, q.data_ptr(), 10, pl.data_ptr(), nprobe, od.data_ptr(), oi.data_ptr(), sp=sp)
    assert np.array_equal(oi.cpu().numpy(), wi)
    assert np.array_equal(od.cpu().numpy().view(np.uint32), wd.view(np.uint32))


def test_coarse_device_rejects_bad_range():
    require_gpu()
    import torch
    ix, xb, ids = _build(b200vs.L2, 2000, 32, 16, 1)
    q = torch.zeros((2, 32), device="cuda")
    s = torch.empty((2, 4), dtype=torch.float32, device="cuda")
    l = torch.empty((2, 4), dtype=torch.int64, device="cuda")
    for a, b, npb in ((-1, 8, 4), (0, 17, 4), (8, 8, 4), (0, 2, 4)):
        with pytest.raises(b200vs.B200VSError):
            ix.coarse_device(2, q.data_ptr(), npb, a, b, s.data_ptr(), l.data_ptr())
