"""Range search through the list-sharded deployment (b200vs_shard_range_search[_device]) on one GPU.

At a world of one the sharded call runs the whole flow (coarse slice, probe-driven range scan, packed all-gather payload,
merge, counts) and must equal b200vs_range_search on the same index bit for bit: ids, distance bits and counts.  A world
of W is emulated with W indexes holding one list slice each: their range results, merged by b200vs_merge_topk_device,
must equal the unsharded call."""
import numpy as np
import pytest

import b200vs
from b200vs import COSINE, IP, IVF_FLAT, IVF_PQ, L2
from gpu_util import require_gpu
from test_gpu_exact_edges import prep, radius_for, raw_fp32

pytestmark = pytest.mark.gpu
D, NLIST, M = 32, 16, 8


@pytest.fixture(autouse=True)
def _gpu():
    require_gpu()


def _rows(n, seed):
    return np.random.default_rng(seed).standard_normal((n, D)).astype(np.float32)


def _same(a, b):
    Da, Ia, Ca = a
    Db, Ib, Cb = b
    assert np.array_equal(Ca, Cb), "counts differ"
    assert np.array_equal(Ia, Ib), "ids differ"
    assert np.array_equal(Da.view(np.uint32), Db.view(np.uint32)), "distance bits differ"


def _ivf_flat(o, metric, n=12000, seed=2):
    xb = _rows(n, seed)
    ix = b200vs.Index(IVF_FLAT, metric, D, nlist=NLIST)
    cent = prep(o, metric, xb[np.random.default_rng(seed).choice(n, NLIST, replace=False)])
    ix.set_trained_state(b200vs.ivf_state_blob(cent, metric))
    ix.add(xb, np.arange(1, n + 1, dtype=np.int64))
    return ix


def _ivf_pq(metric, nbits, n=9000, seed=3):
    ix = b200vs.Index(IVF_PQ, metric, D, nlist=NLIST, pq_m=M, pq_nbits=nbits)
    ix.train(_rows(max(256 * NLIST, 256 << nbits) + 1000, seed))
    assert ix.sub_type() == IVF_PQ
    ix.add(_rows(n, seed + 1), np.arange(1, n + 1, dtype=np.int64))
    return ix


def _radius(o, ix, metric, xq, hits):
    """A radius that keeps about `hits` rows of query 0 (from the stored rows; IVF-PQ has none, so the raw rows of an
    IVF-Flat index over the same data would do: the distance scale is what matters)."""
    if ix.sub_type() == IVF_FLAT:
        _, X, _, _ = ix.export_lists(NLIST)
    else:
        X = _rows(9000, 4)
    return radius_for(raw_fp32(X, prep(o, metric, xq[:1])[0], metric), metric, hits)


@pytest.mark.parametrize("kind", ["flat", "pq8", "pq4"])
@pytest.mark.parametrize("metric", [L2, IP, COSINE])
def test_world_of_one_equals_the_plain_call(oracle, metric, kind):
    import torch
    ix = _ivf_flat(oracle, metric) if kind == "flat" else _ivf_pq(metric, 8 if kind == "pq8" else 4)
    ix.coalescing(0)
    sh = b200vs.Shard(ix, 0, 1, None, lanes=3)
    nq, nprobe = 200, 5
    xq = _rows(nq, 9)
    radius = _radius(oracle, ix, metric, xq, 100)
    seq = iter(range(1000))
    for mr in (1, 100, 1024):
        _same(sh.range_search(xq, radius, mr, seq=next(seq), nprobe=nprobe), ix.range_search(xq, radius, mr, nprobe=nprobe))
    # range and top-k batches interleaved by sequence number, over several lanes
    for i in range(4):
        _same(sh.range_search(xq, radius, 256, seq=next(seq), nprobe=nprobe), ix.range_search(xq, radius, 256, nprobe=nprobe))
        Ds, Is = sh.search(xq, 10, seq=next(seq), nprobe=nprobe)
        Dp, Ip = ix.search(xq, 10, nprobe=nprobe)
        assert np.array_equal(Is, Ip) and np.array_equal(Ds.view(np.uint32), Dp.view(np.uint32))
    # filters
    sel = np.arange(5, 12000, 3, dtype=np.int64)
    for filt in (dict(id_range=(300, 7000)), dict(sorted_ids=sel), dict(sorted_ids=sel, negate=True)):
        _same(sh.range_search(xq, radius, 512, seq=next(seq), nprobe=nprobe, **filt),
              ix.range_search(xq, radius, 512, nprobe=nprobe, **filt))
    # device variant on a caller stream, and below 16 queries
    qd = torch.from_numpy(xq).cuda()
    mr = 300
    od = torch.empty((nq, mr), dtype=torch.float32, device="cuda")
    oi = torch.empty((nq, mr), dtype=torch.int64, device="cuda")
    oc = torch.empty((nq,), dtype=torch.int32, device="cuda")
    sp, _keep = b200vs.make_search_params(nprobe=nprobe)
    st = torch.cuda.Stream()
    torch.cuda.synchronize()
    sh.range_search_device(nq, qd.data_ptr(), radius, mr, od.data_ptr(), oi.data_ptr(), oc.data_ptr(), stream=st.cuda_stream, sp=sp, seq=next(seq))
    torch.cuda.synchronize()
    _same((od.cpu().numpy(), oi.cpu().numpy(), oc.cpu().numpy()), ix.range_search(xq, radius, mr, nprobe=nprobe))
    _same(sh.range_search(xq[:7], radius, 64, seq=next(seq), nprobe=nprobe), ix.range_search(xq[:7], radius, 64, nprobe=nprobe))
    # refusals: the same status from both variants, and the lane moves on
    for bad in (0, 4097):
        for call in (lambda s: sh.range_search(xq, radius, bad, seq=s, nprobe=nprobe),
                     lambda s: sh.range_search_device(nq, qd.data_ptr(), radius, bad, od.data_ptr(), oi.data_ptr(), oc.data_ptr(), sp=sp, seq=s)):
            with pytest.raises(b200vs.B200VSError) as e:
                call(next(seq))
            assert e.value.code == b200vs.EILLEGAL_PARAMETERS
    with pytest.raises(b200vs.B200VSError) as e:
        sh.range_search_device(nq, qd.data_ptr(), radius, mr, od.data_ptr(), oi.data_ptr(), 0, sp=sp, seq=next(seq))
    assert e.value.code == b200vs.EILLEGAL_PARAMETERS
    _same(sh.range_search(xq, radius, 64, seq=next(seq), nprobe=nprobe), ix.range_search(xq, radius, 64, nprobe=nprobe))
    sh.close()


def test_merge_orders_by_the_raw_key(oracle):
    """Two inner products a < b that round to the same 1 - ip: the single-index select ranks b first (its key -ip is
    smaller) although b's id is larger; a merge on the API distance would put a first.  The sharded call must not."""
    a = np.float32(2.0 ** -10)
    b = np.nextafter(a, np.float32(1))
    assert a != b and np.float32(1) - a == np.float32(1) - b, "premise: the pair collides in 1 - ip"
    rng = np.random.default_rng(6)
    n = 4000
    xb = rng.standard_normal((n, D)).astype(np.float32)
    xb[:, 0] = -np.abs(xb[:, 0]) - 1  # every other row has a negative inner product with e0
    xb[0] = 0; xb[0, 0] = a  # id 1: ip a
    xb[1] = 0; xb[1, 0] = b  # id 2: ip b > a
    ix = b200vs.Index(IVF_FLAT, IP, D, nlist=NLIST)
    ix.set_trained_state(b200vs.ivf_state_blob(xb[rng.choice(n, NLIST, replace=False)], IP))
    ix.add(xb, np.arange(1, n + 1, dtype=np.int64))
    sh = b200vs.Shard(ix, 0, 1, None)
    xq = rng.standard_normal((32, D)).astype(np.float32)
    xq[0] = 0
    xq[0, 0] = 1
    for mr in (8, 1024):  # the warp merge (world * k <= 256) and the block merge
        want = ix.range_search(xq, 1.0, mr, nprobe=NLIST)  # ip > 0
        assert want[2][0] == 2 and list(want[1][0, :2]) == [2, 1], "premise: the single index ranks b first"
        _same(sh.range_search(xq, 1.0, mr, nprobe=NLIST), want)
    sh.close()


@pytest.mark.parametrize("parts", [2, 4])
@pytest.mark.parametrize("metric", [L2, IP, COSINE])
def test_list_slices_on_one_gpu(oracle, metric, parts):
    """W ranks emulated by W indexes that hold one slice of the lists each (same trained state): their range results on
    the same probes, merged, equal the unsharded call."""
    import torch
    full = _ivf_flat(oracle, metric)
    off, X, _, ids = full.export_lists(NLIST)
    state = full.get_trained_state()
    per = NLIST // parts
    nq, nprobe, mr = 64, 6, 512
    xq = _rows(nq, 13)
    radius = _radius(oracle, full, metric, xq, 150)
    pd = torch.empty((parts, nq, mr), dtype=torch.float32, device="cuda")
    pi = torch.empty((parts, nq, mr), dtype=torch.int64, device="cuda")
    for r in range(parts):
        lo, hi = off[r * per], off[(r + 1) * per]
        ix = b200vs.Index(IVF_FLAT, metric, D, nlist=NLIST)
        ix.set_trained_state(state)
        if hi > lo:
            ix.add(X[lo:hi], ids[lo:hi])
        Dr, Ir, _ = ix.range_search(xq, radius, mr, nprobe=nprobe)
        pd[r].copy_(torch.from_numpy(Dr))
        pi[r].copy_(torch.from_numpy(Ir))
    od = torch.empty((nq, mr), dtype=torch.float32, device="cuda")
    oi = torch.empty((nq, mr), dtype=torch.int64, device="cuda")
    torch.cuda.synchronize()
    b200vs.merge_topk_device(0, parts, nq, mr, pd.data_ptr(), pi.data_ptr(), od.data_ptr(), oi.data_ptr())
    torch.cuda.synchronize()
    Dw, Iw, Cw = full.range_search(xq, radius, mr, nprobe=nprobe)
    I = oi.cpu().numpy()
    assert np.array_equal((I >= 0).sum(1), Cw)
    assert np.array_equal(I, Iw) and np.array_equal(od.cpu().numpy().view(np.uint32), Dw.view(np.uint32))


def test_two_ranks_match_oracle():
    """torchrun --nproc-per-node 2 (tests/shard_worker_range.py): sharded range search over two ranks == the expectation
    on the gathered index."""
    import os
    import subprocess
    import sys
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
           "--master-port", "29523", os.path.join(root, "tests", "shard_worker_range.py")]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "SHARD_WORKER_RANGE OK" in r.stdout, (r.stdout[-3000:], r.stderr[-3000:])
