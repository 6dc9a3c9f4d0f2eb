"""List-sharded IVF-PQ (b200vs_shard_* and the single-index building blocks on an IVF_PQ index).

The sharded search must equal b200vs_search on the unsharded index bit for bit: the probes merged from the centroid
slices are the plain search's probes, and the coarse value (dis0) every LUT scan starts from is recomputed on the rank with
the coarse pass's arithmetic.  The oracle is the CPU IVF-PQ search (tests/pq_codes.py) on the exported lists."""
import os
import subprocess
import sys
import threading

import numpy as np
import pytest

import b200vs
import oracle_lib
import pq_codes
from b200vs import COSINE, IP, IVF_FLAT, IVF_PQ, L2
from gpu_util import assert_same_results, require_gpu

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
D, M, NLIST = 32, 8, 16


@pytest.fixture(autouse=True)
def _gpu():
    require_gpu()


def _rows(n, seed):
    return np.random.default_rng(seed).standard_normal((n, D)).astype(np.float32)


def _n_train(nbits):
    return max(256 * NLIST, 256 << nbits) + 1000  # enough for the IVF-PQ mode of b200vs_train


def _state(ix, nbits):
    """(centroids [nlist, d], codebooks [M, 2^nbits, d / M]) of a trained-state blob."""
    b = ix.get_trained_state()
    hdr = b[:48].view(np.int64)
    nl, ks = int(hdr[1]), 1 << int(hdr[5])
    f = b[48:].view(np.float32)
    return f[:nl * D].reshape(nl, D), f[nl * D:].reshape(M, ks, D // M)


def _export(ix, nbits):
    off, _, codes, ids = ix.export_lists(NLIST, with_vectors=False, code_size=pq_codes.code_size(M, nbits))
    return off, codes, ids


def _oracle(o, ix, metric, nbits, xq, k, nprobe, **filt):
    cent, cb = _state(ix, nbits)
    off, codes, ids = _export(ix, nbits)
    return pq_codes.ivfpq_search(o, metric, cent, cb, off, codes, ids, xq, k, nprobe, nthreads=8, **filt)


def _same_export(a, b, nbits):
    ea, eb = _export(a, nbits), _export(b, nbits)
    for x, y, what in zip(ea, eb, ("list offsets", "codes", "ids")):
        assert np.array_equal(x, y), f"{what} differ"


def _filled(metric, nbits, n=12000, seed=3):
    """An index trained by b200vs_train and filled by a host add: the unsharded reference."""
    ix = b200vs.Index(IVF_PQ, metric, D, nlist=NLIST, pq_m=M, pq_nbits=nbits)
    ix.train(_rows(_n_train(nbits), seed))
    assert ix.sub_type() == IVF_PQ
    xb = _rows(n, seed + 1)
    ids = np.arange(10, 10 + n, dtype=np.int64)
    ix.add(xb, ids)
    return ix, xb, ids


def _fresh(ref, metric, nbits):
    ix = b200vs.Index(IVF_PQ, metric, D, nlist=NLIST, pq_m=M, pq_nbits=nbits)
    ix.set_trained_state(ref.get_trained_state())
    return ix


@pytest.mark.parametrize("nbits", [8, 4])
@pytest.mark.parametrize("metric", [L2, IP, COSINE])
def test_world_of_one(oracle, metric, nbits):
    import torch
    xt = _rows(_n_train(nbits), 7)
    plain = b200vs.Index(IVF_PQ, metric, D, nlist=NLIST, pq_m=M, pq_nbits=nbits)
    plain.train(xt)
    ix = b200vs.Index(IVF_PQ, metric, D, nlist=NLIST, pq_m=M, pq_nbits=nbits)
    sh = b200vs.Shard(ix, 0, 1, None, lanes=2)
    sh.train(xt)
    assert np.array_equal(ix.get_trained_state(), plain.get_trained_state()), "shard_train differs from b200vs_train"
    assert sh.list_range() == (0, NLIST)
    n = 9000
    xb, ids = _rows(n, 8), np.arange(1, n + 1, dtype=np.int64)
    plain.add(xb, ids)
    sh.add(xb[:4000], ids[:4000])
    xd, idd = torch.from_numpy(xb[4000:]).cuda(), torch.from_numpy(ids[4000:]).cuda()
    torch.cuda.synchronize()
    sh.add_device(n - 4000, xd.data_ptr(), idd.data_ptr())
    _same_export(ix, plain, nbits)
    nq, k, nprobe = 70, 10, 6
    xq = _rows(nq, 9)
    seq = iter(range(1000))

    def check(D_, I_, k_, **kw):
        Dp, Ip = plain.search(xq, k_, nprobe=nprobe, **kw)
        assert_same_results(D_, I_, Dp, Ip)
        Do, Io = _oracle(oracle, plain, metric, nbits, xq, k_, nprobe, **kw)
        assert_same_results(D_, I_, Do, Io)

    check(*sh.search(xq, k, seq=next(seq), nprobe=nprobe), k)
    # device calls on two caller streams, explicit sequence numbers
    qd = torch.from_numpy(xq).cuda()
    outs = [(torch.empty((nq, k), dtype=torch.float32, device="cuda"), torch.empty((nq, k), dtype=torch.int64, device="cuda")) for _ in range(3)]
    sts = [torch.cuda.Stream() for _ in range(2)]
    sp, _keep = b200vs.make_search_params(nprobe=nprobe)
    torch.cuda.synchronize()
    for i in range(3):
        sh.search_device(nq, qd.data_ptr(), k, outs[i][0].data_ptr(), outs[i][1].data_ptr(), stream=sts[i % 2].cuda_stream, sp=sp, seq=next(seq))
    torch.cuda.synchronize()
    for od, oi in outs:
        check(od.cpu().numpy(), oi.cpu().numpy(), k)
    # concurrent callers taking turns by sequence number
    base = next(seq)
    res = {}

    def call(s):
        res[s] = sh.search(xq, k, seq=s, nprobe=nprobe)
    ths = [threading.Thread(target=call, args=(base + t,)) for t in (2, 0, 1)]
    for t in ths:
        t.start()
    for t in ths:
        t.join()
    seq = iter(range(base + 3, 1000))
    for s in res:
        check(*res[s], k)
    # filters, with and without negation
    check(*sh.search(xq, k, seq=next(seq), nprobe=nprobe, id_range=(300, 7000)), k, id_range=(300, 7000))
    sel = np.arange(5, n, 3, dtype=np.int64)
    for neg in (False, True):
        check(*sh.search(xq, k, seq=next(seq), nprobe=nprobe, sorted_ids=sel, negate=neg), k, sorted_ids=sel, negate=neg)
    # k wide enough to leave the warp merge (world * k > 256 records)
    D3, I3 = sh.search(xq, 300, seq=next(seq), nprobe=nprobe)
    check(D3, I3, 300)
    # tombstones from the collective delete
    dead = ids[::5]
    assert sh.delete(dead) == dead.size
    assert plain.delete(dead) == dead.size
    check(*sh.search(xq, k, seq=next(seq), nprobe=nprobe), k)
    # a k whose select pool does not fit the LUT scan's shared memory is refused before any work, and the lane moves on
    with pytest.raises(b200vs.B200VSError) as e:
        sh.search(xq, 60000, seq=next(seq), nprobe=nprobe)
    assert e.value.code == b200vs.EILLEGAL_PARAMETERS
    check(*sh.search(xq, k, seq=next(seq), nprobe=nprobe), k)
    sh.close()


@pytest.mark.parametrize("parts", [2, 4])
@pytest.mark.parametrize("metric,nbits", [(L2, 8), (IP, 4), (COSINE, 8)])
def test_list_slices_on_one_gpu(oracle, metric, nbits, parts):
    import torch
    ix, xb, ids = _filled(metric, nbits)
    nq, k = 90, 10
    nprobe = min(5, NLIST // parts)  # a slice ranks at most its own rows, so it can hand over nprobe of them
    xq = _rows(nq, 21)
    q = torch.from_numpy(xq).cuda()
    torch.cuda.synchronize()
    ts = torch.cuda.Stream()
    st = ts.cuda_stream
    per = NLIST // parts
    gs = torch.empty((parts, nq, nprobe), dtype=torch.float32, device="cuda")
    gl = torch.empty((parts, nq, nprobe), dtype=torch.int64, device="cuda")
    for r in range(parts):
        ix.coarse_device(nq, q.data_ptr(), nprobe, r * per, (r + 1) * per, gs[r].data_ptr(), gl[r].data_ptr(), stream=st)
    ps = torch.empty((nq, nprobe), dtype=torch.float32, device="cuda")
    pl = torch.empty((nq, nprobe), dtype=torch.int64, device="cuda")
    b200vs.merge_topk_device(0, parts, nq, nprobe, gs.data_ptr(), gl.data_ptr(), ps.data_ptr(), pl.data_ptr(), st)
    sp, _keep = b200vs.make_search_params(nprobe=nprobe)
    od = torch.empty((nq, k), dtype=torch.float32, device="cuda")
    oi = torch.empty((nq, k), dtype=torch.int64, device="cuda")
    ix.search_probes_device(nq, q.data_ptr(), k, pl.data_ptr(), nprobe, od.data_ptr(), oi.data_ptr(), stream=st, sp=sp)
    wd = torch.empty((nq, k), dtype=torch.float32, device="cuda")
    wi = torch.empty((nq, k), dtype=torch.int64, device="cuda")
    ix.search_device(nq, q.data_ptr(), k, wd.data_ptr(), wi.data_ptr(), stream=st, sp=sp)
    torch.cuda.synchronize()
    assert_same_results(od.cpu().numpy(), oi.cpu().numpy(), wd.cpu().numpy(), wi.cpu().numpy())
    Do, Io = _oracle(oracle, ix, metric, nbits, xq, k, nprobe)
    assert_same_results(od.cpu().numpy(), oi.cpu().numpy(), Do, Io)
    # the merged probe table is the oracle's coarse ranking over the whole centroid table
    cent, _ = _state(ix, nbits)
    qn = oracle.normalize_faiss(xq) if metric == COSINE else xq
    om = oracle_lib.L2 if metric == L2 else oracle_lib.IP
    cd, ci = oracle.flat_search(om, cent, np.arange(NLIST, dtype=np.int64), qn, nprobe)
    assert np.array_equal(pl.cpu().numpy(), ci)
    if metric == L2:  # the merged score is the ranking score: the L2 distance itself (-ip for IP)
        assert np.array_equal(ps.cpu().numpy().view(np.uint32), cd.view(np.uint32))


@pytest.mark.parametrize("metric,nbits", [(L2, 4), (IP, 8), (COSINE, 4)])
def test_per_rank_data_split_on_one_gpu(metric, nbits):
    """W indexes with one trained state, each fed only its own lists' rows through add_with_ids_device(lists_dev),
    searched with the merged probes and merged: the unsharded index's answer."""
    import torch
    W = 4
    ref, xb, ids = _filled(metric, nbits, seed=31)
    n = xb.shape[0]
    xd, idd = torch.from_numpy(xb).cuda(), torch.from_numpy(ids).cuda()
    lst = torch.empty(n, dtype=torch.int64, device="cuda")
    torch.cuda.synchronize()
    ref.assign_device(n, xd.data_ptr(), lst.data_ptr())
    h = lst.cpu().numpy()
    per = NLIST // W
    parts = [_fresh(ref, metric, nbits) for _ in range(W)]
    for w, p in enumerate(parts):
        sel = torch.from_numpy(np.nonzero(h // per == w)[0]).cuda()
        xs, ids_s, ls = xd[sel].contiguous(), idd[sel].contiguous(), lst[sel].contiguous()
        torch.cuda.synchronize()
        p.add_device(int(sel.numel()), xs.data_ptr(), ids_s.data_ptr(), ls.data_ptr())
    nq, k, nprobe = 64, 20, NLIST // W
    xq = _rows(nq, 33)
    q = torch.from_numpy(xq).cuda()
    gs = torch.empty((W, nq, nprobe), dtype=torch.float32, device="cuda")
    gl = torch.empty((W, nq, nprobe), dtype=torch.int64, device="cuda")
    torch.cuda.synchronize()
    for w, p in enumerate(parts):
        p.coarse_device(nq, q.data_ptr(), nprobe, w * per, (w + 1) * per, gs[w].data_ptr(), gl[w].data_ptr())
    ps = torch.empty((nq, nprobe), dtype=torch.float32, device="cuda")
    pl = torch.empty((nq, nprobe), dtype=torch.int64, device="cuda")
    b200vs.merge_topk_device(0, W, nq, nprobe, gs.data_ptr(), gl.data_ptr(), ps.data_ptr(), pl.data_ptr())
    torch.cuda.synchronize()
    sp, _keep = b200vs.make_search_params(nprobe=nprobe)
    pd = torch.empty((W, nq, k), dtype=torch.float32, device="cuda")
    pi = torch.empty((W, nq, k), dtype=torch.int64, device="cuda")
    for w, p in enumerate(parts):
        p.search_probes_device(nq, q.data_ptr(), k, pl.data_ptr(), nprobe, pd[w].data_ptr(), pi[w].data_ptr(), sp=sp)
    od = torch.empty((nq, k), dtype=torch.float32, device="cuda")
    oi = torch.empty((nq, k), dtype=torch.int64, device="cuda")
    b200vs.merge_topk_device(0, W, nq, k, pd.data_ptr(), pi.data_ptr(), od.data_ptr(), oi.data_ptr())
    torch.cuda.synchronize()
    Dr, Ir = ref.search(xq, k, nprobe=nprobe)
    assert_same_results(od.cpu().numpy(), oi.cpu().numpy(), Dr, Ir)


@pytest.mark.parametrize("metric,nbits", [(L2, 8), (IP, 5), (COSINE, 8), (COSINE, 3)])
def test_device_write_path(oracle, metric, nbits):
    import torch
    ref, xb, ids = _filled(metric, nbits, seed=41)
    n = xb.shape[0]
    xd, idd = torch.from_numpy(xb).cuda(), torch.from_numpy(ids).cuda()
    lst = torch.empty(n, dtype=torch.int64, device="cuda")
    torch.cuda.synchronize()
    # assignment = the oracle's nearest centroid
    a = _fresh(ref, metric, nbits)
    a.assign_device(n, xd.data_ptr(), lst.data_ptr())
    cent, _ = _state(ref, nbits)
    assert np.array_equal(lst.cpu().numpy(), oracle.assign(metric, xb, cent).astype(np.int64)), "assignment differs from the oracle"
    # rows from device memory, library-side assignment for some chunks and precomputed lists for others
    for c, s in enumerate(range(0, n, 5000)):
        m = min(5000, n - s)
        a.add_device(m, xd[s:].data_ptr(), idd[s:].data_ptr(), lst[s:].data_ptr() if c % 2 else None)
    assert np.array_equal(xd.cpu().numpy(), xb), "add_with_ids_device changed the caller's rows"
    _same_export(a, ref, nbits)
    # upsert removes first, as the host upsert does
    xu = (xb[:300] + 0.25).astype(np.float32)
    xud = torch.from_numpy(xu).cuda()
    torch.cuda.synchronize()
    a.add_device(300, xud.data_ptr(), idd.data_ptr(), upsert=True)
    ref.upsert(xu, ids[:300])
    _same_export(a, ref, nbits)
    assert a.get_count() == ref.get_count() == n
    # reserved lists: later adds neither relocate a list nor re-allocate the arena
    r = _fresh(ref, metric, nbits)
    r.reserve_lists(np.bincount(lst.cpu().numpy(), minlength=NLIST))
    mem0 = r.get_memory_size()
    for s in range(0, n, 3000):
        r.add_device(min(3000, n - s), xd[s:].data_ptr(), idd[s:].data_ptr(), lst[s:].data_ptr())
    assert r.get_memory_size() == mem0, "a reserved index must not re-allocate its arena"
    h = _fresh(ref, metric, nbits)
    h.add(xb, ids)
    _same_export(r, h, nbits)
    xq = _rows(40, 43)
    Dr, Ir = r.search(xq, 10, nprobe=4)
    Do, Io = _oracle(oracle, h, metric, nbits, xq, 10, 4)
    assert_same_results(Dr, Ir, Do, Io)
    # out-of-range caller lists are refused
    bad = torch.full((4,), NLIST, dtype=torch.int64, device="cuda")
    torch.cuda.synchronize()
    with pytest.raises(b200vs.B200VSError) as e:
        r.add_device(4, xd.data_ptr(), idd.data_ptr(), bad.data_ptr())
    assert e.value.code == b200vs.EILLEGAL_PARAMETERS


def _codes(calls):
    out = []
    for c in calls:
        try:
            c()
            out.append(b200vs.OK)
        except b200vs.B200VSError as e:
            out.append(e.code)
    return out


def _block_calls(ix, torch):
    x = torch.zeros((4, D), device="cuda")
    i64 = torch.arange(4, dtype=torch.int64, device="cuda")
    f = torch.empty((4, 4), dtype=torch.float32, device="cuda")
    l = torch.zeros((4, 4), dtype=torch.int64, device="cuda")
    torch.cuda.synchronize()
    return [lambda: ix.add_device(4, x.data_ptr(), i64.data_ptr()),
            lambda: ix.assign_device(4, x.data_ptr(), i64.data_ptr()),
            lambda: ix.reserve_lists(np.ones(NLIST, np.int64)),
            lambda: ix.coarse_device(4, x.data_ptr(), 2, 0, NLIST, f.data_ptr(), l.data_ptr()),
            lambda: ix.search_probes_device(4, x.data_ptr(), 4, l.data_ptr(), 4, f.data_ptr(), l.data_ptr())], (x, i64, f, l)


def test_refusals():
    import torch
    # inner-Flat mode (too few training rows for IVF-PQ) has no lists
    fl = b200vs.Index(IVF_PQ, L2, D, nlist=NLIST, pq_m=M, pq_nbits=8)
    fl.train(_rows(500, 51))
    assert fl.sub_type() == b200vs.FLAT
    calls, _keep = _block_calls(fl, torch)
    assert _codes(calls) == [b200vs.EVECTOR_NOT_SUPPORT] * len(calls)
    with pytest.raises(b200vs.B200VSError) as e:
        b200vs.Shard(fl, 0, 1, None)
    assert e.value.code == b200vs.EVECTOR_NOT_SUPPORT
    # untrained: the statuses IVF_FLAT returns
    pq = b200vs.Index(IVF_PQ, L2, D, nlist=NLIST, pq_m=M, pq_nbits=8)
    iv = b200vs.Index(IVF_FLAT, L2, D, nlist=NLIST)
    c_pq, _k1 = _block_calls(pq, torch)
    c_iv, _k2 = _block_calls(iv, torch)
    assert _codes(c_pq) == _codes(c_iv)
    # too few training rows for shard_train: fewer than nlist / world, or fewer than 256 * 2^nbits on rank 0
    sh = b200vs.Shard(pq, 0, 1, None)
    for rows in (NLIST - 1, 256 * 256 - 1):
        with pytest.raises(b200vs.B200VSError) as e:
            sh.train(_rows(rows, 52))
        assert e.value.code == b200vs.EILLEGAL_PARAMETERS
    assert not pq.is_trained()
    sh.close()


def test_two_ranks_match_oracle():
    """torchrun --nproc-per-node 2 (tests/shard_worker_pq.py): distributed training, row routing, sharded search == oracle."""
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
           "--master-port", "29519", os.path.join(ROOT, "tests", "shard_worker_pq.py")]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "SHARD_WORKER_PQ OK" in r.stdout, (r.stdout[-3000:], r.stderr[-3000:])
