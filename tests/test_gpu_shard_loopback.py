"""Sharded indexes at world > 1 on one GPU.

Every path of b200vs_shard_* that depends on the world size (the owner routing kernels, the merge of several ranks'
records, query and probe slicing, list ownership when nlist % W != 0 or nlist < W, the grouped send / receive, the status
agreement and the collectives of the write path) runs here with W ranks as W threads of one process
(tests/shard_loopback.py) over the loopback NCCL (tests/nccl_loopback).  Each case runs in a subprocess of its own; the
case functions below are what that subprocess calls.  References need no second GPU: a plain single index with the same
trained state built in the same process, standalone per-rank HNSW graphs merged by b200vs.shard.merge_topk, and the
float32 restatement of range search on the gathered rows.  Ids and distance bits must be identical."""
import ctypes
import threading

import numpy as np
import pytest

import b200vs
from b200vs import COSINE, FLAT, HNSW, IP, IVF_FLAT, IVF_PQ, L2
from b200vs import shard as shard_py
from gpu_util import require_gpu
from shard_loopback import LIB, run_case, run_world

pytestmark = pytest.mark.gpu
WORLDS = (2, 3, 5, 8)


@pytest.fixture(autouse=True)
def _gpu():
    require_gpu()


def _assert_same(got, want, what):
    for x, y in zip(got, want):
        if x.dtype == np.float32:
            bad = np.argwhere(x.view(np.uint32) != y.view(np.uint32))
        else:
            bad = np.argwhere(x != y)
        assert bad.size == 0, f"{what}: differs at {bad[:4].tolist()}: got {x[tuple(bad[0])]}, want {y[tuple(bad[0])]}"


def each_world(case, worlds, *args):
    """globals()[case](W, *args) for every W of `worlds`, in one subprocess (the CUDA and torch start-up is paid once)."""
    for W in worlds:
        try:
            globals()[case](W, *args)
        except AssertionError as e:
            raise AssertionError(f"world {W}: {e}") from e


def _run(case, *args, worlds=WORLDS):
    run_case("each_world", case, list(worlds), *args)


def _status(fn):
    try:
        fn()
        return b200vs.OK
    except b200vs.B200VSError as e:
        return e.code


# ---------------------------------------------------------------------------------------------
# 1. the loopback library itself, against numpy
# ---------------------------------------------------------------------------------------------
NCCL_INT64, NCCL_FLOAT64, NCCL_SUM, NCCL_INVALID_USAGE = 4, 8, 0, 5


class _UniqueId(ctypes.Structure):
    _fields_ = [("internal", ctypes.c_char * 128)]


def case_selftest(W):
    import torch
    L = ctypes.CDLL(LIB)
    vp, sz = ctypes.c_void_p, ctypes.c_size_t
    L.ncclAllGather.argtypes = [vp, vp, sz, ctypes.c_int, vp, vp]
    L.ncclBroadcast.argtypes = [vp, vp, sz, ctypes.c_int, ctypes.c_int, vp, vp]
    L.ncclAllReduce.argtypes = [vp, vp, sz, ctypes.c_int, ctypes.c_int, vp, vp]
    L.ncclSend.argtypes = [vp, sz, ctypes.c_int, ctypes.c_int, vp, vp]
    L.ncclRecv.argtypes = [vp, sz, ctypes.c_int, ctypes.c_int, vp, vp]
    L.ncclCommInitRank.argtypes = [ctypes.POINTER(vp), ctypes.c_int, _UniqueId, ctypes.c_int]
    L.ncclCommSplit.argtypes = [vp, ctypes.c_int, ctypes.c_int, ctypes.POINTER(vp), vp]
    L.ncclCommDestroy.argtypes = [vp]
    uid = _UniqueId()
    assert L.ncclGetUniqueId(ctypes.byref(uid)) == 0
    dev = torch.device("cuda", 0)

    def cnt(s, d):  # uneven send counts, zeros (self-sends included) among them
        return ((s * 7 + d * 3) % 5) * 3

    def payload(s, d):
        return s * 10 ** 6 + d * 10 ** 3 + np.arange(cnt(s, d), dtype=np.int64)

    def rank(r, world):
        torch.cuda.set_device(0)
        st = torch.cuda.Stream(device=dev)
        sp = st.cuda_stream
        comm = vp()
        assert L.ncclCommInitRank(ctypes.byref(comm), W, uid, r) == 0
        lane = vp()
        assert L.ncclCommSplit(comm, 0, r, ctypes.byref(lane), None) == 0
        out = {}
        for c, name in ((comm, "comm"), (lane, "split")):
            n = 37
            send = torch.arange(n, dtype=torch.int64, device=dev) + r * 1000
            recv = torch.full((W * n,), -7, dtype=torch.int64, device=dev)
            torch.cuda.synchronize()
            assert L.ncclAllGather(send.data_ptr(), recv.data_ptr(), n, NCCL_INT64, c, sp) == 0
            inplace = torch.full((W * n,), -7, dtype=torch.int64, device=dev)
            inplace[r * n:(r + 1) * n] = send
            torch.cuda.synchronize()
            assert L.ncclAllGather(inplace[r * n:].data_ptr(), inplace.data_ptr(), n, NCCL_INT64, c, sp) == 0
            st.synchronize()
            out[name + " allgather"] = (recv.cpu().numpy(), inplace.cpu().numpy())
        for root in (0, W - 1):
            buf = torch.full((19,), r, dtype=torch.int64, device=dev) * 100 + torch.arange(19, device=dev)
            dst = torch.zeros(19, dtype=torch.int64, device=dev)
            torch.cuda.synchronize()
            assert L.ncclBroadcast(buf.data_ptr(), dst.data_ptr(), 19, NCCL_INT64, root, comm, sp) == 0
            assert L.ncclBroadcast(buf.data_ptr(), buf.data_ptr(), 19, NCCL_INT64, root, comm, sp) == 0  # in place
            st.synchronize()
            out[f"broadcast {root}"] = (dst.cpu().numpy(), buf.cpu().numpy())
        vi = torch.arange(11, dtype=torch.int64, device=dev) * (r + 1)
        vf = torch.full((5,), 0.1 * (r + 1), dtype=torch.float64, device=dev)
        torch.cuda.synchronize()
        assert L.ncclAllReduce(vi.data_ptr(), vi.data_ptr(), 11, NCCL_INT64, NCCL_SUM, comm, sp) == 0
        assert L.ncclAllReduce(vf.data_ptr(), vf.data_ptr(), 5, NCCL_FLOAT64, NCCL_SUM, comm, sp) == 0
        st.synchronize()
        out["allreduce"] = (vi.cpu().numpy(), vf.cpu().numpy())
        # grouped send / receive with uneven and zero counts, self included
        snd = [torch.from_numpy(payload(r, d)).to(dev) for d in range(W)]
        rcv = [torch.full((cnt(s, r),), -1, dtype=torch.int64, device=dev) for s in range(W)]
        torch.cuda.synchronize()
        assert L.ncclGroupStart() == 0
        for d in range(W):
            if cnt(r, d):
                assert L.ncclSend(snd[d].data_ptr(), cnt(r, d), NCCL_INT64, d, comm, sp) == 0
        for s in range(W):
            if cnt(s, r):
                assert L.ncclRecv(rcv[s].data_ptr(), cnt(s, r), NCCL_INT64, s, comm, sp) == 0
        assert L.ncclGroupEnd() == 0
        st.synchronize()
        out["sendrecv"] = [t.cpu().numpy() for t in rcv]
        # a count mismatch on the last rank: every rank gets an error, none hangs, and the next call still works
        n = 4 + (r == W - 1)
        send = torch.zeros(5, dtype=torch.int64, device=dev)
        recv = torch.zeros(5 * W, dtype=torch.int64, device=dev)
        torch.cuda.synchronize()
        out["mismatch"] = L.ncclAllGather(send.data_ptr(), recv.data_ptr(), n, NCCL_INT64, comm, sp)
        send += r
        torch.cuda.synchronize()
        assert L.ncclAllGather(send.data_ptr(), recv.data_ptr(), 5, NCCL_INT64, comm, sp) == 0
        st.synchronize()
        out["after mismatch"] = recv.cpu().numpy()
        world.barrier.wait()
        assert L.ncclCommDestroy(lane) == 0 and L.ncclCommDestroy(comm) == 0
        return out

    res = run_world(W, rank)
    n = 37
    gathered = np.concatenate([np.arange(n) + w * 1000 for w in range(W)])
    for r, o in enumerate(res):
        for name in ("comm", "split"):
            assert np.array_equal(o[name + " allgather"][0], gathered), f"rank {r} {name}: AllGather"
            assert np.array_equal(o[name + " allgather"][1], gathered), f"rank {r} {name}: in-place AllGather"
        for root in (0, W - 1):
            want = root * 100 + np.arange(19)
            assert np.array_equal(o[f"broadcast {root}"][0], want) and np.array_equal(o[f"broadcast {root}"][1], want), f"rank {r}: Broadcast {root}"
        assert np.array_equal(o["allreduce"][0], np.arange(11) * sum(range(1, W + 1))), f"rank {r}: AllReduce int64"
        acc = np.zeros(5)
        for w in range(W):
            acc += np.full(5, 0.1 * (w + 1))
        assert np.array_equal(o["allreduce"][1], acc), f"rank {r}: AllReduce float64"
        for s in range(W):
            assert np.array_equal(o["sendrecv"][s], payload(s, r)), f"rank {r}: receive from {s}"
        assert o["mismatch"] == NCCL_INVALID_USAGE, f"rank {r}: a count mismatch returned {o['mismatch']}"
        assert np.array_equal(o["after mismatch"], np.repeat(np.arange(W), 5)), f"rank {r}: call after the mismatch"


def test_loopback_library():
    _run("case_selftest")


# ---------------------------------------------------------------------------------------------
# 2. routing: every owner holds exactly its rows, in rank order then the sender's order
# ---------------------------------------------------------------------------------------------
def _row_counts(W, big):
    """Rows each rank sends: none on rank 0, less than one 256-row tile on rank 1, `big` on the last rank."""
    n = [0] + [97 + 31 * r for r in range(1, W)]
    n[-1] = big
    return n


def case_route_rows(W):
    """Row-sharded FLAT, d = 13 (the routing copy's scalar path): arrival order and contents on every rank."""
    import torch
    d = 13
    big = 256 * (1024 // W + 3) + 77  # ntiles * W > 1024: route_offsets_kernel carries across 1024-entry chunks
    n = _row_counts(W, big)
    rng = np.random.default_rng(W)
    xs = [rng.standard_normal((m, d)).astype(np.float32) for m in n]
    ids = [rng.choice(10 ** 7, m, replace=False).astype(np.int64) + r * 10 ** 7 for r, m in enumerate(n)]
    # second call: every rank sends 300 rows that all belong to the last rank, through a misaligned device pointer (d = 16)
    cand = np.arange(10 ** 8, 10 ** 8 + 40 * 300 * W, dtype=np.int64)
    mine = cand[shard_py.row_owner(cand, W) == W - 1][:300 * W].reshape(W, 300)
    x2 = [rng.standard_normal((300, d)).astype(np.float32) for _ in range(W)]

    def rank(r, world):
        ix = b200vs.Index(FLAT, L2, d)
        sh = world.connect(ix, r)
        x = np.empty(xs[r].size + 1, np.float32)[1:].reshape(xs[r].shape)  # a host slice off the 16-byte grid
        x[:] = xs[r]
        sh.add(x, ids[r])
        dx = torch.empty(x2[r].size + 1, dtype=torch.float32, device="cuda:0")
        dx[1:] = torch.from_numpy(x2[r].reshape(-1)).cuda()
        di = torch.from_numpy(mine[r]).cuda()
        torch.cuda.synchronize()
        sh.add_device(300, dx[1:].data_ptr(), di.data_ptr())
        off, vec, _, got = ix.export_lists(1)
        sh.close()
        return vec, got

    res = run_world(W, rank)
    own = [shard_py.row_owner(i, W) for i in ids]
    for r, (vec, got) in enumerate(res):
        want_i = np.concatenate([ids[s][own[s] == r] for s in range(W)] + ([mine.reshape(-1)] if r == W - 1 else []))
        want_x = np.concatenate([xs[s][own[s] == r] for s in range(W)] + ([np.concatenate(x2)] if r == W - 1 else []))
        assert np.array_equal(got, want_i), f"rank {r}: ids or their arrival order differ"
        assert np.array_equal(vec.view(np.uint32), want_x.view(np.uint32)), f"rank {r}: row contents differ"


def test_route_rows():
    _run("case_route_rows")


# ---------------------------------------------------------------------------------------------
# 3. list-sharded IVF-Flat and IVF-PQ against a plain index with the same trained state
# ---------------------------------------------------------------------------------------------
def _ivf_index(kind, metric, d, nlist, nbits):
    if kind == "pq":
        return b200vs.Index(IVF_PQ, metric, d, nlist=nlist, pq_m=4, pq_nbits=nbits)
    return b200vs.Index(IVF_FLAT, metric, d, nlist=nlist)


def case_ivf(W, kind, metric, lists, data, nbits=8):
    """kind "flat" | "pq"; lists "uneven" (nlist = 2W + 1: nlist % W != 0), "few" (nlist = 3 < W: some ranks own no list);
    data "normal" | "ties" (0 / 1 coordinates: many exact ties across ranks)."""
    import torch
    nlist = 2 * W + 1 if lists == "uneven" else 3
    d = 16
    rng = np.random.default_rng(1000 * W + nlist)
    n = _row_counts(W, 700)
    if data == "ties":
        xs = [rng.integers(0, 2, (m, d)).astype(np.float32) for m in n]
        for x in xs:
            x[:, 0] = 1  # no zero row (cosine)
    else:
        xs = [rng.standard_normal((m, d)).astype(np.float32) for m in n]
    ids = [np.arange(m, dtype=np.int64) * W + r + 1 for r, m in enumerate(n)]  # interleaved ids: ties resolve across ranks
    allx = np.concatenate(xs)
    cent = allx[rng.choice(len(allx), nlist, replace=False)].copy() + rng.standard_normal((nlist, d)).astype(np.float32) * 0.01
    if kind == "pq":
        cb = rng.standard_normal((4, 1 << nbits, d // 4)).astype(np.float32)
        blob = b200vs.ivfpq_state_blob(cent, cb, metric)
    else:
        blob = b200vs.ivf_state_blob(cent, metric)
    h = [m // 2 for m in n]  # each rank adds its first half through host pointers, then the rest through device pointers
    plain = _ivf_index(kind, metric, d, nlist, nbits)
    plain.set_trained_state(blob)
    plain.add(np.concatenate([x[:hh] for x, hh in zip(xs, h)]), np.concatenate([i[:hh] for i, hh in zip(ids, h)]))
    plain.add(np.concatenate([x[hh:] for x, hh in zip(xs, h)]), np.concatenate([i[hh:] for i, hh in zip(ids, h)]))
    p_off, p_vec, _, p_ids = plain.export_lists(nlist)
    if data == "ties":
        xq = rng.integers(0, 2, (64, d)).astype(np.float32)
        xq[:, 0] = 1
    else:
        xq = rng.standard_normal((64, d)).astype(np.float32)
    nprobe = min(nlist, 5)
    kw_sets = [dict(), dict(id_range=(3, 400)), dict(sorted_ids=np.arange(1, 900, 3)), dict(sorted_ids=np.arange(1, 900, 3), negate=True)]
    shapes = [(nq, k) for nq in (1, W - 1, W + 1, 64) if nq > 0 for k in (1, 10)] + [(W + 1, 256 // W), (W + 1, 256 // W + 1)]
    want = {}
    for nq, k in shapes:
        want[(nq, k)] = plain.search(xq[:nq], k, nprobe=nprobe)
    for j, kw in enumerate(kw_sets):
        want[("filter", j)] = plain.search(xq, 10, nprobe=nprobe, **kw)
    broadcast = nlist < W

    def rank(r, world):
        ix = _ivf_index(kind, metric, d, nlist, nbits)
        if not broadcast or r == W - 1:
            ix.set_trained_state(blob)
        sh = world.connect(ix, r)
        if broadcast:  # nlist < W: the state comes from the last rank, and some ranks own no list
            sh.broadcast_state(W - 1)
        sh.add(xs[r][:h[r]], ids[r][:h[r]])
        world.barrier.wait()
        rest = xs[r][h[r]:]
        xd, idd = torch.from_numpy(rest.copy()).cuda(), torch.from_numpy(ids[r][h[r]:].copy()).cuda()
        torch.cuda.synchronize()
        sh.add_device(len(rest), xd.data_ptr() if len(rest) else None, idd.data_ptr() if len(rest) else None)
        out = {"range": sh.list_range(), "lists": ix.export_lists(nlist, with_vectors=kind == "flat")}
        seq = 0
        for nq, k in shapes:
            out[(nq, k)] = sh.search(xq[:nq], k, seq=seq, nprobe=nprobe)
            seq += 1
        for j, kw in enumerate(kw_sets):
            out[("filter", j)] = sh.search(xq, 10, seq=seq, nprobe=nprobe, **kw)
            seq += 1
        # device pointers: four batches in flight on two streams over two lanes
        qd = torch.from_numpy(xq).cuda()
        sts = [torch.cuda.Stream(device="cuda:0") for _ in range(2)]
        dev_out = [(torch.empty((64, 10), dtype=torch.float32, device="cuda:0"), torch.empty((64, 10), dtype=torch.int64, device="cuda:0"))
                   for _ in range(4)]
        sp, _keep = b200vs.make_search_params(nprobe=nprobe)
        torch.cuda.synchronize()
        for i in range(4):
            sh.search_device(64, qd.data_ptr(), 10, dev_out[i][0].data_ptr(), dev_out[i][1].data_ptr(), stream=sts[i % 2].cuda_stream, sp=sp, seq=seq)
            seq += 1
        torch.cuda.synchronize()
        out["device"] = [(a.cpu().numpy(), b.cpu().numpy()) for a, b in dev_out]
        # concurrent caller threads with explicit sequence numbers, started out of order
        got = {}

        def call(q):
            got[q] = sh.search(xq, 10, seq=q, nprobe=nprobe)
        ths = [threading.Thread(target=call, args=(seq + t,)) for t in (2, 0, 3, 1)]
        for t in ths:
            t.start()
        for t in ths:
            t.join()
        out["threads"] = [got[seq + t] for t in range(4)]
        sh.close()
        return out

    res = run_world(W, rank)
    per = -(-nlist // W)
    for r, o in enumerate(res):
        b, e = o["range"]
        assert (b, e) == (min(nlist, per * r), min(nlist, per * (r + 1))), f"rank {r}: list range {(b, e)}"
        off, vec, _, lid = o["lists"]
        lens = np.diff(off)
        assert lens[:b].sum() == 0 and lens[e:].sum() == 0, f"rank {r} holds rows of lists it does not own"
        for l in range(b, e):
            assert np.array_equal(lid[off[l]:off[l + 1]], p_ids[p_off[l]:p_off[l + 1]]), f"rank {r} list {l}: ids or arrival order differ"
            if kind == "flat":
                assert np.array_equal(vec[off[l]:off[l + 1]].view(np.uint32), p_vec[p_off[l]:p_off[l + 1]].view(np.uint32)), f"rank {r} list {l}: rows differ"
        for key, w in want.items():
            _assert_same(o[key], w, f"rank {r} search {key}")
        for i, got in enumerate(o["device"]):
            _assert_same(got, want[(64, 10)], f"rank {r} device batch {i}")
        for i, got in enumerate(o["threads"]):
            _assert_same(got, want[(64, 10)], f"rank {r} threaded batch {i}")


@pytest.mark.parametrize("metric", (L2, IP, COSINE))
def test_ivf_flat_matches_plain_index(metric):
    _run("case_ivf", "flat", metric, "uneven", "normal")


@pytest.mark.parametrize("metric", (L2, IP))
def test_ivf_flat_exact_ties(metric):
    _run("case_ivf", "flat", metric, "uneven", "ties")


def test_ivf_flat_fewer_lists_than_ranks():
    _run("case_ivf", "flat", L2, "few", "normal", worlds=(5, 8))


@pytest.mark.parametrize("nbits", (8, 4))
def test_ivf_pq_matches_plain_index(nbits):
    _run("case_ivf", "pq", L2, "uneven", "normal", nbits)


# ---------------------------------------------------------------------------------------------
# 4. row-sharded Flat and HNSW
# ---------------------------------------------------------------------------------------------
def _pair_ids(W):
    cand = np.arange(1, 1000, dtype=np.int64) + 10 ** 7
    own = shard_py.row_owner(cand, W)
    return cand[own == 0][0], cand[own == W - 1][0]


def case_rows_flat(W, metric):
    d = 24
    rng = np.random.default_rng(77 + W)
    n = _row_counts(W, 900)
    xs = [rng.standard_normal((m, d)).astype(np.float32) for m in n]
    ids = [rng.choice(10 ** 6, m, replace=False).astype(np.int64) + r * 10 ** 6 for r, m in enumerate(n)]
    xq = rng.standard_normal((40, d)).astype(np.float32)
    if metric == IP:  # ip 2e-9 (id a, owned by rank 0) and 1e-9 (id b, owned by rank W - 1): both 1 - ip round to 1
        a, b = _pair_ids(W)
        for r in range(1, W):
            xs[r][:, 0] = -1.0  # every other row scores ip < 0 against e0
        for j, (rid, v) in enumerate(((a, 2e-9), (b, 1e-9))):
            xs[W - 1][j] = 0
            xs[W - 1][j, 0] = np.float32(v)
            ids[W - 1][j] = rid
        xq[:] = 0
        xq[:, 0] = 1
    plain = b200vs.Index(FLAT, metric, d)
    plain.add(np.concatenate(xs), np.concatenate(ids))
    shapes = [(nq, k) for nq in (1, W - 1, W + 1, 40) if nq > 0 for k in (1, 10)] + [(W + 1, 256 // W), (W + 1, 256 // W + 1), (7, 300)]
    Dp, _ = plain.search(xq[:1], 150)
    radius = float(Dp[0, -1])
    want = {s: plain.search(xq[:s[0]], s[1]) for s in shapes}
    want["range"] = plain.range_search(xq, radius, 64)

    def rank(r, world):
        ix = b200vs.Index(FLAT, metric, d)
        sh = world.connect(ix, r)
        sh.add(xs[r], ids[r])
        out = {s: sh.search(xq[:s[0]], s[1]) for s in shapes}
        out["range"] = sh.range_search(xq, radius, 64)
        sh.close()
        return out

    for r, o in enumerate(run_world(W, rank)):
        for key, w in want.items():
            _assert_same(o[key], w, f"rank {r} {key}")
    if metric == IP:
        I = want[(W + 1, 10)][1]
        assert (I[:, 0] == a).all() and (I[:, 1] == b).all()


@pytest.mark.parametrize("metric", (L2, IP, COSINE))
def test_rows_flat_matches_plain_index(metric):
    _run("case_rows_flat", metric)


def case_rows_hnsw(W, metric):
    d = 16
    rng = np.random.default_rng(5 + W)
    n = _row_counts(W, 500)
    xs = [rng.standard_normal((m, d)).astype(np.float32) for m in n]
    ids = [rng.choice(10 ** 6, m, replace=False).astype(np.int64) + r * 10 ** 6 for r, m in enumerate(n)]
    allx, alli = np.concatenate(xs), np.concatenate(ids)
    own = shard_py.row_owner(alli, W)
    xq = rng.standard_normal((W + 1, d)).astype(np.float32)
    cap = len(alli)
    for batched in (False, True):
        parts = []
        for r in range(W):  # standalone graphs of each rank's rows, in arrival order
            p = b200vs.Index(HNSW, metric, d, hnsw_m=8, hnsw_efc=40, max_elements=cap)
            if (own == r).any():
                if batched:
                    p.add_batched(allx[own == r], alli[own == r], 32)
                else:
                    p.add(allx[own == r], alli[own == r])
            parts.append((p.search(xq, 10, efsearch=32), p.get_trained_state()))
        want = shard_py.merge_topk(np.stack([p[0][0] for p in parts]), np.stack([p[0][1] for p in parts]), 10)

        def rank(r, world):
            g = b200vs.Index(HNSW, metric, d, hnsw_m=8, hnsw_efc=40, max_elements=cap)
            sh = world.connect(g, r)
            if batched:
                sh.hnsw_add_batched(xs[r], ids[r], 32)
            else:
                sh.add(xs[r], ids[r])
            out = sh.search(xq, 10, efsearch=32), g.get_trained_state()
            sh.close()
            return out

        for r, (got, state) in enumerate(run_world(W, rank)):
            assert np.array_equal(state, parts[r][1]), f"batched {batched}: rank {r}'s graph differs from its standalone graph"
            _assert_same(got, want, f"batched {batched}: rank {r} search")


@pytest.mark.parametrize("metric", (L2, COSINE))
def test_rows_hnsw_matches_merged_standalone_graphs(metric):
    _run("case_rows_hnsw", metric)


# ---------------------------------------------------------------------------------------------
# 5. sharded range search against the float32 restatement on the gathered rows
# ---------------------------------------------------------------------------------------------
def case_range(W, kind):
    from test_gpu_exact_edges import range_expect
    d = 16
    rng = np.random.default_rng(31 + W)
    n = _row_counts(W, 600)
    xs = [rng.standard_normal((m, d)).astype(np.float32) for m in n]
    ids = [np.arange(m, dtype=np.int64) * W + r + 1 for r, m in enumerate(n)]
    allx, alli = np.concatenate(xs), np.concatenate(ids)
    xq = rng.standard_normal((W + 1, d)).astype(np.float32)
    xq[-1] = 50  # far from every row: zero hits
    nlist = 2 * W + 1
    cent = allx[rng.choice(len(allx), nlist, replace=False)].copy()
    blob = b200vs.ivf_state_blob(cent, L2)
    # radius: ~120 hits for the first query, over max_results 64 for most queries
    radius = float(np.sort(((allx - xq[0]) ** 2).sum(1))[120])

    def rank(r, world):
        if kind == "rows":
            ix = b200vs.Index(FLAT, L2, d)
        else:
            ix = b200vs.Index(IVF_FLAT, L2, d, nlist=nlist)
            ix.set_trained_state(blob)
        sh = world.connect(ix, r)
        sh.add(xs[r], ids[r])
        kw = {} if kind == "rows" else {"nprobe": nlist}
        out = [sh.range_search(xq, radius, mr, **kw) for mr in (64, 4096)]
        out.append(sh.range_search(xq, float("nan"), 16, **kw))
        sh.close()
        return out

    for r, o in enumerate(run_world(W, rank)):
        for (D, I, C), mr in zip(o[:2], (64, 4096)):
            for qi in range(len(xq)):
                wi, wd, hits = range_expect(allx, alli, xq[qi], L2, radius, mr)
                assert C[qi] == len(wi), f"rank {r} max_results {mr} query {qi}: {C[qi]} hits, expected {len(wi)}"
                assert np.array_equal(I[qi, :C[qi]], wi) and (I[qi, C[qi]:] == -1).all(), f"rank {r} max_results {mr} query {qi}: ids"
                assert np.array_equal(D[qi, :C[qi]].view(np.uint32), wd.view(np.uint32)), f"rank {r} max_results {mr} query {qi}: distances"
                assert (D[qi, C[qi]:] == 0).all()
                if mr == 64 and qi == 0:
                    assert hits > 64, "the first query must overflow max_results"
                if qi == len(xq) - 1:
                    assert hits == 0
        D, I, C = o[2]
        assert (C == 0).all() and (I == -1).all(), f"rank {r}: a NaN radius admits no row"


@pytest.mark.parametrize("kind", ("rows", "lists"))
def test_range_matches_restatement(kind):
    _run("case_range", kind)


# ---------------------------------------------------------------------------------------------
# 6. collectives of the write path
# ---------------------------------------------------------------------------------------------
def case_write_path(W):
    import torch
    d = 16
    nlist = 2 * W + 1
    rng = np.random.default_rng(9 + W)
    n = _row_counts(W, 500)
    xs = [rng.standard_normal((m, d)).astype(np.float32) for m in n]
    ids = [np.arange(m, dtype=np.int64) * W + r + 1 for r, m in enumerate(n)]
    allx, alli = np.concatenate(xs), np.concatenate(ids)
    cent = allx[rng.choice(len(allx), nlist, replace=False)].copy()
    blob = b200vs.ivf_state_blob(cent, L2)
    plain = b200vs.Index(IVF_FLAT, L2, d, nlist=nlist)
    plain.set_trained_state(blob)
    plain.add(allx, alli)
    p_off, _, _, p_ids = plain.export_lists(nlist)
    list_of = {int(i): l for l in range(nlist) for i in p_ids[p_off[l]:p_off[l + 1]]}
    per = -(-nlist // W)
    owner_of = {i: l // per for i, l in list_of.items()}
    one = next(i for i in alli.tolist() if owner_of[i] == max(owner_of.values()))
    several = [next(i for i in alli.tolist() if owner_of[i] == o) for o in sorted(set(owner_of.values()))]
    # upsert of a row that moves: its new vector is a copy of a row of a list owned by another rank
    mover = next(i for i in alli.tolist() if i not in (one, *several))
    target = next(i for i in alli.tolist() if owner_of[i] != owner_of[mover])
    x_new = allx[alli.tolist().index(target)].copy()
    xq = rng.standard_normal((W + 1, d)).astype(np.float32)

    def rank(r, world):
        ix = b200vs.Index(IVF_FLAT, L2, d, nlist=nlist)
        if r == W - 1:
            ix.set_trained_state(blob)
        sh = world.connect(ix, r)
        sh.broadcast_state(W - 1)
        out = {"state": ix.get_trained_state()}
        # bulk build: plan every rank's rows, commit, then add: the owned lists are pre-sized and nothing grows
        xd = torch.from_numpy(xs[r].copy()).cuda() if n[r] else None
        idd = torch.from_numpy(ids[r].copy()).cuda() if n[r] else None
        torch.cuda.synchronize()
        if n[r]:
            sh.plan_add_device(n[r], xd.data_ptr())
        sh.plan_commit()
        mem = ix.get_memory_size()
        sh.add_device(n[r], xd.data_ptr() if n[r] else None, idd.data_ptr() if n[r] else None)
        out["mem"] = (mem, ix.get_memory_size())
        out["lists"] = ix.export_lists(nlist, with_vectors=False)
        out["range"] = sh.list_range()
        out["rm_one"] = sh.delete(np.array([one], np.int64))
        out["rm_several"] = sh.delete(np.array(several, np.int64))
        out["rm_none"] = _status(lambda: sh.delete(np.array([-5, -6], np.int64)))
        out["count"] = ix.get_count()
        # upsert as remove + add: the row moves to the owner of its new list
        out["upsert_rm"] = sh.delete(np.array([mover], np.int64))
        if r == 0:
            sh.add(x_new[None], np.array([mover], np.int64))
        else:
            sh.add(np.zeros((0, d), np.float32), np.zeros(0, np.int64))
        out["upsert"] = ix.export_lists(nlist, with_vectors=False)
        out["search"] = sh.search(xq, 10, nprobe=nlist)
        sh.close()
        return out

    res = run_world(W, rank)
    removed_ids = {one, *several}
    for r, o in enumerate(res):
        assert np.array_equal(o["state"], res[W - 1]["state"]), f"rank {r}: broadcast state from root {W - 1} differs"
        m0, m1 = o["mem"]
        assert m0 == m1, f"rank {r}: memory grew from {m0} to {m1} bytes after plan_commit"
        b, e = o["range"]
        off = o["lists"][0]
        lens = np.diff(off)
        assert lens[:b].sum() == 0 and lens[e:].sum() == 0, f"rank {r} holds rows of lists it does not own"
        assert np.array_equal(lens[b:e], np.diff(p_off)[b:e]), f"rank {r}: list sizes differ from the plain index"
        # plan_commit reserved exactly the lists this rank owns: a single index reserving those holds as many bytes
        owned = np.diff(p_off).copy()
        owned[:b], owned[e:] = 0, 0
        ref = b200vs.Index(IVF_FLAT, L2, d, nlist=nlist)
        ref.set_trained_state(blob)
        ref.reserve_lists(owned)
        assert m0 == ref.get_memory_size(), f"rank {r}: {m0} bytes after plan_commit, {ref.get_memory_size()} for its own lists"
        assert o["rm_one"] == 1 and o["rm_several"] == len(set(several) - {one}), f"rank {r}: removed {o['rm_one']}, {o['rm_several']}"
        assert o["rm_none"] == b200vs.EVECTOR_INVALID, f"rank {r}: removing unknown ids returned {o['rm_none']}"
        assert o["upsert_rm"] == 1
    total = sum(o["count"] for o in res)
    assert total == len(alli) - len(removed_ids)
    removed_ids.add(mover)
    # the moved row lives on the owner of its new list, with the rows of every other rank unchanged
    keep = ~np.isin(alli, list(removed_ids))
    ref = b200vs.Index(IVF_FLAT, L2, d, nlist=nlist)
    ref.set_trained_state(blob)
    ref.add(allx[keep], alli[keep])
    ref.add(x_new[None], np.array([mover], np.int64))
    want = ref.search(xq, 10, nprobe=nlist)
    lt = list_of[target]
    holder = [r for r, o in enumerate(res) if mover in o["upsert"][3].tolist()]
    assert holder == [lt // per], f"moved row held by ranks {holder}, expected rank {lt // per}"
    for r, o in enumerate(res):
        _assert_same(o["search"], want, f"rank {r}: search after upsert")


def test_write_path_collectives():
    _run("case_write_path")


def case_shard_train(W):
    d = 16
    nlist = 2 * W
    rng = np.random.default_rng(3 + W)
    xs = [rng.standard_normal((400 + 50 * r, d)).astype(np.float32) for r in range(W)]
    parts = []
    for r in range(W):  # standalone trains of nlist / W centroids on each rank's rows
        p = b200vs.Index(IVF_FLAT, L2, d, nlist=nlist // W)
        p.train(xs[r])
        parts.append(p.get_trained_state()[32:].view(np.float32).reshape(nlist // W, d))
    want = np.concatenate(parts)

    def rank(r, world):
        ix = b200vs.Index(IVF_FLAT, L2, d, nlist=nlist)
        sh = world.connect(ix, r)
        out = {"short": _status(lambda: sh.train(xs[r][:nlist // W - 1] if r == W - 1 else xs[r])),
               "untrained root": _status(lambda: sh.broadcast_state(W - 1)), "trained": ix.is_trained()}
        sh.train(xs[r])
        out["cent"] = ix.get_trained_state()[32:].view(np.float32).reshape(nlist, d)
        sh.close()
        return out

    for r, o in enumerate(run_world(W, rank)):
        assert o["short"] == b200vs.EILLEGAL_PARAMETERS and o["untrained root"] == b200vs.EVECTOR_NOT_TRAIN and not o["trained"], \
            f"rank {r}: refusals {o['short']}, {o['untrained root']}"
        assert np.array_equal(o["cent"].view(np.uint32), want.view(np.uint32)), f"rank {r}: centroids differ from the standalone trains"


def test_shard_train():
    _run("case_shard_train")


# ---------------------------------------------------------------------------------------------
# 7. status agreement: a refusal on one rank is every rank's, and no rank changes
# ---------------------------------------------------------------------------------------------
def case_status(W):
    d = 16
    rng = np.random.default_rng(17 + W)
    xs = [rng.standard_normal((200, d)).astype(np.float32) for _ in range(W)]
    ids = [np.arange(200, dtype=np.int64) * W + r + 1 for r in range(W)]
    xq = rng.standard_normal((3, d)).astype(np.float32)
    cand = np.arange(10 ** 8, 10 ** 8 + 400 * W, dtype=np.int64)
    to_last = cand[shard_py.row_owner(cand, W) == W - 1][:60]

    def rank(r, world):
        out = {}
        # FLAT: rank 0 re-adds an id that already lives on its owner
        ix = b200vs.Index(FLAT, L2, d)
        sh = world.connect(ix, r)
        sh.add(xs[r], ids[r])
        before = (ix.get_count(), ix.get_memory_size())
        # ranks 0 and 1 each send a row with one new id: its owner receives the id twice
        out["dup"] = _status(lambda: sh.add(xs[r][:1], np.array([10 ** 9], np.int64)) if r < 2 else sh.add(xs[r][:0], ids[r][:0]))
        out["dup_state"] = before == (ix.get_count(), ix.get_memory_size())
        for what, fn in (("mr0", lambda: sh.range_search(xq, 1.0, 0)), ("mr4097", lambda: sh.range_search(xq, 1.0, 4097))):
            out[what] = _status(fn)
        out["after"] = sh.search(xq, 5)
        sh.close()
        # HNSW: max_elements exceeded on the last rank only
        g = b200vs.Index(HNSW, L2, d, hnsw_m=8, hnsw_efc=40, max_elements=40)
        sh = world.connect(g, r)
        before = (g.get_count(), g.get_memory_size())
        # rank 0 sends 60 rows that all belong to the last rank, whose max_elements is 40
        out["cap"] = _status(lambda: sh.add(xs[r][:60], to_last) if r == 0 else sh.add(xs[r][:0], ids[r][:0]))
        out["cap_state"] = before == (g.get_count(), g.get_memory_size())
        out["hnsw_range"] = _status(lambda: sh.range_search(xq, 1.0, 8))
        sh.add(xs[r][:5], ids[r][:5])
        out["hnsw_after"] = g.get_count()
        sh.close()
        return out

    res = run_world(W, rank)
    for r, o in enumerate(res):
        assert o["dup"] == b200vs.EVECTOR_ID_DUPLICATED, f"rank {r}: repeated id returned {o['dup']}"
        assert o["dup_state"] and o["cap_state"], f"rank {r}: a refused add changed the index"
        assert o["mr0"] == o["mr4097"] == b200vs.EILLEGAL_PARAMETERS
        assert o["cap"] != b200vs.OK and o["cap"] == res[0]["cap"], f"rank {r}: max_elements refusal {o['cap']}"
        assert o["hnsw_range"] == b200vs.EVECTOR_NOT_SUPPORT
    plain = b200vs.Index(FLAT, L2, d)
    plain.add(np.concatenate(xs), np.concatenate(ids))
    want = plain.search(xq, 5)
    for r, o in enumerate(res):
        _assert_same(o["after"], want, f"rank {r}: search after the refusals")
    assert sum(o["hnsw_after"] for o in res) == 5 * W


def test_status_agreement():
    _run("case_status")
