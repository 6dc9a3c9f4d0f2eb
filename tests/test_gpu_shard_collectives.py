"""The collective write path and the read prologue of b200vs_shard_* at a world of one (csrc/shard.cu).

A world of one runs the same routing, status agreement, trainer and read prologue as a world of W, with the NCCL calls
left out, so these checks cover the W-rank code paths on one GPU:
  - a list-sharded add (host and device rows, several chunks, one chunk of more than 1024 routing tiles) lays its lists
    out byte for byte as a plain add of the same rows;
  - the IVF-Flat sharded trainer gives b200vs_train's trained state, and refuses too few rows, no rows and a null x
    while the index stays untrained;
  - broadcast_state from an untrained root refuses with EVECTOR_NOT_TRAIN;
  - a refused or k = 0 top-k search uses up its sequence number, so a later batch never waits for it."""
import ctypes

import numpy as np
import pytest

import b200vs
import pq_codes
from b200vs import COSINE, EILLEGAL_PARAMETERS, EVECTOR_NOT_TRAIN, IVF_FLAT, IVF_PQ, L2, B200VSError
from gpu_util import require_gpu

pytestmark = pytest.mark.gpu
D, NLIST = 16, 16
BIG = 300001  # > 1024 routing tiles of 256 rows, and not a multiple of 256


@pytest.fixture(autouse=True)
def _gpu():
    require_gpu()


def _rows(n, seed):
    return np.random.default_rng(seed).standard_normal((n, D)).astype(np.float32)


def _index(kind, metric, nbits):
    if kind == IVF_PQ:
        return b200vs.Index(IVF_PQ, metric, D, nlist=NLIST, pq_m=4, pq_nbits=nbits)
    return b200vs.Index(IVF_FLAT, metric, D, nlist=NLIST)


def _refused(code, fn, *args, **kw):
    with pytest.raises(B200VSError) as e:
        fn(*args, **kw)
    assert e.value.code == code, e.value.msg
    return e.value.msg


@pytest.mark.parametrize("kind,metric,nbits", [(IVF_FLAT, L2, 0), (IVF_FLAT, COSINE, 0), (IVF_PQ, L2, 8), (IVF_PQ, L2, 4)])
def test_list_sharded_add_lays_out_lists_as_a_plain_add(kind, metric, nbits):
    import torch
    trainer = _index(kind, metric, nbits)
    trainer.train(_rows(max(256 * NLIST, 256 << max(nbits, 1)) + 1000, 1))
    state = trainer.get_trained_state()
    ref, ix = _index(kind, metric, nbits), _index(kind, metric, nbits)
    ref.set_trained_state(state)
    ix.set_trained_state(state)
    sh = b200vs.Shard(ix, 0, 1, None)
    xb = _rows(BIG + 7000, 2)
    ids = np.arange(100, 100 + xb.shape[0], dtype=np.int64)
    chunks = [(0, 3000, "host"), (3000, 5000, "device"), (5000, 5000, "host"), (5000, 5000 + BIG, "device"), (5000 + BIG, xb.shape[0], "host")]
    for a, b, where in chunks:
        if b > a:
            ref.add(xb[a:b], ids[a:b])
        if where == "host":
            sh.add(xb[a:b], ids[a:b])
        else:
            xd, idd = torch.from_numpy(xb[a:b]).cuda(), torch.from_numpy(ids[a:b]).cuda()
            torch.cuda.synchronize()
            sh.add_device(b - a, xd.data_ptr() if b > a else None, idd.data_ptr() if b > a else None)
    assert ix.get_count() == ref.get_count() == xb.shape[0]
    code_size = pq_codes.code_size(4, nbits) if kind == IVF_PQ else 0
    got = ix.export_lists(NLIST, with_vectors=kind == IVF_FLAT, code_size=code_size)
    want = ref.export_lists(NLIST, with_vectors=kind == IVF_FLAT, code_size=code_size)
    for g, w, what in zip(got, want, ("list offsets", "vectors", "codes", "ids")):
        if w is None:
            continue
        assert g.tobytes() == w.tobytes(), f"{what} differ from a plain add's"
    sh.close()


@pytest.mark.parametrize("metric", [L2, COSINE])
def test_ivf_flat_shard_train_equals_train_and_refuses_alike(metric):
    x = _rows(5000, 7)
    ref = _index(IVF_FLAT, metric, 0)
    ref.train(x)
    ix = _index(IVF_FLAT, metric, 0)
    sh = b200vs.Shard(ix, 0, 1, None)
    _refused(EILLEGAL_PARAMETERS, sh.train, x[:0])
    with pytest.raises(B200VSError) as e:
        b200vs._check(b200vs.lib().b200vs_shard_train(sh.h, 100, None))  # the raw ABI: rows claimed, null x
    assert e.value.code == EILLEGAL_PARAMETERS
    _refused(EILLEGAL_PARAMETERS, sh.train, x[:NLIST - 1])
    assert not ix.is_trained(), "a refused shard_train must leave the index untrained"
    sh.train(x)
    assert ix.is_trained()
    assert ix.get_trained_state().tobytes() == ref.get_trained_state().tobytes(), "shard_train's state differs from train's"
    sh.close()


def test_broadcast_state_from_an_untrained_root_refuses():
    ix = _index(IVF_FLAT, L2, 0)
    sh = b200vs.Shard(ix, 0, 1, None)
    _refused(EVECTOR_NOT_TRAIN, sh.broadcast_state, 0)
    assert not ix.is_trained()
    sh.close()


@pytest.mark.parametrize("device", [False, True])
def test_refused_and_empty_topk_searches_use_their_sequence_number(device):
    import torch
    ix = _index(IVF_FLAT, L2, 0)
    ix.train(_rows(5000, 3))
    ix.add(_rows(4000, 4), np.arange(4000, dtype=np.int64))
    sh = b200vs.Shard(ix, 0, 1, None)
    nq, k = 8, 5
    xq = _rows(nq, 5)
    want_d, want_i = ix.search(xq, k, nprobe=4)
    sp, _ = b200vs.make_search_params(nprobe=4)
    xq_t = torch.from_numpy(xq).cuda()
    torch.cuda.synchronize()
    od = np.zeros((nq, k), np.float32)
    oi = np.zeros((nq, k), np.int64)
    od_t = torch.zeros((nq, k), dtype=torch.float32, device="cuda")
    oi_t = torch.zeros((nq, k), dtype=torch.int64, device="cuda")
    if device:
        xp, dp, ip = xq_t.data_ptr(), od_t.data_ptr(), oi_t.data_ptr()
    else:
        xp, dp, ip = xq.ctypes.data, od.ctypes.data, oi.ctypes.data

    def call(seq, nq_=nq, k_=k, xp_=xp, dp_=dp, ip_=ip):
        if device:
            rc = b200vs.lib().b200vs_shard_search_device(sh.h, seq, nq_, xp_, k_, ctypes.byref(sp), dp_, ip_, None)
        else:
            rc = b200vs.lib().b200vs_shard_search(sh.h, seq, nq_, xp_, k_, ctypes.byref(sp), dp_, ip_)
        return rc, b200vs.lib().b200vs_last_error().decode()

    def results():
        if device:
            torch.cuda.synchronize()
            return od_t.cpu().numpy(), oi_t.cpu().numpy()
        return od, oi

    seq = 0
    for name, kw, rc_want in [("k = 0", dict(k_=0), 0), ("null output", dict(ip_=None), EILLEGAL_PARAMETERS),
                              ("nq = 0", dict(nq_=0), EILLEGAL_PARAMETERS)]:
        rc, msg = call(seq, **kw)
        assert rc == rc_want, f"{name}: {rc} {msg}"
        # asserted before the next sequence number is tried: if the refused call had left `seq` unused, the batch
        # seq + 1 would wait for it forever
        rc, msg = call(seq)
        assert rc == EILLEGAL_PARAMETERS and "sequence number already used" in msg, f"{name}: seq {seq} was not used up ({rc} {msg})"
        rc, msg = call(seq + 1)
        assert rc == 0, f"{name}: the next batch failed: {msg}"
        got_d, got_i = results()
        assert np.array_equal(got_i, want_i) and np.array_equal(got_d.view(np.uint32), want_d.view(np.uint32))
        seq += 2
    sh.close()
