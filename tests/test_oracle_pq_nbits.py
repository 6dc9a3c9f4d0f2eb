"""The oracle's IVF-PQ at nbits 1-8 (CPU only): sub-byte codebooks go through the 8-bit oracle padded to 256 codewords
(tests/pq_codes.py).  Pinned here, independently of the engine, against numpy restatements:
  * packed codes == numpy packbits(bitorder='little') of a numpy FP32 argmin encoder (first minimum wins), pad bits zero;
  * search == a numpy FP32 restatement (sequential over dsub for the LUT entries, sequential over m for the row sums,
    results in (distance, id) order), bit for bit, for L2, IP and cosine."""
import numpy as np
import pytest

import pq_codes
from oracle_lib import COSINE, IP, L2

# (nbits, M, d): code_size = ceil(M * nbits / 8) is ragged (pad bits in the last byte) except where noted
CASES = [(1, 5, 20), (2, 7, 14), (3, 5, 20), (4, 7, 28), (5, 12, 24), (6, 3, 12), (7, 9, 9), (8, 6, 12), (4, 8, 16), (2, 4, 8)]


def seq_ip(a, b):
    """<a, b> over the last axis, summed left to right in FP32."""
    acc = np.zeros(np.broadcast(a[..., 0], b[..., 0]).shape, np.float32)
    for i in range(a.shape[-1]):
        acc = (acc + (a[..., i] * b[..., i]).astype(np.float32)).astype(np.float32)
    return acc


def np_encode(cb, cent, x, asg):
    M, ksub, dsub = cb.shape
    r = (x - cent[asg]).astype(np.float32)
    codes = np.zeros((len(x), M), np.uint8)
    for m in range(M):
        acc = np.zeros((len(x), ksub), np.float32)
        for i in range(dsub):
            t = (r[:, None, m * dsub + i] - cb[m][None, :, i]).astype(np.float32)
            acc = (acc + (t * t).astype(np.float32)).astype(np.float32)
        codes[:, m] = np.argmin(acc, axis=1)
    return codes


def np_search(o, metric, cent, cb, off, codes, ids, xq, k, nprobe):
    M, ksub, dsub = cb.shape
    nlist = cent.shape[0]
    D = np.zeros((len(xq), k), np.float32)
    I = np.full((len(xq), k), -1, np.int64)
    for qi, q in enumerate(xq):
        Q = o.normalize_faiss(q[None])[0] if metric == COSINE else q.astype(np.float32)
        coarse = np.array([o.l2sqr(Q, c) if metric == L2 else o.ip(Q, c) for c in cent], np.float32)
        probes = np.lexsort((np.arange(nlist), coarse if metric == L2 else -coarse))[:nprobe]
        sim = seq_ip(Q.reshape(M, 1, dsub), cb)  # [M, ksub]
        vals, vids = [], []
        for l in probes:
            tab = sim
            if metric == L2:  # T = ||cw||^2 + 2 <c_m, cw>, then T - 2 sim
                pre = (seq_ip(cb, cb) + np.float32(2) * seq_ip(cent[l].reshape(M, 1, dsub), cb)).astype(np.float32)
                tab = (pre + np.float32(-2) * sim).astype(np.float32)
            rows = np.arange(off[l], off[l + 1])
            v = np.full(len(rows), coarse[l], np.float32)
            for m in range(M):
                v = (v + tab[m, codes[rows, m].astype(np.int64)]).astype(np.float32)
            vals.append(v)
            vids.append(ids[rows])
        v, vi = np.concatenate(vals), np.concatenate(vids)
        order = np.lexsort((vi, v if metric == L2 else -v))[:k]
        c = len(order)
        I[qi, :c] = vi[order]
        D[qi, :c] = v[order] if metric == L2 else (np.float32(1) - v[order]).astype(np.float32)
    return D, I


def lists(o, metric, n, d, nlist, M, nbits, seed):
    rng = np.random.default_rng(seed)
    x = rng.standard_normal((n, d)).astype(np.float32)
    stored = o.normalize_faiss(x) if metric == COSINE else x
    cent = (stored[rng.choice(n, nlist, replace=False)] + 0.1 * rng.standard_normal((nlist, d))).astype(np.float32)
    cb = (0.5 * rng.standard_normal((M, 1 << nbits, d // M))).astype(np.float32)
    asg = o.assign(metric, stored, cent)
    order = np.argsort(asg, kind="stable")
    off = np.concatenate([[0], np.cumsum(np.bincount(asg, minlength=nlist))]).astype(np.int64)
    return stored[order], asg[order], np.arange(1, n + 1, dtype=np.int64)[order], cent, cb, off


def test_pack_layout():
    """LSB first: at 4 bits code 2j is the low nibble of byte j; unused high bits of the last byte are zero."""
    assert pq_codes.pack(np.array([[1, 2, 3]], np.uint8), 4).tolist() == [[0x21, 0x03]]
    assert pq_codes.pack(np.array([[5, 7, 1]], np.uint8), 3).tolist() == [[0b01111101, 0x00]]
    assert pq_codes.pack(np.array([[1, 0, 1, 1, 0, 0, 0, 0, 1]], np.uint8), 1).tolist() == [[0b00001101, 0b1]]
    c = np.random.default_rng(0).integers(0, 256, (9, 5)).astype(np.uint8)
    assert np.array_equal(pq_codes.pack(c, 8), c)


@pytest.mark.parametrize("nbits,M,d", CASES)
def test_packed_codes_equal_numpy_encoder(oracle, nbits, M, d):
    n, nlist = 600, 4
    X, asg, ids, cent, cb, off = lists(oracle, L2, n, d, nlist, M, nbits, seed=nbits * 31 + M)
    want = np_encode(cb, cent, X, asg)
    assert want.max() < (1 << nbits)
    packed = pq_codes.ivfpq_encode(oracle, cb, cent, X, asg)
    assert packed.shape == (n, (M * nbits + 7) // 8)
    assert np.array_equal(packed, pq_codes.pack(want, nbits))
    assert not np.unpackbits(packed, axis=1, bitorder="little")[:, M * nbits:].any(), "pad bits must be zero"
    assert np.array_equal(pq_codes.unpack(packed, M, nbits), want)
    # the issue-level formula of the layout, spelled out once more on the numpy codes
    ref = np.packbits(np.unpackbits(want[:, :, None], axis=2, bitorder="little")[:, :, :nbits].reshape(n, -1), axis=1, bitorder="little")
    assert np.array_equal(packed, ref)


@pytest.mark.parametrize("metric", [L2, IP, COSINE])
@pytest.mark.parametrize("nbits,M,d", CASES)
def test_search_equals_numpy_restatement(oracle, metric, nbits, M, d):
    n, nlist, nprobe, k = 500, 5, 3, 25
    X, asg, ids, cent, cb, off = lists(oracle, metric, n, d, nlist, M, nbits, seed=nbits * 17 + M + metric)
    packed = pq_codes.ivfpq_encode(oracle, cb, cent, X, asg)
    xq = np.random.default_rng(metric + nbits).standard_normal((4, d)).astype(np.float32)
    Do, Io = pq_codes.ivfpq_search(oracle, metric, cent, cb, off, packed, ids, xq, k, nprobe, nthreads=2)
    Dn, In = np_search(oracle, metric, cent, cb, off, pq_codes.unpack(packed, M, nbits), ids, xq, k, nprobe)
    assert (Io >= 0).all()
    assert np.array_equal(Io, In)
    assert np.array_equal(Do.view(np.uint32), Dn.view(np.uint32))
