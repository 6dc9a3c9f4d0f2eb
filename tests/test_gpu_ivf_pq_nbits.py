"""IVF-PQ with sub-byte codes (nbits 1-7, and 8 as a control through the same blob path): bit-packed rows and
pq_scan_packed_kernel, on synthetic trained states as in test_gpu_ivf_pq_edges.py.  Every case checks that the exported
packed codes equal the oracle's encoder packed by numpy (tests/pq_codes.py), that the search equals the oracle's search
bit for bit, and the float64 bound on the decoded rows c[list] + concat_m cw[m][code_m].
Code-read branches of the packed kernel: code_size % 16 == 0 (16-byte loads), code_size % 4 == 0 (4-byte loads), other
(bytes); M > 128 runs full 128-code chunks before the tail chunk."""
import os
import tempfile

import numpy as np
import pytest

import b200vs
import pq_codes
from b200vs import COSINE, FLAT, IP, IVF_PQ, L2
from gpu_util import assert_same_results, recall, require_gpu
from test_gpu_ivf_pq_edges import Synth, check_range

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _gpu():
    require_gpu()


class SynthN(Synth):
    """Synth with codebooks [M, 2^nbits, d/M].  self.packed holds the exported rows as stored; self.codes holds them
    unpacked, so the float64 checks and the FP32 restatement inherited from Synth apply unchanged."""

    def __init__(self, oracle, metric, n, d, nlist, M, nbits, seed=0):
        rng = np.random.default_rng(seed)
        self.o, self.metric, self.d, self.nlist, self.M, self.nbits = oracle, metric, d, nlist, M, nbits
        xb = rng.standard_normal((n, d)).astype(np.float32)
        stored = oracle.normalize_faiss(xb) if metric == COSINE else xb
        self.cent = (stored[rng.choice(n, nlist, replace=False)] + 0.1 * rng.standard_normal((nlist, d))).astype(np.float32)
        self.cb = (0.5 * rng.standard_normal((M, 1 << nbits, d // M))).astype(np.float32)
        self.ix = b200vs.Index(IVF_PQ, metric, d, nlist=nlist, pq_m=M, pq_nbits=nbits)
        self.ix.set_trained_state(b200vs.ivfpq_state_blob(self.cent, self.cb, metric))
        self.rows = {}
        self.add(xb, np.arange(1, n + 1, dtype=np.int64))

    def export(self):
        cs = pq_codes.code_size(self.M, self.nbits)
        off, _, packed, lids = self.ix.export_lists(self.nlist, with_vectors=False, code_size=cs)
        assert off[-1] == len(self.rows) == self.ix.get_count()
        lst = np.repeat(np.arange(self.nlist), np.diff(off)).astype(np.int32)
        if len(lids):
            X = np.stack([self.rows[i] for i in lids.tolist()])
            assert np.array_equal(self.o.assign(self.metric, X, self.cent), lst), "list assignment differs from the oracle"
            assert np.array_equal(packed, pq_codes.ivfpq_encode(self.o, self.cb, self.cent, X, lst)), "codes differ from the oracle encoder"
            assert not np.unpackbits(packed, axis=1, bitorder="little")[:, self.M * self.nbits:].any(), "pad bits must be zero"
        self.off, self.packed, self.lids, self.lst = off, packed, lids, lst
        self.codes = pq_codes.unpack(packed, self.M, self.nbits)
        return off, packed, lids

    def search(self, xq, k, nprobe, **filt):
        Dg, Ig = self.ix.search(xq, k, nprobe=nprobe, **filt)
        Do, Io = pq_codes.ivfpq_search(self.o, self.metric, self.cent, self.cb, self.off, self.packed, self.lids, xq, k, nprobe, nthreads=8, **filt)
        assert_same_results(Dg, Ig, Do, Io)
        self.check_f64(xq, Dg, Ig, every_row=min(nprobe, self.nlist) == self.nlist, **filt)
        return Dg, Ig


# nbits -> M per code-read branch: code_size % 16 == 0, % 4 == 0 (not 16), neither
BRANCH_M = {1: (128, 32, 12), 2: (64, 16, 10), 3: (128, 32, 5), 4: (32, 8, 6), 5: (128, 32, 9), 6: (64, 16, 3), 7: (128, 32, 5), 8: (16, 4, 6)}
WIDTH_CASES = [(nb, M) for nb, ms in BRANCH_M.items() for M in ms]
LONG_ROWS = [(4, 256), (5, 160), (3, 200), (7, 261)]  # M > 128: code_size 128 (% 16), 100 (% 4), 75, 229


def dim_for(M):
    return M * max(1, 64 // M)


@pytest.mark.parametrize("metric", [L2, IP, COSINE])
@pytest.mark.parametrize("nbits,M", WIDTH_CASES + LONG_ROWS)
def test_widths_and_code_read_branches(oracle, metric, nbits, M):
    d = dim_for(M)
    s = SynthN(oracle, metric, 3000, d, 8, M, nbits, seed=nbits * 1000 + M)
    s.export()
    xq = np.random.default_rng(M + nbits).standard_normal((6, d)).astype(np.float32)
    s.search(xq, 50, nprobe=8)
    s.search(xq, 20, nprobe=3)
    s.search(xq, 10, nprobe=8, id_range=(500, 2500))
    s.search(xq, 10, nprobe=8, sorted_ids=np.arange(3, 3000, 7, dtype=np.int64))
    s.search(xq, 10, nprobe=8, sorted_ids=np.arange(3, 3000, 7, dtype=np.int64), negate=True)


@pytest.mark.parametrize("metric", [L2, IP])
def test_large_k(oracle, metric):
    s = SynthN(oracle, metric, 6000, 128, 4, 64, 4, seed=21 + metric)
    s.export()
    xq = np.random.default_rng(3).standard_normal((3, 128)).astype(np.float32)
    for k in (1, 129, 1024, 4096):
        s.search(xq, k, nprobe=4)


def test_shared_memory_boundary(oracle):
    """k = 4096 on a 256-thread CTA: select pool 8192 entries = 98336 B, leaving 134112 B of the 227 KB for the LUT.  At
    nbits = 7 (512 B per sub-space) M = 261 needs 133632 B and runs; M = 262 needs 134144 B and is refused on the host with
    EILLEGAL_PARAMETERS, after which the index still serves smaller k."""
    s = SynthN(oracle, IP, 5000, 261, 4, 261, 7, seed=31)
    s.export()
    xq = np.random.default_rng(32).standard_normal((2, 261)).astype(np.float32)
    s.search(xq, 4096, nprobe=4)
    t = SynthN(oracle, L2, 1500, 262, 4, 262, 7, seed=33)
    t.export()
    xq = np.random.default_rng(34).standard_normal((2, 262)).astype(np.float32)
    for call in (lambda: t.ix.search(xq, 4096, nprobe=4), lambda: t.ix.range_search(xq, 1e9, 4096, nprobe=4)):
        with pytest.raises(b200vs.B200VSError) as e:
            call()
        assert e.value.code == b200vs.EILLEGAL_PARAMETERS
    t.search(xq, 1024, nprobe=4)


@pytest.mark.parametrize("metric", [L2, IP, COSINE])
@pytest.mark.parametrize("nbits,M", [(4, 16), (3, 20)])
def test_range_search(oracle, metric, nbits, M):
    """More hits than max_results keeps the max_results closest; a radius equal to a row's raw value excludes that row."""
    s = SynthN(oracle, metric, 5000, 80, 8, M, nbits, seed=41 + metric + M)
    s.export()
    xq = np.random.default_rng(42).standard_normal((4, 80)).astype(np.float32)
    Do, Io = pq_codes.ivfpq_search(oracle, metric, s.cent, s.cb, s.off, s.packed, s.lids, xq, 5000, 8, nthreads=8)
    pos = {int(i): r for r, i in enumerate(s.lids.tolist())}
    for qi in range(len(xq)):  # the FP32 restatement the range checks use is bit-exact against the oracle
        raw = s.raw_fp32(xq[qi])[[pos[int(i)] for i in Io[qi]]]
        api = raw if metric == L2 else (np.float32(1) - raw).astype(np.float32)
        assert np.array_equal(api.view(np.uint32), Do[qi].view(np.uint32))
    radius = float(np.max(Do[:, 600]))  # >= 600 hits for every query (their spread is wide at 3 bits)
    hits = check_range(s, xq, radius, 64)
    assert min(hits) > 64
    check_range(s, xq[:1], radius, 1024)
    if metric == COSINE:
        return
    raw = s.raw_fp32(xq[0])
    order = np.argsort(raw) if metric == L2 else np.argsort(-raw)
    r = None
    for j in order[30:]:
        if metric == L2:
            r = float(raw[j])
            break
        up = down = np.float32(1) - raw[j]
        cands = [up]
        for _ in range(4):
            up, down = np.nextafter(up, np.float32(np.inf)), np.nextafter(down, np.float32(-np.inf))
            cands += [up, down]
        ok = [c for c in cands if np.float32(1) - c == raw[j]]
        if ok:
            r = float(ok[0])
            break
    assert r is not None, "no radius maps onto a row's raw value"
    D, I, C = s.ix.range_search(xq[:1], r, 256, nprobe=s.nlist)
    assert s.lids[j] not in I[0], "the row on the boundary must be excluded"
    check_range(s, xq[:1], r, 256)


@pytest.mark.parametrize("metric", [L2, IP])
@pytest.mark.parametrize("nbits,M", [(3, 20), (6, 16)])
def test_delete_compaction_upsert(oracle, metric, nbits, M):
    """Deleting more than half the rows compacts the lists (packed rows relocated by move_codes_kernel); an upsert over
    existing ids replaces their codes.  Each time the lists are exported again and compared with the oracle."""
    s = SynthN(oracle, metric, 12000, 80, 16, M, nbits, seed=51 + metric)
    s.export()
    rng = np.random.default_rng(52)
    xq = rng.standard_normal((6, 80)).astype(np.float32)
    dead = np.sort(rng.choice(np.arange(1, 12001), 7000, replace=False))
    assert s.delete(dead) == 7000
    assert s.ix.get_deleted_count() == 0, "the lists were not compacted"
    s.export()
    s.search(xq, 40, nprobe=16)
    s.search(xq, 40, nprobe=4)
    live = np.array(sorted(s.rows), np.int64)
    up = np.sort(rng.choice(live, 800, replace=False))
    s.add(rng.standard_normal((800, 80)).astype(np.float32), up, upsert=True)
    assert s.ix.get_count() == 5000
    s.export()
    s.search(xq, 40, nprobe=16)
    s.search(xq, 40, nprobe=4, sorted_ids=up)


def test_save_load_and_width_mismatch(oracle):
    s = SynthN(oracle, L2, 4000, 40, 8, 8, 5, seed=61)
    s.export()
    xq = np.random.default_rng(62).standard_normal((5, 40)).astype(np.float32)
    D, I = s.search(xq, 30, nprobe=8)
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "pq5.idx")
        s.ix.save(path)
        fresh = b200vs.Index(IVF_PQ, L2, 40, nlist=8, pq_m=8, pq_nbits=5)
        fresh.load(path)
        D2, I2 = fresh.search(xq, 30, nprobe=8)
        assert np.array_equal(I, I2) and np.array_equal(D.view(np.uint32), D2.view(np.uint32))
        off, _, packed, lids = fresh.export_lists(8, with_vectors=False, code_size=5)
        assert np.array_equal(off, s.off) and np.array_equal(lids, s.lids) and np.array_equal(packed, s.packed)
        other = b200vs.Index(IVF_PQ, L2, 40, nlist=8, pq_m=8, pq_nbits=4)
        with pytest.raises(b200vs.B200VSError) as e:
            other.load(path)
        assert e.value.code == b200vs.EINTERNAL
        eight = SynthN(oracle, L2, 500, 40, 8, 8, 8, seed=63)
        path8 = os.path.join(tmp, "pq8.idx")
        eight.ix.save(path8)
        with pytest.raises(b200vs.B200VSError) as e:
            b200vs.Index(IVF_PQ, L2, 40, nlist=8, pq_m=8, pq_nbits=5).load(path8)
        assert e.value.code == b200vs.EINTERNAL
    with pytest.raises(b200vs.B200VSError) as e:
        b200vs.Index(IVF_PQ, L2, 40, nlist=8, pq_m=8, pq_nbits=4).set_trained_state(s.ix.get_trained_state())
    assert e.value.code == b200vs.EILLEGAL_PARAMETERS


def test_create_refuses_9_to_16():
    for nbits in (9, 12, 16, 17):
        with pytest.raises(b200vs.B200VSError) as e:
            b200vs.Index(IVF_PQ, L2, 64, nlist=8, pq_m=8, pq_nbits=nbits)
        assert e.value.code == b200vs.EILLEGAL_PARAMETERS
    b200vs.Index(IVF_PQ, L2, 64, nlist=8, pq_m=8, pq_nbits=0)  # 0 -> the default 8


def test_memory_size_shrinks_with_nbits(oracle):
    xb = np.random.default_rng(71).standard_normal((4000, 64)).astype(np.float32)
    ids = np.arange(4000, dtype=np.int64)
    sizes = []
    for nbits in (8, 6, 4, 2, 1):
        s = SynthN(oracle, L2, 10, 64, 8, 32, nbits, seed=72)
        s.ix.add(xb, ids + 100)
        sizes.append(s.ix.get_memory_size())
    assert all(a > b for a, b in zip(sizes, sizes[1:])), sizes


def test_training_threshold_at_4_bits(oracle):
    """Fewer than max(256 * nlist, 256 * 2^nbits) training vectors -> inner Flat index; with nlist = 8 the 2^nbits term
    (4096 at 4 bits) decides."""
    rng = np.random.default_rng(81)
    xb = rng.standard_normal((4096, 32)).astype(np.float32)
    ids = np.arange(1, 4097, dtype=np.int64)
    xq = rng.standard_normal((5, 32)).astype(np.float32)
    small = b200vs.Index(IVF_PQ, L2, 32, nlist=8, pq_m=8, pq_nbits=4)
    small.train(xb[:4095])
    assert small.sub_type() == FLAT
    small.add(xb, ids)
    D, I = small.search(xq, 10)
    Do, Io = oracle.flat_search(L2, xb, ids, xq, 10)
    assert_same_results(D, I, Do, Io)
    full = b200vs.Index(IVF_PQ, L2, 32, nlist=8, pq_m=8, pq_nbits=4)
    full.train(xb)
    assert full.sub_type() == IVF_PQ


@pytest.mark.parametrize("metric", [L2, IP])
@pytest.mark.parametrize("M", [16, 8])
def test_gpu_training_small_dsub(oracle, metric, M):
    """dsub = 1 and 2 at 4 bits: 16 codewords per sub-space trained on the GPU; the trained state, read back, drives the
    oracle to the engine's results."""
    rng = np.random.default_rng(91 + M)
    d, nlist = 16, 4
    xb = rng.standard_normal((5000, d)).astype(np.float32)
    ix = b200vs.Index(IVF_PQ, metric, d, nlist=nlist, pq_m=M, pq_nbits=4)
    ix.train(xb)
    assert ix.sub_type() == IVF_PQ
    ix.add(xb, np.arange(1, 5001, dtype=np.int64))
    blob = ix.get_trained_state()
    hdr = blob[:48].view(np.int64)
    assert hdr[5] == 4 and hdr[4] == M
    cent = blob[48:48 + nlist * d * 4].view(np.float32).reshape(nlist, d)
    cb = blob[48 + nlist * d * 4:].view(np.float32).reshape(M, 16, d // M)
    off, _, packed, lids = ix.export_lists(nlist, with_vectors=False, code_size=pq_codes.code_size(M, 4))
    xq = rng.standard_normal((6, d)).astype(np.float32)
    D, I = ix.search(xq, 20, nprobe=nlist)
    Do, Io = pq_codes.ivfpq_search(oracle, metric, cent, cb, off, packed, lids, xq, 20, nlist, nthreads=8)
    assert_same_results(D, I, Do, Io)


def test_gpu_trained_recall_at_4_bits(oracle):
    """Full GPU training at 4 bits (M = 16: the bytes of 8-bit M = 8); a sanity floor, not a quality claim."""
    rng = np.random.default_rng(3)
    n, d, nlist, M = 70000, 32, 64, 16
    centers = rng.standard_normal((500, d)).astype(np.float32)
    xb = (centers[rng.integers(0, 500, n)] + 0.3 * rng.standard_normal((n, d))).astype(np.float32)
    ids = np.arange(n, dtype=np.int64)
    ix = b200vs.Index(IVF_PQ, L2, d, nlist=nlist, pq_m=M, pq_nbits=4)
    ix.train(xb)
    assert ix.sub_type() == IVF_PQ
    ix.add(xb, ids)
    xq = xb[:100] + 0.01 * rng.standard_normal((100, d)).astype(np.float32)
    D, I = ix.search(xq, 10, nprobe=16)
    Df, If = oracle.flat_search(L2, xb, ids, xq, 10, nthreads=8)
    assert recall(I, If) > 0.2
    assert (I[:, 0] == ids[:100]).mean() > 0.7
