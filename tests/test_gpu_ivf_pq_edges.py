"""IVF-PQ at the edges of pq_scan_select_kernel and pq_encode_kernel, on synthetic trained states (random centroids and
codebooks: training is not under test here).  Every case checks three things:
  * the GPU codes equal oracle.ivfpq_encode row for row, and the list assignment equals oracle.assign;
  * the search equals oracle.ivfpq_search bit for bit;
  * independently of the oracle, every returned distance is the float64 distance to the decoded row c[list] + concat_m
    cw[m][code_m] within gamma * S (S = summed magnitudes of the terms the kernel adds, gamma = (M + d + 2) 2^-24),
    results are sorted, and no row left out is closer than the k-th by more than that bound.
Code-read branches: M % 16 != 0 reads code bytes one by one; M % 16 == 0 && M <= 128 loads all code words of a row up
front; M % 16 == 0 && M > 128 loads 16 codes at a time in a loop."""
import numpy as np
import pytest

import b200vs
from b200vs import COSINE, IP, IVF_PQ, L2
from gpu_util import assert_same_results, require_gpu

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _gpu():
    require_gpu()


class Synth:
    """An IVF-PQ index on a random trained state, plus what the checks need: stored rows by id, the exported lists."""

    def __init__(self, oracle, metric, n, d, nlist, M, seed=0, far_lists=0):
        rng = np.random.default_rng(seed)
        self.o, self.metric, self.d, self.nlist, self.M = oracle, metric, d, nlist, M
        xb = rng.standard_normal((n, d)).astype(np.float32)
        stored = oracle.normalize_faiss(xb) if metric == COSINE else xb
        cent = stored[rng.choice(n, nlist, replace=False)] + 0.1 * rng.standard_normal((nlist, d)).astype(np.float32)
        if far_lists:  # centroids no row is closest to: empty lists (L2)
            cent[nlist - far_lists:] += 50.0
        self.cent = cent.astype(np.float32)
        self.cb = (0.5 * rng.standard_normal((M, 256, d // M))).astype(np.float32)
        self.ix = b200vs.Index(IVF_PQ, metric, d, nlist=nlist, pq_m=M, pq_nbits=8)
        self.ix.set_trained_state(b200vs.ivfpq_state_blob(self.cent, self.cb, metric))
        self.rows = {}
        self.add(xb, np.arange(1, n + 1, dtype=np.int64))

    def add(self, x, ids, upsert=False):
        self.ix.add(x, ids, upsert=upsert)
        stored = self.o.normalize_faiss(x) if self.metric == COSINE else x
        self.rows.update(zip(ids.tolist(), stored))

    def delete(self, ids):
        n = self.ix.delete(ids)
        for i in ids.tolist():
            self.rows.pop(i, None)
        return n

    def export(self):
        """Exported lists; asserts the codes and the list assignment equal the oracle's."""
        off, _, codes, lids = self.ix.export_lists(self.nlist, with_vectors=False, code_size=self.M)
        assert off[-1] == len(self.rows) == self.ix.get_count()
        lst = np.repeat(np.arange(self.nlist), np.diff(off)).astype(np.int32)
        X = np.stack([self.rows[i] for i in lids.tolist()]) if len(lids) else np.zeros((0, self.d), np.float32)
        if len(lids):
            assert np.array_equal(self.o.assign(self.metric, X, self.cent), lst), "list assignment differs from the oracle"
            assert np.array_equal(codes, self.o.ivfpq_encode(self.cb, self.cent, X, lst)), "codes differ from the oracle encoder"
        self.off, self.codes, self.lids, self.lst = off, codes, lids, lst
        return off, codes, lids

    def queries(self, xq):
        return self.o.normalize_faiss(xq) if self.metric == COSINE else xq

    def f64(self, q):
        """(true distance, S) of every exported row to one query, in float64, in API units."""
        cb = self.cb.astype(np.float64)
        R = cb[np.arange(self.M)[None, :], self.codes.astype(np.int64)].reshape(len(self.lids), self.d)
        C = self.cent.astype(np.float64)[self.lst]
        Q = self.queries(q[None, :]).astype(np.float64)[0]
        if self.metric == L2:
            qc = Q - C
            return ((qc - R) ** 2).sum(1), (qc ** 2).sum(1) + (R ** 2).sum(1) + 2 * np.abs(C * R).sum(1) + 2 * np.abs(Q * R).sum(1)
        return 1.0 - (C @ Q + R @ Q), np.abs(C * Q).sum(1) + np.abs(R * Q).sum(1) + 1.0

    def search(self, xq, k, nprobe, **filt):
        """Engine search == oracle search (bit for bit), then the float64 checks."""
        Dg, Ig = self.ix.search(xq, k, nprobe=nprobe, **filt)
        Do, Io = self.o.ivfpq_search(self.metric, self.cent, self.cb, self.off, self.codes, self.lids, xq, k, nprobe, nthreads=8, **filt)
        assert_same_results(Dg, Ig, Do, Io)
        self.check_f64(xq, Dg, Ig, every_row=min(nprobe, self.nlist) == self.nlist, **filt)
        return Dg, Ig

    def check_f64(self, xq, D, I, every_row, id_range=None, sorted_ids=None, negate=False):
        gamma = (self.M + self.d + 2) * 2.0 ** -24
        pos = {int(i): r for r, i in enumerate(self.lids.tolist())}
        cand = np.ones(len(self.lids), bool)
        if id_range is not None:
            cand &= (self.lids >= id_range[0]) & (self.lids < id_range[1])
        if sorted_ids is not None:
            cand &= np.isin(self.lids, sorted_ids) != negate
        k = I.shape[1]
        for qi in range(len(xq)):
            valid = I[qi] >= 0
            c = int(valid.sum())
            assert valid[:c].all() and not valid[c:].any(), "-1 padding must come last"
            assert (np.diff(D[qi][:c]) >= 0).all(), "distances not ascending"
            true, S = self.f64(xq[qi])
            r = np.array([pos[int(i)] for i in I[qi][:c]], np.int64)
            err = np.abs(D[qi][:c].astype(np.float64) - true[r])
            assert (err <= gamma * S[r]).all(), f"query {qi}: |gpu - f64| / bound = {(err / (gamma * S[r])).max():.3f}"
            if not every_row:
                continue
            left = cand.copy()
            left[r] = False
            if c < k:  # fewer hits than k: every candidate row came back
                assert not left.any(), f"query {qi}: {left.sum()} rows missing"
            else:  # gpu(left) >= gpu(k-th) and |gpu - f64| <= gamma S
                assert (true[left] >= float(D[qi][k - 1]) - gamma * S[left]).all(), f"query {qi}: an omitted row is closer"

    def raw_fp32(self, q):
        """The kernel's raw FP32 value of every exported row (L2: squared distance, IP: inner product), restated in numpy
        in the kernel's order: coarse value, then the LUT entries added sequentially over m."""
        o, M, dsub = self.o, self.M, self.d // self.M
        Q = self.queries(q[None, :])[0]
        dis0 = np.array([o.l2sqr(Q, c) if self.metric == L2 else o.ip(Q, c) for c in self.cent], np.float32)

        def seq_ip(a, b):  # a [..., dsub] * b [..., dsub], summed left to right in FP32
            acc = np.zeros(np.broadcast(a[..., 0], b[..., 0]).shape, np.float32)
            for i in range(dsub):
                acc = (acc + (a[..., i] * b[..., i]).astype(np.float32)).astype(np.float32)
            return acc

        sim = seq_ip(Q.reshape(M, 1, dsub), self.cb)  # [M, 256]
        vals = dis0[self.lst]
        for m in range(M):
            tab = sim[m][None, :]  # [1 or nlist, 256]
            if self.metric == L2:  # T = ||cw||^2 + 2 <c_m, cw>, then T - 2 sim
                cw = self.cb[m]
                pre = (seq_ip(cw, cw)[None, :] + np.float32(2) * seq_ip(self.cent[:, None, m * dsub:(m + 1) * dsub], cw[None])).astype(np.float32)
                tab = (pre + np.float32(-2) * sim[m][None, :]).astype(np.float32)
            vals = (vals + tab[self.lst if self.metric == L2 else 0, self.codes[:, m].astype(np.int64)]).astype(np.float32)
        return vals


BRANCH_CASES = [  # (M, d): the code-read branch each one reaches
    (1, 16), (2, 32), (8, 64), (12, 48),            # M % 16 != 0: byte loop
    (16, 16), (48, 96), (64, 128), (128, 128),      # M % 16 == 0, M <= 128: all code words up front (16 and 128: dsub = 1)
    (144, 144), (192, 384),                         # M % 16 == 0, M > 128: 16 codes per step (144: dsub = 1)
]


@pytest.mark.parametrize("metric", [L2, IP, COSINE])
@pytest.mark.parametrize("M,d", BRANCH_CASES)
def test_code_read_branches(oracle, metric, M, d):
    s = Synth(oracle, metric, 3000, d, 8, M, seed=M * 7 + d)
    s.export()
    xq = np.random.default_rng(M).standard_normal((6, d)).astype(np.float32)
    s.search(xq, 50, nprobe=8)
    s.search(xq, 20, nprobe=3)
    s.search(xq, 10, nprobe=8, id_range=(500, 2500))


@pytest.mark.parametrize("metric", [L2, IP])
@pytest.mark.parametrize("M", [64, 128])
def test_large_k(oracle, metric, M):
    """k up to 4096; at M = 128 the LUT plus the 4096-entry select pool come within 3 KB of the 227 KB shared-memory cap."""
    s = Synth(oracle, metric, 6000, 128, 4, M, seed=M + metric)
    s.export()
    xq = np.random.default_rng(3).standard_normal((3, 128)).astype(np.float32)
    for k in (1, 129, 1024, 4096):
        s.search(xq, k, nprobe=4)


def test_limits_are_refused_on_the_host(oracle):
    """Shapes whose LUT + select pool exceed shared memory fail with EILLEGAL_PARAMETERS before anything is launched, and
    the index keeps working."""
    s = Synth(oracle, L2, 2000, 384, 4, 192, seed=1)
    s.export()
    xq = np.random.default_rng(2).standard_normal((2, 384)).astype(np.float32)
    for call in (lambda: s.ix.search(xq, 4096, nprobe=4), lambda: s.ix.range_search(xq, 1e9, 4096, nprobe=4)):
        with pytest.raises(b200vs.B200VSError) as e:
            call()
        assert e.value.code == b200vs.EILLEGAL_PARAMETERS
    s.search(xq, 1024, nprobe=4)  # 192 x 1 KB LUT + a 2048-entry pool still fit
    big = Synth(oracle, IP, 1000, 256, 2, 256, seed=2)  # 256 KB of LUT alone
    big.export()
    with pytest.raises(b200vs.B200VSError) as e:
        big.ix.search(np.ones((1, 256), np.float32), 1, nprobe=2)
    assert e.value.code == b200vs.EILLEGAL_PARAMETERS


@pytest.mark.parametrize("metric", [L2, IP])
def test_probing(oracle, metric):
    """nq = 1 with 512 probed lists (the scan splits each query over min(nprobe, 2 x SMs) CTAs, the merge sees nsplit x k
    entries); nprobe > nlist is clamped; nlist = 1."""
    s = Synth(oracle, metric, 20000, 32, 512, 8, seed=5)
    s.export()
    rng = np.random.default_rng(6)
    xq = rng.standard_normal((1, 32)).astype(np.float32)
    s.search(xq, 100, nprobe=512)
    s.search(xq, 1, nprobe=512)
    t = Synth(oracle, metric, 4000, 32, 16, 8, seed=7)
    t.export()
    xq = rng.standard_normal((5, 32)).astype(np.float32)
    D1, I1 = t.search(xq, 30, nprobe=1000)
    D2, I2 = t.search(xq, 30, nprobe=16)
    assert_same_results(D1, I1, D2, I2)
    u = Synth(oracle, metric, 3000, 32, 1, 8, seed=8)
    u.export()
    u.search(xq, 40, nprobe=1)
    u.search(xq, 40, nprobe=5)


def test_empty_and_dead_lists(oracle):
    """Probed lists with no rows, and a probed list whose rows are all deleted: results padded with -1, count below k."""
    s = Synth(oracle, L2, 300, 32, 16, 8, seed=9, far_lists=6)
    off, codes, lids = s.export()
    assert (np.diff(off)[10:] == 0).all()
    xq = np.concatenate([s.cent[:2], np.random.default_rng(10).standard_normal((3, 32)).astype(np.float32)])
    D, I = s.search(xq, 512, nprobe=16)
    assert ((I >= 0).sum(1) == 300).all()
    s.search(xq, 64, nprobe=12)
    dead = lids[off[0]:off[1]]  # all of list 0
    assert len(dead) > 0 and s.delete(dead) == len(dead)
    s.export()
    D, I = s.search(s.cent[:1], 16, nprobe=1)  # probes list 0 only
    assert (I == -1).all()
    D, I = s.search(xq, 512, nprobe=3)
    assert ((I >= 0).sum(1) < 512).all()


@pytest.mark.parametrize("metric", [L2, IP])
def test_compaction_and_upsert(oracle, metric):
    """Deleting more than half of the rows compacts the lists (move_codes_kernel relocates the survivors); an upsert over
    existing ids replaces their codes.  Each time the lists are exported again and compared with the oracle."""
    s = Synth(oracle, metric, 12000, 64, 16, 16, seed=11)
    s.export()
    rng = np.random.default_rng(12)
    xq = rng.standard_normal((6, 64)).astype(np.float32)
    dead = np.sort(rng.choice(np.arange(1, 12001), 7000, replace=False))
    assert s.delete(dead) == 7000
    assert s.ix.get_deleted_count() == 0, "the lists were not compacted"
    s.export()
    s.search(xq, 40, nprobe=16)
    s.search(xq, 40, nprobe=4)
    live = np.array(sorted(s.rows), np.int64)
    up = np.sort(rng.choice(live, 800, replace=False))
    s.add(rng.standard_normal((800, 64)).astype(np.float32), up, upsert=True)
    assert s.ix.get_count() == 5000
    s.export()
    s.search(xq, 40, nprobe=16)
    s.search(xq, 40, nprobe=4, sorted_ids=up)


def range_expect(s, q, radius, max_results):
    """(ids, API distances, hit count) the range search must return for one query: every row strictly inside the raw
    threshold (L2: dis < radius; IP: ip > 1 - radius in FP32), closest first, at most max_results."""
    raw = s.raw_fp32(q)
    if s.metric == L2:
        keep, order_key, api = raw < np.float32(radius), raw, raw
    else:
        keep = raw > np.float32(1) - np.float32(radius)
        order_key, api = -raw, (np.float32(1) - raw).astype(np.float32)
    idx = np.nonzero(keep)[0]
    idx = idx[np.lexsort((s.lids[idx], order_key[idx]))]
    c = min(len(idx), max_results)
    return s.lids[idx[:c]], api[idx[:c]], len(idx)


def check_range(s, xq, radius, max_results):
    D, I, C = s.ix.range_search(xq, radius, max_results, nprobe=s.nlist)
    total = []
    for qi in range(len(xq)):
        want_i, want_d, hits = range_expect(s, xq[qi], radius, max_results)
        assert C[qi] == len(want_i)
        assert np.array_equal(I[qi, :C[qi]], want_i) and (I[qi, C[qi]:] == -1).all()
        assert np.array_equal(D[qi, :C[qi]].view(np.uint32), want_d.view(np.uint32))
        total.append(hits)
    s.check_f64(xq, D, I, every_row=False)
    return total


@pytest.mark.parametrize("metric", [L2, IP, COSINE])
def test_range_search_limits(oracle, metric):
    """More hits than max_results keeps exactly the max_results closest; a radius equal to an existing distance excludes
    that row (strict); nq = 1.  The expected hits come from a numpy restatement of the kernel's FP32 sums over every row
    (all lists probed), itself checked against the oracle's top-k distances."""
    s = Synth(oracle, metric, 5000, 64, 8, 16, seed=13 + metric)
    s.export()
    xq = np.random.default_rng(14).standard_normal((4, 64)).astype(np.float32)
    Do, Io = oracle.ivfpq_search(metric, s.cent, s.cb, s.off, s.codes, s.lids, xq, 5000, 8, nthreads=8)
    pos = {int(i): r for r, i in enumerate(s.lids.tolist())}
    for qi in range(len(xq)):  # the restatement is bit-exact
        raw = s.raw_fp32(xq[qi])[[pos[int(i)] for i in Io[qi]]]
        api = raw if metric == L2 else (np.float32(1) - raw).astype(np.float32)
        assert np.array_equal(api.view(np.uint32), Do[qi].view(np.uint32))
    radius = float(np.median(Do[:, 600]))  # ~600 hits per query
    hits = check_range(s, xq, radius, 64)
    assert min(hits) > 64
    check_range(s, xq[:1], radius, 64)   # nq = 1
    check_range(s, xq[:1], radius, 1024)
    if metric == COSINE:
        return
    # strict boundary: the radius (L2) / the FP32 threshold 1 - radius (IP) equals one row's raw value exactly
    raw = s.raw_fp32(xq[0])
    order = np.argsort(raw) if metric == L2 else np.argsort(-raw)
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
    else:
        pytest.fail("no radius maps onto a row's raw value")
    D, I, C = s.ix.range_search(xq[:1], r, 256, nprobe=s.nlist)
    assert s.lids[j] not in I[0], "the row on the boundary must be excluded"
    check_range(s, xq[:1], r, 256)


@pytest.mark.parametrize("metric", [L2, IP])
def test_large_dimension(oracle, metric):
    """d = 4096 with M = 64: the encoder keeps one residual row per warp in shared memory (64 KB for 4 warps), past the 48 KB
    a launch gets without opting in."""
    s = Synth(oracle, metric, 1500, 4096, 4, 64, seed=15)
    s.export()
    xq = np.random.default_rng(16).standard_normal((3, 4096)).astype(np.float32)
    s.search(xq, 20, nprobe=4)
    s.search(xq, 100, nprobe=2)
