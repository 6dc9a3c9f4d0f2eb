"""The exact FP32 path at its edges: flat_small_kernel (Flat, nq < 16), scan_select_kernel + merge_select_kernel with
BlockSelect (k > 128, exact_only, IVF batches below 16 queries), and Flat / IVF-Flat range search (the same scan with a
fixed threshold).  Every search case checks three things:
  * bit parity with oracle.flat_search / oracle.ivfflat_search: ids and distance bits, -1 / 0 padding included;
  * independently of the oracle, in float64 from the rows the index stores (FP32-normalised rows and queries for cosine):
    every returned distance is within gamma * S of the true one (S = sum of the term magnitudes), results ascend with the
    -1 padding last, and, when every row is a candidate, no omitted row is closer than the k-th by more than the bound;
  * the route: ix.stats()[0] counts the launches of the last search (reset by the host search path): 1 = flat_small_kernel,
    2 = scan + merge, >= 5 = tensor-core path; cosine adds one for the query normaliser.

gamma: quad_distance keeps 16 lane partials; lane j adds the terms j, j + 16, ... one after the other (ceil(d / 16) adds),
then the lanes are folded 16 -> 8 -> 4 with the 8-, 4- and 1..3-wide tails added in between (at most 5 more adds on any
term's path) and 4 -> 1 by two more adds.  A term itself is rounded once (IP: x * q) or twice ((x - q), then its square),
so every term goes through at most m = ceil(d / 16) + 10 roundings, and |fp32 - exact| <= gamma_m * sum|terms| with
gamma_m = m u / (1 - m u), u = 2^-24.  The API value 1 - ip of IP / cosine rounds once more (m + 1, S + 1).  At d = 128
gamma is ~1.1e-6 relative, three orders below the neighbour gaps of the data here."""
import numpy as np
import pytest

import b200vs
from b200vs import COSINE, FLAT, IP, IVF_FLAT, L2
from gpu_util import assert_same_results, require_gpu

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
FS_PAIRS, FS_CT = 3072, 128   # csrc/flat_small.cu
SCAN_THREADS = 256            # csrc/scan_kernels.cuh
MAX_SMEM = 227 * 1024         # csrc/kernels.cu kMaxDynSmem
MAX_NQ = 65535                # grid.y of scan_select_kernel


@pytest.fixture(autouse=True)
def _gpu():
    require_gpu()


@pytest.fixture(scope="module")
def sms():
    require_gpu()
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


# ---- the launchers' formulas, restated to derive shapes ----

def next_pow2(v):
    p = 1
    while p < v:
        p <<= 1
    return p


def pool_cap(k):
    """select_pool_cap(k, SCAN_THREADS) (csrc/select.cuh)."""
    c = next_pow2(k + SCAN_THREADS)
    if c < 2 * k:
        c = next_pow2(2 * k)
    return max(c, 512)


def pad16(b):
    return (b + 15) // 16 * 16


def scan_smem(d, nseg, k):
    return pad16(4 * d) + pad16(4 * (nseg + 1)) + pool_cap(k) * 12 + 32


def scan_nsplit(nq, cand, sms):
    """run_scan_impl: clamp(ceil(4 SMs / nq), 1, min(128, cand / 512))."""
    nsplit = max(1, -(-4 * sms // nq))
    return max(1, min(nsplit, min(max(1, int(cand / 512.0)), 128)))


def fs_eligible(nq, n, d, k, sms):
    """flat_small_eligible (csrc/flat_small.cu)."""
    if nq < 1 or nq >= 16 or n < 4096 or 2 * k > FS_CT or d > 2048:
        return False
    if nq > 4 and n * d * 4 > 40e6:
        return False
    nslices = min(2 * sms, FS_PAIRS // max(1, k))
    return -(-n // nslices) <= FS_PAIRS


def fs_slice_rows(n, k, sms):
    nslices = min(min(2 * sms, FS_PAIRS // max(1, k)), max(1, n // 64))
    return -(-n // nslices)


# ---- float64 and FP32 restatements ----

def prep(o, metric, xq):
    xq = np.ascontiguousarray(xq, np.float32)
    return o.normalize_faiss(xq) if metric == COSINE else xq


def cand_mask(ids, id_range=None, sorted_ids=None, negate=False):
    m = np.ones(len(ids), bool)
    if id_range is not None:
        m &= (ids >= id_range[0]) & (ids < id_range[1])
    if sorted_ids is not None:
        m &= np.isin(ids, sorted_ids) != negate
    return m


def f64_true(X, q, metric):
    """(true API distance, S) of every row in float64."""
    X64, q64 = X.astype(np.float64), q.astype(np.float64)
    if metric == L2:
        t = ((X64 - q64) ** 2).sum(1)
        return t, t
    return 1.0 - X64 @ q64, np.abs(X64 * q64).sum(1) + 1.0


def gamma(d, metric):
    m = -(-d // 16) + 10 + (0 if metric == L2 else 1)
    return m * U / (1 - m * U)


def check_f64(X, ids, Q, metric, D, I, every_row, cand=None, queries=None):
    """The float64 checks of the module docstring; Q holds the prepared (normalised for cosine) queries."""
    g = gamma(X.shape[1], metric)
    pos = {int(i): r for r, i in enumerate(ids.tolist())}
    cand = np.ones(len(ids), bool) if cand is None else cand
    k = I.shape[1]
    for qi in (range(len(Q)) if queries is None else queries):
        valid = I[qi] >= 0
        c = int(valid.sum())
        assert valid[:c].all() and not valid[c:].any(), "-1 padding must come last"
        assert (D[qi][c:] == 0).all(), "padding distances must be 0"
        assert (np.diff(D[qi][:c]) >= 0).all(), "distances not ascending"
        true, S = f64_true(X, Q[qi], metric)
        r = np.array([pos[int(i)] for i in I[qi][:c]], np.int64)
        assert cand[r].all(), f"query {qi}: a row outside the candidates came back"
        err = np.abs(D[qi][:c].astype(np.float64) - true[r])
        assert (err <= g * S[r]).all(), f"query {qi}: |gpu - f64| / bound = {(err / (g * S[r])).max():.3f}"
        if not every_row:
            continue
        left = cand.copy()
        left[r] = False
        if c < k:
            assert not left.any(), f"query {qi}: {left.sum()} candidate rows missing"
        elif left.any():
            assert (true[left] >= float(D[qi][k - 1]) - g * S[left]).all(), f"query {qi}: an omitted row is closer"


def raw_fp32(X, q, metric):
    """The kernel's raw FP32 value (L2: squared distance, IP: inner product) of every row to q, restated in numpy in
    quad_distance's order: 16 lane partials, fold 16 -> 8, 8-wide tail, fold 8 -> 4, 4-wide tail, masked 1..3 tail,
    (m0 + m1) + (m2 + m3)."""
    n, d = X.shape
    T = (X - q) * (X - q) if metric == L2 else X * q
    T = T.astype(np.float32)
    nfull = d // 16
    acc = np.zeros((n, 16), np.float32)
    for c in range(nfull):
        acc = acc + T[:, 16 * c:16 * c + 16]
    m1 = acc[:, 8:16] + acc[:, 0:8]
    base, rem = 16 * nfull, d - 16 * nfull
    if rem >= 8:
        m1 = m1 + T[:, base:base + 8]
        base, rem = base + 8, rem - 8
    m2 = m1[:, 4:8] + m1[:, 0:4]
    if rem >= 4:
        m2 = m2 + T[:, base:base + 4]
        base, rem = base + 4, rem - 4
    if rem > 0:
        tail = np.zeros((n, 4), np.float32)
        tail[:, :rem] = T[:, base:base + rem]
        m2 = m2 + tail
    return ((m2[:, 0] + m2[:, 1]) + (m2[:, 2] + m2[:, 3])).astype(np.float32)


def api_of(raw, metric):
    return raw if metric == L2 else (np.float32(1) - raw).astype(np.float32)


class FlatCase:
    """A Flat index plus what the checks need: the stored rows and ids as exported (re-read after deletes)."""

    def __init__(self, o, metric, xb, ids):
        self.o, self.metric, self.d = o, metric, xb.shape[1]
        self.ix = b200vs.Index(FLAT, metric, self.d)
        for a in range(0, len(ids), 32768):
            self.ix.add(xb[a:a + 32768], ids[a:a + 32768])
        self.ix.coalescing(0)
        self.refresh()

    def refresh(self):
        _, self.X, _, self.ids = self.ix.export_lists(1)

    def delete(self, ids):
        n = self.ix.delete(ids)
        self.refresh()
        return n

    def rows_total(self):
        return self.ix.get_count() + self.ix.get_deleted_count()

    def search(self, xq, k, route=None, f64_queries=None, **kw):
        D, I = self.ix.search(xq, k, **kw)
        launches = self.ix.stats()[0]
        filt = {a: kw[a] for a in ("id_range", "sorted_ids", "negate") if a in kw}
        Do, Io = self.o.flat_search(self.metric, self.X, self.ids, xq, k, nthreads=8, **filt)
        assert_same_results(D, I, Do, Io)
        if route is not None:
            base = 1 if self.metric == COSINE else 0
            if route == "small":
                assert launches == base + 1, f"expected flat_small_kernel, {launches} launches"
            elif route == "scan":
                assert launches == base + 2, f"expected scan + merge, {launches} launches"
            else:
                assert launches >= base + 5, f"expected the tensor-core path, {launches} launches"
        check_f64(self.X, self.ids, prep(self.o, self.metric, xq), self.metric, D, I, every_row=True,
                  cand=cand_mask(self.ids, **filt), queries=f64_queries)
        return D, I


def rows(rng, n, d):
    return rng.standard_normal((n, d)).astype(np.float32)


# =====================================================================================================================
# A. flat_small_kernel
# =====================================================================================================================

# (name, n, d, k, nq): one case on each side of every condition of flat_small_eligible; n may depend on the SM count
ELIGIBILITY = [
    ("n4095", lambda s: 4095, 32, 10, 1),
    ("n4096", lambda s: 4096, 32, 10, 1),
    ("k64", lambda s: 8192, 32, 64, 2),
    ("k65", lambda s: 8192, 32, 65, 2),
    ("d1592", lambda s: 4096, 1592, 10, 2),
    ("d1593", lambda s: 4096, 1593, 10, 2),
    ("d2048", lambda s: 4096, 2048, 10, 2),
    ("d2049", lambda s: 4096, 2049, 10, 2),
    ("40MB-nq4", lambda s: 100_000, 100, 10, 4),
    ("40MB-nq5", lambda s: 100_000, 100, 10, 5),
    ("40MBplus1row-nq4", lambda s: 100_001, 100, 10, 4),
    ("40MBplus1row-nq5", lambda s: 100_001, 100, 10, 5),
    ("slices-fit", lambda s: min(2 * s, FS_PAIRS // 64) * FS_PAIRS, 16, 64, 1),
    ("slices-fit-plus1", lambda s: min(2 * s, FS_PAIRS // 64) * FS_PAIRS + 1, 16, 64, 1),
    ("nq15", lambda s: 4096, 32, 10, 15),
    ("nq16", lambda s: 4096, 32, 10, 16),
]


@pytest.mark.parametrize("metric", [L2, IP])
@pytest.mark.parametrize("name,nf,d,k,nq", ELIGIBILITY, ids=[c[0] for c in ELIGIBILITY])
def test_flat_small_eligibility(oracle, sms, metric, name, nf, d, k, nq):
    """Each side of each condition of flat_small_eligible takes the route the code gives it and answers exactly.  The
    d = 1593 and 2048 cases need the launcher to opt the kernel in past 48 KB of shared memory."""
    n = nf(sms)
    small = fs_eligible(nq, n, d, k, sms)
    tc = not small and nq >= 16 and d % 4 == 0 and d >= 32 and k <= 128
    expect = {"n4095": False, "k65": False, "d2049": False, "40MBplus1row-nq5": False, "slices-fit-plus1": False, "nq16": False}
    assert small == expect.get(name, True), "premise: the shape is not on the intended side of the condition"
    rng = np.random.default_rng(n + d + k)
    c = FlatCase(oracle, metric, rows(rng, n, d), rng.permutation(np.arange(1, n + 1, dtype=np.int64)))
    xq = rows(rng, nq, d)
    c.search(xq, k, route="small" if small else ("tc" if tc else "scan"), f64_queries=range(min(nq, 5)))


@pytest.mark.parametrize("metric", [L2, IP, COSINE])
def test_flat_small_slices_filters_and_tombstones(oracle, sms, metric):
    """Slices with <= 128 live pairs (rank-all) and with more (radix select + rank sort); filters that reject whole slices
    (ids follow the row order, so an id range is a row range), every filter form and their combinations, fewer passing rows
    than k, and tombstoned slices."""
    rng = np.random.default_rng(7 + metric)
    n, d = 4096, 32
    assert fs_slice_rows(n, 10, sms) <= FS_CT, "premise: slices of at most 128 rows"
    few = FlatCase(oracle, metric, rows(rng, n, d), np.arange(1, n + 1, dtype=np.int64))
    few.search(rows(rng, 3, d), 10, route="small")
    n = 60000
    assert fs_slice_rows(n, 10, sms) > FS_CT and fs_slice_rows(n, 64, sms) > FS_CT, "premise: slices of more than 128 rows"
    c = FlatCase(oracle, metric, rows(rng, n, d), np.arange(1, n + 1, dtype=np.int64))
    xq = rows(rng, 3, d)
    sub = np.sort(rng.choice(np.arange(1, n + 1), 500, replace=False))
    for k in (10, 64):
        c.search(xq, k, route="small")
        c.search(xq, k, route="small", id_range=(20000, 40000))
        c.search(xq, k, route="small", sorted_ids=sub)
        c.search(xq, k, route="small", sorted_ids=sub, negate=True)
        c.search(xq, k, route="small", id_range=(10000, 50000), sorted_ids=sub)
        c.search(xq, k, route="small", id_range=(10000, 50000), sorted_ids=sub, negate=True)
    D, I = c.search(xq, 64, route="small", sorted_ids=sub[:20])  # 20 rows pass: padding
    assert ((I >= 0).sum(1) == 20).all()
    D, I = c.search(xq, 64, route="small", id_range=(59990, 70000))
    assert ((I >= 0).sum(1) == 11).all()
    assert c.delete(np.arange(1, 25001, dtype=np.int64)) == 25000  # the first ~40% of the slices hold no live row
    assert c.rows_total() == n, "premise: tombstones, no compaction"
    c.search(xq, 10, route="small")
    c.search(xq, 64, route="small", id_range=(1, 30000))


@pytest.mark.parametrize("id_base", ["small", "2^62", "2^63-2"])
def test_flat_small_mass_ties(oracle, sms, id_base):
    """More than 128 rows of one slice tied at the k-th key (the slice's mass-tie path) and more than 128 tied pairs in the
    merge, at k = 64, with a few strictly closer rows scattered in; ids near 2^62 and up to 2^63 - 2 (warp_min_ll)."""
    n, d, k = 100_000, 64, 64
    assert fs_eligible(1, n, d, k, sms) and fs_slice_rows(n, k, sms) > FS_CT, "premise: flat_small with slices > 128 rows"
    rng = np.random.default_rng(11)
    base = rng.random((4, d)).astype(np.float32)
    xb = np.repeat(base, n // 4, axis=0)
    q = base[0] + np.float32(0.001)
    close = rng.choice(n, 10, replace=False)
    xb[close] = q + (0.0001 * rng.standard_normal((10, d))).astype(np.float32)  # 10 rows strictly below the tied key
    perm = rng.permutation(n).astype(np.int64)
    ids = {"small": perm + 1, "2^62": perm + (1 << 62), "2^63-2": (2 ** 63 - 2) - perm}[id_base]
    c = FlatCase(oracle, L2, xb, ids)
    xq = np.stack([q, base[2] + np.float32(0.001), base[3] - np.float32(0.002)])
    D, I = c.search(xq, k, route="small")
    assert (D[0, 10:] == D[0, k - 1]).all() and (D[0, :10] < D[0, k - 1]).all(), "premise: 10 rows below the tied k-th key"
    c.search(xq, k, route="small", sorted_ids=np.sort(ids[:n // 2]))
    c.search(xq[:2], 1, route="small")


@pytest.mark.parametrize("metric", [L2, IP])
@pytest.mark.parametrize("n,d", [(4096, 1), (5000, 3), (4096, 2047)])
def test_flat_small_unaligned_dimensions(oracle, metric, n, d):
    """d % 4 != 0: scalar loads (d = 1: nearly every row ties with many others)."""
    rng = np.random.default_rng(d)
    c = FlatCase(oracle, metric, rows(rng, n, d), rng.permutation(np.arange(1, n + 1, dtype=np.int64)))
    xq = rows(rng, 3, d)
    c.search(xq, 10, route="small")
    c.search(xq, 64, route="small")


# =====================================================================================================================
# B. scan_select_kernel + merge_select_kernel
# =====================================================================================================================

@pytest.mark.parametrize("metric", [L2, IP])
def test_exact_scan_prunes_at_large_k(oracle, sms, metric):
    """Each split holds more rows than its select pool, so BlockSelect prunes during the scan, at k = 129, 1024, 4096."""
    nq, d = 2, 20
    n = 128 * pool_cap(4096) + 4099
    rng = np.random.default_rng(21 + metric)
    c = FlatCase(oracle, metric, rows(rng, n, d), rng.permutation(np.arange(1, n + 1, dtype=np.int64)))
    xq = rows(rng, nq, d)
    for k in (129, 1024, 4096):
        nsplit = scan_nsplit(nq, n, sms)
        assert nsplit == 128 and n // nsplit > pool_cap(k), "premise: rows per split exceed the pool"
        c.search(xq, k, route="scan")


def test_largest_k(oracle):
    """The largest k whose select pool fits 227 KB is answered exactly; one more is refused with EILLEGAL_PARAMETERS and
    the index keeps answering."""
    d, n = 8, 20000
    kmax = max(k for k in range(1, 20000) if scan_smem(d, 1, k) <= MAX_SMEM)
    assert kmax == 8192 and pool_cap(kmax) == 16384, "premise: the pool formula"
    rng = np.random.default_rng(31)
    c = FlatCase(oracle, L2, rows(rng, n, d), rng.permutation(np.arange(1, n + 1, dtype=np.int64)))
    xq = rows(rng, 2, d)
    c.search(xq, kmax, route="scan")
    for call in (lambda: c.ix.search(xq, kmax + 1), lambda: c.ix.range_search(xq, 1e9, kmax + 1)):
        with pytest.raises(b200vs.B200VSError) as e:
            call()
        assert e.value.code == b200vs.EILLEGAL_PARAMETERS
    c.search(xq, 100, route="scan")
    c.search(xq[:1], 10, route="small")


@pytest.mark.parametrize("metric", [L2, IP, COSINE])
def test_exact_merge_branches(oracle, sms, metric):
    """nsplit = 1 (the merge copies through) from a full batch and from a small table; nsplit = 128 from one query."""
    rng = np.random.default_rng(41 + metric)
    d = 24
    n = 5000
    c = FlatCase(oracle, metric, rows(rng, n, d), rng.permutation(np.arange(1, n + 1, dtype=np.int64)))
    nq = 4 * sms
    assert scan_nsplit(nq, n, sms) == 1
    c.search(rows(rng, nq, d), 10, route="scan", exact_only=True, f64_queries=range(0, nq, 61))
    small = FlatCase(oracle, metric, rows(rng, 1000, d), np.arange(1, 1001, dtype=np.int64))
    assert scan_nsplit(3, 1000, sms) == 1
    small.search(rows(rng, 3, d), 50, route="scan", exact_only=True)
    small.search(rows(rng, 3, d), 1000, route="scan")  # k = every row
    n = 70000
    big = FlatCase(oracle, metric, rows(rng, n, d), rng.permutation(np.arange(1, n + 1, dtype=np.int64)))
    assert scan_nsplit(1, n, sms) == 128
    big.search(rows(rng, 1, d), 50, route="scan", exact_only=True)
    big.search(rows(rng, 1, d), 200, route="scan")


def test_grid_limit(oracle):
    """65,535 queries are answered on the exact path; 65,536 are refused with EILLEGAL_PARAMETERS."""
    rng = np.random.default_rng(51)
    n, d = 300, 8
    c = FlatCase(oracle, L2, rows(rng, n, d), np.arange(1, n + 1, dtype=np.int64))
    xq = rows(rng, MAX_NQ + 1, d)
    c.search(xq[:MAX_NQ], 5, route="scan", exact_only=True, f64_queries=[0, 1, MAX_NQ // 2, MAX_NQ - 1])
    with pytest.raises(b200vs.B200VSError) as e:
        c.ix.search(xq, 5, exact_only=True)
    assert e.value.code == b200vs.EILLEGAL_PARAMETERS
    c.search(xq[:3], 5, route="scan", exact_only=True)


class IvfCase:
    """An IVF-Flat index on given centroids (rows are assigned by the engine, checked against oracle.assign)."""

    def __init__(self, o, metric, cent, xb, ids):
        self.o, self.metric, self.cent, self.nlist, self.d = o, metric, np.ascontiguousarray(cent, np.float32), len(cent), cent.shape[1]
        self.ix = b200vs.Index(IVF_FLAT, metric, self.d, nlist=self.nlist)
        self.ix.set_trained_state(b200vs.ivf_state_blob(self.cent, metric))
        self.ix.add(xb, ids)
        self.ix.coalescing(0)
        self.refresh()

    def refresh(self):
        self.off, self.X, _, self.ids = self.ix.export_lists(self.nlist)

    def probe_order(self, q):
        """Lists in the coarse quantiser's order (exact FP32 ranking, ties by list id)."""
        _, order = self.o.flat_search(self.metric, self.cent, np.arange(self.nlist, dtype=np.int64), q[None, :], self.nlist)
        return order[0]

    def search(self, xq, k, nprobe, **filt):
        D, I = self.ix.search(xq, k, nprobe=nprobe, **filt)
        Do, Io = self.o.ivfflat_search(self.metric, self.cent, self.off, self.X, self.ids, xq, k, nprobe, nthreads=8, **filt)
        assert_same_results(D, I, Do, Io)
        check_f64(self.X, self.ids, prep(self.o, self.metric, xq), self.metric, D, I, every_row=min(nprobe, self.nlist) == self.nlist,
                  cand=cand_mask(self.ids, **filt))
        return D, I


def subspace_ivf(o, metric, n, nbig, islands, seed, d=16, h=10.0):
    """Rows (u, 0) with u uniform in [0, 1)^(d/2); nbig centroids among them; one island centroid (a, h e_0) per entry of
    `islands` = [(a, rows)] (or a function of the big centroids returning it), each with `rows` rows at exactly its
    centroid.  A row (u, 0) is at least h from every island centroid and within sqrt(d/2) of every big one, so island
    lists hold exactly their own rows; a query (q, h/2 e_0) is h/2 off every centroid in the second half, so its probe
    order is the order of the first halves."""
    rng = np.random.default_rng(seed)
    half = d // 2
    xb = np.zeros((n, d), np.float32)
    xb[:, :half] = rng.random((n, half))
    big = np.zeros((nbig, d), np.float32)
    big[:, :half] = xb[rng.choice(n, nbig, replace=False), :half] + 0.01 * rng.standard_normal((nbig, half))
    if callable(islands):
        islands = islands(big)
    cent = np.concatenate([big, np.zeros((len(islands), d), np.float32)])
    extra = []
    for j, (a, r) in enumerate(islands):
        cent[nbig + j, :half] = a
        cent[nbig + j, half] = h
        extra += [cent[nbig + j]] * r
    if extra:
        xb = np.concatenate([xb, np.stack(extra)])
    ids = np.arange(1, len(xb) + 1, dtype=np.int64)
    return IvfCase(o, metric, cent, xb, ids), rng


def test_ivf_probing_and_empty_lists(oracle):
    """nlist = 2085 (>= 2048, not a multiple of 32), nprobe 1 / 31 / 32 / 33 / 100 / nlist: the warp-chunked prefix scan of
    the probed list lengths and its carry.  Empty lists first, in the middle and last in the query's probe order; then a
    probed list whose rows are all deleted."""
    nlist, nbig = 2085, 2082
    q1 = np.random.default_rng(61).random(8).astype(np.float32)
    qf = np.concatenate([q1, [5.0], np.zeros(7)]).astype(np.float32)

    def islands(big):  # the island in the middle sits next to the big centroid 15th closest to the query
        mid = big[np.argsort(((big[:, :8] - q1).astype(np.float64) ** 2).sum(1))[15], :8] + np.float32(1e-3)
        return [(q1, 0), (mid, 0), (q1 + 20, 0)]
    s, rng = subspace_ivf(oracle, L2, 40000, nbig, islands, seed=62)
    assert s.nlist == nlist and nlist % 32 and (np.diff(s.off)[nbig:] == 0).all(), "premise: three empty lists"
    order = s.probe_order(qf).tolist()
    ranks = [order.index(nbig), order.index(nbig + 1), order.index(nbig + 2)]
    assert ranks[0] == 0 and 1 < ranks[1] < 30 and ranks[2] == nlist - 1, f"premise: probe ranks {ranks}"
    xq = np.stack([qf, np.concatenate([rng.random(8), [5.0], np.zeros(7)]).astype(np.float32)])
    D, I = s.search(xq[:1], 20, nprobe=1)  # the one probed list is empty
    assert (I == -1).all()
    for nprobe in (1, 31, 32, 33, 100, nlist):
        s.search(xq, 20, nprobe)
    s.search(xq, 300, 100)
    dead = order[1]  # the first non-empty list of the query
    lo, hi = s.off[dead], s.off[dead + 1]
    assert hi > lo and s.ix.delete(s.ids[lo:hi]) == hi - lo
    s.refresh()
    assert s.off[dead + 1] == s.off[dead]
    D, I = s.search(xq[:1], 20, nprobe=2)  # an empty list and a dead one
    assert (I == -1).all()
    for nprobe in (3, 33, nlist):
        s.search(xq, 20, nprobe)


@pytest.mark.parametrize("metric", [L2, IP])
def test_ivf_probing_random(oracle, metric):
    """The same probe counts on unstructured data, nq below 16 (the list scan is the exact path), with filters."""
    rng = np.random.default_rng(71 + metric)
    n, d, nlist = 40000, 16, 2085
    xb = rows(rng, n, d)
    cent = xb[rng.choice(n, nlist, replace=False)] + (0.1 * rng.standard_normal((nlist, d))).astype(np.float32)
    s = IvfCase(oracle, metric, cent, xb, np.arange(1, n + 1, dtype=np.int64))
    assert np.array_equal(np.diff(s.off), np.bincount(oracle.assign(metric, xb, cent), minlength=nlist))
    xq = rows(rng, 5, d)
    for nprobe in (1, 31, 32, 33, 100, nlist):
        s.search(xq, 20, nprobe)
    s.search(xq, 129, 100)
    s.search(xq, 20, 33, id_range=(1000, 30000))
    s.search(xq, 20, nlist, sorted_ids=np.arange(1, n + 1, 7), negate=True)


def test_ivf_splits_that_scan_nothing(oracle, sms):
    """A query whose probed lists hold fewer rows than the splits its scan is cut into (the split count follows the
    index-wide average list length): some splits scan nothing."""
    s, rng = subspace_ivf(oracle, L2, 30000, 20, [(np.full(8, 0.5, np.float32), 1), (np.full(8, 0.51, np.float32), 1),
                                                  (np.full(8, 0.52, np.float32), 0), (np.full(8, 0.53, np.float32), 1)], seed=81)
    nprobe = 4
    q = s.cent[20].copy()
    order = s.probe_order(q)
    assert set(order[:nprobe].tolist()) == {20, 21, 22, 23}, "premise: the query probes the islands"
    probed = int(sum(s.off[l + 1] - s.off[l] for l in order[:nprobe]))
    nsplit = scan_nsplit(1, s.ix.get_count() * nprobe / s.nlist, sms)
    assert probed == 3 and nsplit > probed, f"premise: {probed} probed rows over {nsplit} splits"
    D, I = s.search(q[None, :], 10, nprobe)
    assert (I[0, :3] >= 0).all() and (I[0, 3:] == -1).all()
    s.search(np.stack([q, s.cent[0]]), 10, nprobe)


# =====================================================================================================================
# C. range search
# =====================================================================================================================

def range_expect(X, ids, q, metric, radius, max_results, cand=None):
    """(ids, API distances, hit count) one query must return: every candidate row strictly inside the FP32 threshold
    (L2: raw < radius; IP / cosine: raw > fl32(1 - fl32(radius))), in (key, id) order, at most max_results."""
    raw = raw_fp32(X, q, metric)
    if metric == L2:
        keep, key = raw < np.float32(radius), raw
    else:
        keep, key = raw > np.float32(1) - np.float32(radius), -raw
    if cand is not None:
        keep &= cand
    idx = np.nonzero(keep)[0]
    idx = idx[np.lexsort((ids[idx], key[idx]))]
    c = min(len(idx), max_results)
    return ids[idx[:c]], api_of(raw, metric)[idx[:c]], len(idx)


def check_range(ix, X, ids, Q, xq, metric, radius, max_results, cand=None, **kw):
    """Range search == the restated expectation (ids, counts, distance bits); returns the hit counts."""
    D, I, C = ix.range_search(xq, radius, max_results, **kw)
    hits = []
    for qi in range(len(xq)):
        want_i, want_d, h = range_expect(X, ids, Q[qi], metric, radius, max_results, cand)
        assert C[qi] == len(want_i), f"query {qi}: {C[qi]} hits, expected {len(want_i)}"
        assert np.array_equal(I[qi, :C[qi]], want_i) and (I[qi, C[qi]:] == -1).all()
        assert np.array_equal(D[qi, :C[qi]].view(np.uint32), want_d.view(np.uint32))
        assert (D[qi, C[qi]:] == 0).all()
        hits.append(h)
    check_f64(X, ids, Q, metric, D, I, every_row=False, queries=range(min(len(xq), 8)))
    return hits


def check_restatement(o, metric, X, ids, xq, Q, k=300):
    """raw_fp32 reproduces the kernel's distances bit for bit (the oracle's top-k)."""
    Do, Io = o.flat_search(metric, X, ids, xq, k, nthreads=8)
    pos = {int(i): r for r, i in enumerate(ids.tolist())}
    for qi in range(len(xq)):
        r = [pos[int(i)] for i in Io[qi] if i >= 0]
        api = api_of(raw_fp32(X[r], Q[qi], metric), metric)
        assert np.array_equal(api.view(np.uint32), Do[qi][:len(r)].view(np.uint32)), "numpy restatement is not bit-exact"


def radius_for(raw, metric, hits):
    """A radius that keeps about `hits` rows of one query."""
    srt = np.sort(raw) if metric == L2 else np.sort(raw)[::-1]
    t = srt[min(hits, len(srt) - 1)]
    return float(t) if metric == L2 else float(np.float32(1) - t)


def boundary_radius(raw, metric, start=30):
    """(row, radius) with the FP32 threshold equal to that row's raw value: the row must be excluded."""
    order = np.argsort(raw) if metric == L2 else np.argsort(-raw)
    for j in order[start:]:
        if metric == L2:
            return j, float(raw[j])
        up = down = np.float32(1) - raw[j]
        cands = [up]
        for _ in range(4):
            up, down = np.nextafter(up, np.float32(np.inf)), np.nextafter(down, np.float32(-np.inf))
            cands += [up, down]
        ok = [c for c in cands if np.float32(1) - c == raw[j]]
        if ok:
            return j, float(ok[0])
    pytest.fail("no radius maps onto a row's raw value")


@pytest.mark.parametrize("metric", [L2, IP, COSINE])
def test_flat_range_search(oracle, sms, metric):
    """More hits than max_results (1, 64, 4096) with splits that see more hits than their pool (it prunes against the fixed
    threshold), the strict boundary, zero hits, filters and tombstones, nq = 1 and a batch with one split per query."""
    rng = np.random.default_rng(91 + metric)
    n, d = 30000, 24
    c = FlatCase(oracle, metric, rows(rng, n, d), rng.permutation(np.arange(1, n + 1, dtype=np.int64)))
    X, ids = c.X, c.ids
    xq = rows(rng, 3, d)
    Q = prep(oracle, metric, xq)
    check_restatement(oracle, metric, X, ids, xq, Q)
    nsplit = scan_nsplit(1, n, sms)
    assert n // nsplit > pool_cap(64), "premise: a split sees more hits than the pool holds"
    for mr in (1, 64, 4096):
        hits = check_range(c.ix, X, ids, Q[:1], xq[:1], metric, 1e30, mr)  # every row is a hit
        assert hits[0] == n
    radius = radius_for(raw_fp32(X, Q[0], metric), metric, 6000)
    for mr in (1, 64, 4096):
        hits = check_range(c.ix, X, ids, Q[:1], xq[:1], metric, radius, mr)
        assert hits[0] > mr
    check_range(c.ix, X, ids, Q, xq, metric, radius, 64)
    # strict boundary
    raw = raw_fp32(X, Q[0], metric)
    j, r = boundary_radius(raw, metric)
    D, I, C = c.ix.range_search(xq[:1], r, 256)
    assert ids[j] not in I[0, :C[0]], "the row on the boundary must be excluded"
    check_range(c.ix, X, ids, Q[:1], xq[:1], metric, r, 256)
    # zero hits
    top = max(raw_fp32(X, Q[qi], metric).max() for qi in range(len(xq)))
    none = 0.0 if metric == L2 else float(np.float32(1) - top - np.float32(0.01))
    D, I, C = c.ix.range_search(xq, none, 64)
    assert (C == 0).all() and (I == -1).all() and (D == 0).all()
    # filters, then tombstones
    sub = np.sort(rng.choice(ids, 4000, replace=False))
    for filt in (dict(id_range=(5000, 20000)), dict(sorted_ids=sub), dict(sorted_ids=sub, negate=True),
                 dict(id_range=(5000, 20000), sorted_ids=sub)):
        check_range(c.ix, X, ids, Q, xq, metric, radius, 512, cand=cand_mask(ids, **filt), **filt)
    c.delete(np.arange(1, 10001, dtype=np.int64))
    check_range(c.ix, c.X, c.ids, Q, xq, metric, radius, 4096)
    # a batch large enough for one split per query
    m = 3000
    b = FlatCase(oracle, metric, rows(rng, m, d), np.arange(1, m + 1, dtype=np.int64))
    nq = 4 * sms
    assert scan_nsplit(nq, m, sms) == 1 and m > pool_cap(64)
    xb = rows(rng, nq, d)
    Qb = prep(oracle, metric, xb)
    rb = radius_for(raw_fp32(b.X, Qb[0], metric), metric, 1500)
    check_range(b.ix, b.X, b.ids, Qb, xb, metric, rb, 64)


@pytest.mark.parametrize("metric", [L2, IP, COSINE])
def test_ivf_range_search(oracle, metric):
    """Untrained: no hits.  Trained: every probed row inside the threshold and nothing else; with nprobe < nlist the
    candidates are exactly the probed lists' rows (taken from oracle.ivfflat_search at k = every row)."""
    rng = np.random.default_rng(101 + metric)
    n, d, nlist = 8000, 24, 40
    un = b200vs.Index(IVF_FLAT, metric, d, nlist=nlist)
    D, I, C = un.range_search(rows(rng, 2, d), 1e9, 16)
    assert (C == 0).all() and (I == -1).all()
    xb = rows(rng, n, d)
    stored = prep(oracle, metric, xb)
    cent = stored[rng.choice(n, nlist, replace=False)] + (0.05 * rng.standard_normal((nlist, d))).astype(np.float32)
    s = IvfCase(oracle, metric, cent, xb, np.arange(1, n + 1, dtype=np.int64))
    xq = rows(rng, 4, d)
    Q = prep(oracle, metric, xq)
    check_restatement(oracle, metric, s.X, s.ids, xq, Q)
    radius = radius_for(raw_fp32(s.X, Q[0], metric), metric, 1500)
    check_range(s.ix, s.X, s.ids, Q, xq, metric, radius, 4096, nprobe=nlist)
    check_range(s.ix, s.X, s.ids, Q, xq, metric, radius, 64, nprobe=nlist)
    for nprobe, filt in ((5, {}), (5, dict(id_range=(1000, 6000))), (12, dict(sorted_ids=np.arange(1, n + 1, 3), negate=True))):
        _, Io = oracle.ivfflat_search(metric, s.cent, s.off, s.X, s.ids, xq, n, nprobe, nthreads=8)
        for qi in range(len(xq)):
            probed = np.isin(s.ids, Io[qi][Io[qi] >= 0])
            cand = probed & cand_mask(s.ids, **filt)
            D, I, C = s.ix.range_search(xq[qi:qi + 1], radius, 2048, nprobe=nprobe, **filt)
            want_i, want_d, h = range_expect(s.X, s.ids, Q[qi], metric, radius, 2048, cand)
            assert C[0] == len(want_i) and np.array_equal(I[0, :C[0]], want_i)
            assert np.array_equal(D[0, :C[0]].view(np.uint32), want_d.view(np.uint32))
    s.ix.delete(np.arange(1, 2001, dtype=np.int64))
    s.refresh()
    check_range(s.ix, s.X, s.ids, Q, xq, metric, radius, 4096, nprobe=nlist)
