"""Range search at its edges: the parts of the tile range scan (tc_range_search, DESIGN.md 4.6) that benign data does not
reach, and the radii no data can make ordinary.

* Capture-window decoys: R is a hit by one FP32 step of the threshold while its tile score lies well above its true
  score (tf32_emu / fp16_emu decoys), so only a capture threshold widened by the full eps keeps it.
* Whole-list coverage: radii that admit exactly one list, on lists whose lengths sit around the 32-row box, 128-row
  tile, 512-row chunk and 2048-row span, so a dropped row of any of them is an error.
* Partial capture overflow: only some queries of a batch overflow the capture buffer, at non-contiguous positions, so
  the exact re-run must write each one back to its own row (qmap), also through the sharded step's raw output.
* The finish without tc_final_hybrid_kernel (d * 4 > 96 KB) and the largest dimensions.
* Non-finite and extreme radii on every float range path: a NaN radius admits no row.

Every search is compared with exact_only (ids, distance bits, counts) and with the restated rule range_expect, and the
route is read from stats(): [1] = queries served by the tile pass, [2] = queries it handed to the exact scan."""
import numpy as np
import pytest

import b200vs
import fp16_emu as H
import tf32_emu as E
from b200vs import COSINE, FLAT, IP, IVF_FLAT, L2
from gpu_util import assert_same_results, require_gpu
from test_gpu_exact_edges import MAX_SMEM, cand_mask, check_f64, pool_cap, prep, radius_for, raw_fp32, scan_smem
from test_gpu_range_tile import Case
from test_gpu_tc_adversarial import LENGTHS, far_centroids

gpu = pytest.mark.gpu
FLT_MAX = float(np.finfo(np.float32).max)


def tc_cand_cap(k):
    """tc_cand_cap (csrc/tc_scan.cu): capture slots per query."""
    return min(16384, max(8192, 1 << max(0, (256 * k - 1).bit_length())))


class Built(Case):
    """Case's checks (range == exact_only with the route asserted, expect == range_expect) on an index built by the
    test itself: a hand-made list layout or decoy rows."""

    def __init__(self, o, kind, metric, rows, ids, cent=None):
        self.o, self.kind, self.metric, self.d = o, kind, metric, rows.shape[1]
        self.nlist = 1 if kind == FLAT else len(cent)
        if kind == FLAT:
            self.ix = b200vs.Index(FLAT, metric, self.d)
        else:
            self.ix = b200vs.Index(IVF_FLAT, metric, self.d, nlist=self.nlist)
            self.ix.set_trained_state(b200vs.ivf_state_blob(cent, metric))
        for a in range(0, len(ids), 32768):
            self.ix.add(rows[a:a + 32768], ids[a:a + 32768])
        self.ix.coalescing(0)
        self.ix.set_profiling(True)
        self.refresh()

    def refresh(self):
        self.off, self.X, _, self.ids = self.ix.export_lists(self.nlist)

    def kw(self, nprobe):
        return {} if self.kind == FLAT else dict(nprobe=self.nlist)


def same(a, b):
    assert np.array_equal(a[2], b[2]), "counts differ"
    assert np.array_equal(a[1], b[1]), "ids differ"
    assert np.array_equal(a[0].view(np.uint32), b[0].view(np.uint32)), "distance bits differ"


# =====================================================================================================================
# 1. capture-window decoys
# =====================================================================================================================
# name -> (index kind, metric, generator, d): Flat scans TF32 rows, IVF-Flat at d % 8 == 0 its FP16 mirror and at
# d = 132 (no mirror) its rows in the TF32 list form
DECOYS = {"tf32-L2": (FLAT, L2, E.decoy_l2, 128), "tf32-IP": (FLAT, IP, E.decoy_ip, 128),
          "fp16-L2": (IVF_FLAT, L2, H.decoy_l2, 128), "fp16-IP": (IVF_FLAT, IP, H.decoy_ip, 128),
          "fp16-cos": (IVF_FLAT, COSINE, H.decoy_cos, 128),
          "tf32list-L2": (IVF_FLAT, L2, E.decoy_l2, 132), "tf32list-IP": (IVF_FLAT, IP, E.decoy_ip, 132)}
NPAIR = 32


def decoy_pairs(name):
    gen, d = DECOYS[name][2:]
    return [gen(np.random.default_rng(7000 + p), d, 1, nfill=1500) for p in range(NPAIR)]


def decoy_centroids(d):
    """Centroid 0 = 0, the others far out on filler axes: every pair row lands in list 0 (as in test_decoys)."""
    cent = np.zeros((4, d), np.float32)
    cent[1:, d // 2:d // 2 + 3] = -1000 * np.eye(3, dtype=np.float32)
    return cent


def tight_radius(rows, q, r, metric):
    """(radius, FP32 threshold) that makes row r a hit by the smallest margin FP32 allows.  L2: the next float above R's
    raw distance.  IP: the first radius, walking up from 1 - ip_R, whose fl(1 - r) lies below R's raw inner product."""
    raw = raw_fp32(rows[r:r + 1], q, metric)[0]
    if metric == L2:
        rad = np.nextafter(raw, np.float32(np.inf))
        return float(rad), rad
    rad = np.float32(1) - raw
    for _ in range(16):
        if np.float32(1) - rad < raw:
            return float(rad), np.float32(1) - rad
        rad = np.nextafter(rad, np.float32(np.inf))
    pytest.fail("no radius puts the threshold just below R")


def window_share(approx_r, rows, q, r, thr, eps, metric):
    """(R's tile score - its true score - the threshold's slack) / eps.  The capture threshold is T = thr - ||q||^2 + qerr +
    eps for L2 (-thr + eps for IP); the slack is what thr lies beyond R's true value plus, for L2, twice the qerr
    allowance for the FP32 query norm.  Above 0.5, a threshold widened by eps / 2 misses R."""
    x64, q64 = rows[r].astype(np.float64), q.astype(np.float64)
    d = rows.shape[1]
    if metric == L2:
        qn = float(q64 @ q64)
        true = float(x64 @ x64 - 2 * (q64 @ x64))
        qerr = (d + 64) * 2.0 ** -24 * qn + d * 2.0 ** -149
        slack = float(thr) - (true + qn) + 2 * qerr
    else:
        true = -float(q64 @ x64)
        slack = -true - float(thr)
    assert slack >= 0, "premise: R is a hit"
    return (approx_r - true - slack) / eps


@pytest.mark.parametrize("name", list(DECOYS))
def test_decoy_premise(name):
    """On the CPU emulators: R's tile score sits above its true score by more than half of eps beyond the threshold's
    slack, so the decoy test below fails for a kernel whose capture threshold is widened by eps / 2."""
    kind, metric, _, _ = DECOYS[name]
    l2 = metric == L2
    for p, (rows, q, r, _) in enumerate(decoy_pairs(name)):
        _, thr = tight_radius(rows, q[0], r, metric)
        if name.startswith("fp16"):
            approx, eps = H.approx_scores(rows[r:r + 1], q, l2)[0, 0], H.emulated_eps(rows, q, l2)[0]
        else:
            approx, eps = E.approx_scores(rows[r:r + 1], q, l2, False)[0, 0], E.emulated_eps(rows, q, l2, False)[0]
        share = window_share(float(approx), rows, q[0], r, thr, float(eps), metric)
        assert share > 0.5, f"pair {p}: R uses {share:.3f} eps of the window"


@gpu
@pytest.mark.parametrize("name", list(DECOYS))
def test_decoy_is_captured(oracle, name):
    """Index p holds pair p among filler rows; the radius admits R by one FP32 step.  The whole 32-query batch stays on
    the tile pass (nothing re-run), R comes back, and every answer equals the exact scan and the restated rule."""
    require_gpu()
    kind, metric, _, d = DECOYS[name]
    pairs = decoy_pairs(name)
    xq = np.concatenate([p[1] for p in pairs])
    for p in range(0, NPAIR, 4):
        rows, q, r, _ = pairs[p]
        ids = np.arange(rows.shape[0], dtype=np.int64) * 7 + 3
        c = Built(oracle, kind, metric, rows, ids, cent=decoy_centroids(d) if kind == IVF_FLAT else None)
        radius, thr = tight_radius(rows, q[0], r, metric)
        if kind == FLAT:  # the device's own score and eps (TF32 list-scan arithmetic, rows in insertion order)
            S, Eps = c.ix.tc_scores(np.repeat(q, 16, axis=0))
            share = window_share(float(S[0, r]), rows, q[0], r, thr, float(Eps[0]), metric)
            assert share > 0.5, f"pair {p}: on the device R uses {share:.3f} eps of the window"
        D, I, C = c.range(xq, radius, 64, "tile")
        assert c.stats[2] == 0, f"pair {p}: a query was re-run, stats {c.stats}"
        assert ids[r] in I[p, :C[p]], f"pair {p}: R was not captured"
        c.expect(D, I, C, xq, radius, 64, range(NPAIR))
        check_f64(c.X, c.ids, prep(oracle, metric, xq), metric, D, I, every_row=False, queries=[p])
        # a batch of the decoy query alone
        D, I, C = c.range(np.repeat(q, 16, axis=0), radius, 64, "tile")
        assert c.stats[2] == 0 and (C >= 1).all() and all(ids[r] in I[i, :C[i]] for i in range(16))
        c.ix.close()


# =====================================================================================================================
# 2. whole-list coverage
# =====================================================================================================================
LIST_D, LIST_RADIUS, LIST_MR = 64, 1000.0, 4096


def list_layout(oracle, seed):
    """LENGTHS rows per list around far_centroids (as test_list_length_edges), the longest added last; rows are
    cent + U[0, 1)^d, so a query at cent + 0.5 is within 16 of every row of its list and over 10^4 from every other."""
    rng = np.random.default_rng(seed)
    nlist = len(LENGTHS)
    cent = far_centroids(nlist, LIST_D, 100.0)
    next_id = [1]

    def rows_of(l, m):
        x = (cent[l] + rng.random((m, LIST_D))).astype(np.float32)
        i = np.arange(next_id[0], next_id[0] + m, dtype=np.int64)
        next_id[0] += m
        return x, i

    order = [l for l in np.argsort(LENGTHS, kind="stable") if LENGTHS[l]]
    c = Built(oracle, IVF_FLAT, L2, *rows_of(order[0], LENGTHS[order[0]]), cent=cent)
    for l in order[1:]:
        c.ix.add(*rows_of(l, LENGTHS[l]))
    c.refresh()
    return c, cent, rows_of, rng


def near(cent, lists, rng):
    return (cent[lists] + np.float32(0.5) + (0.01 * rng.standard_normal((len(lists), cent.shape[1])))).astype(np.float32)


def check_whole_lists(c, cent, rng, lengths):
    """Two queries per list: each must return every row of its list, nothing else, on the tile pass."""
    assert list(np.diff(c.off)) == lengths
    lists = np.repeat(np.arange(len(lengths)), 2)
    xq = near(cent, lists, rng)
    D, I, C = c.range(xq, LIST_RADIUS, LIST_MR, "tile")
    assert c.stats[2] == 0, c.stats
    for qi, l in enumerate(lists):
        mine = c.ids[c.off[l]:c.off[l + 1]]
        assert C[qi] == min(len(mine), LIST_MR), f"list {l} ({len(mine)} rows): {C[qi]} hits"
        assert set(I[qi, :C[qi]].tolist()) <= set(mine.tolist())
        if len(mine) <= LIST_MR:
            assert np.array_equal(np.sort(I[qi, :C[qi]]), np.sort(mine)), f"list {l}: rows missing"
    c.expect(D, I, C, xq, LIST_RADIUS, LIST_MR, range(len(xq)))
    # lists longer than max_results: each half by an id filter
    for l in np.nonzero(np.array(lengths) > LIST_MR)[0]:
        mine = np.sort(c.ids[c.off[l]:c.off[l + 1]])
        mid = int(mine[len(mine) // 2])
        xl = near(cent, np.full(16, l), rng)
        for lo, hi in ((int(mine[0]), mid), (mid, int(mine[-1]) + 1)):
            D, I, C = c.range(xl, LIST_RADIUS, LIST_MR, "tile", id_range=(lo, hi))
            part = mine[(mine >= lo) & (mine < hi)]
            assert c.stats[2] == 0 and (C == len(part)).all()
            assert all(np.array_equal(np.sort(I[i, :C[i]]), part) for i in range(16))
            c.expect(D, I, C, xl, LIST_RADIUS, LIST_MR, range(2), cand=cand_mask(c.ids, id_range=(lo, hi)))


@gpu
def test_whole_lists_come_back(oracle):
    """A radius that admits one whole list: every row of every list length, then after a delete in the 2049-row list and
    after an add that outgrows (relocates) the 32-row list."""
    require_gpu()
    c, cent, rows_of, rng = list_layout(oracle, 21)
    check_whole_lists(c, cent, rng, list(LENGTHS))
    l = LENGTHS.index(2049)
    _, lids = c.ix.export_list(l)
    c.ix.delete(lids[::3])
    c.refresh()
    lengths = list(LENGTHS)
    lengths[l] -= len(lids[::3])
    check_whole_lists(c, cent, rng, lengths)
    grow = LENGTHS.index(32)
    c.ix.add(*rows_of(grow, 600))
    c.refresh()
    lengths[grow] += 600
    check_whole_lists(c, cent, rng, lengths)


@gpu
@pytest.mark.parametrize("nq", [127, 128, 129, 257])
def test_whole_list_query_groups(oracle, nq):
    """Every query on the 2048-row list: query groups of 128 columns, with a group of one query at 129 and 257."""
    require_gpu()
    c, cent, _, rng = list_layout(oracle, 30 + nq)
    l = LENGTHS.index(2048)
    mine = np.sort(c.ids[c.off[l]:c.off[l + 1]])
    xq = near(cent, np.full(nq, l), rng)
    D, I, C = c.range(xq, LIST_RADIUS, 2048, "tile")
    assert c.stats[2] == 0 and (C == 2048).all()
    assert all(np.array_equal(np.sort(I[i]), mine) for i in range(nq))
    c.expect(D, I, C, xq, LIST_RADIUS, 2048, [0, 127 % nq, nq - 1])


# =====================================================================================================================
# 3. partial capture overflow
# =====================================================================================================================
@gpu
@pytest.mark.parametrize("kind", [FLAT, IVF_FLAT], ids=["flat", "ivf"])
@pytest.mark.parametrize("metric", [L2, IP], ids=["L2", "IP"])
def test_partial_overflow(oracle, metric, kind):
    """A row duplicated 17 000 times (more than the 16 384 capture slots of max_results 256): the queries on it, at every
    position i % 3 == 1, overflow and are re-run exactly; the random queries (orthogonal to it) stay on the tile pass.
    Both halves must land in their own rows, in the plain call and in the sharded step at world 1 (raw_out re-run)."""
    require_gpu()
    import torch
    rng = np.random.default_rng(40 + metric)
    d, n, ndup, nq, mr = 32, 12000, 17000, 48, 256
    assert ndup > tc_cand_cap(mr), "premise: the duplicates overflow the capture buffer"
    dup = np.zeros(d, np.float32)
    dup[0] = 20
    xb = np.concatenate([rng.standard_normal((n, d)).astype(np.float32), np.repeat(dup[None, :], ndup, axis=0)])
    ids = rng.permutation(np.arange(1, n + ndup + 1, dtype=np.int64))
    cent = xb[rng.choice(n, 32, replace=False)] if kind == IVF_FLAT else None
    c = Built(oracle, kind, metric, xb, ids, cent=cent)
    xq = rng.standard_normal((nq, d)).astype(np.float32)
    xq[:, 0] = 0
    over = np.arange(nq) % 3 == 1
    xq[over] = dup
    radius = radius_for(raw_fp32(c.X, xq[0], metric), metric, 40)
    D, I, C = c.range(xq, radius, mr, "tile")
    assert c.stats[2] == over.sum(), f"exactly the {over.sum()} duplicate queries must be re-run, stats {c.stats}"
    assert (C[over] == mr).all() and C[~over].sum() > 0
    c.expect(D, I, C, xq, radius, mr, range(8))
    check_f64(c.X, c.ids, xq, metric, D, I, every_row=False, queries=[0, 2, 3, 5])
    if kind == FLAT:
        return
    sh = b200vs.Shard(c.ix, 0, 1, None)
    same(sh.range_search(xq, radius, mr, nprobe=c.nlist), (D, I, C))
    assert c.ix.stats()[2] == over.sum(), "the sharded step must re-run the same queries"
    qd = torch.from_numpy(xq).cuda()
    od = torch.empty((nq, mr), dtype=torch.float32, device="cuda")
    oi = torch.empty((nq, mr), dtype=torch.int64, device="cuda")
    oc = torch.empty((nq,), dtype=torch.int32, device="cuda")
    sp, _keep = b200vs.make_search_params(nprobe=c.nlist)
    torch.cuda.synchronize()
    sh.range_search_device(nq, qd.data_ptr(), radius, mr, od.data_ptr(), oi.data_ptr(), oc.data_ptr(), sp=sp)
    torch.cuda.synchronize()
    same((od.cpu().numpy(), oi.cpu().numpy(), oc.cpu().numpy()), (D, I, C))
    sh.close()


# =====================================================================================================================
# 4. the finish without its hybrid kernel, and the largest dimensions
# =====================================================================================================================
FIN_SEG = 2048  # csrc/tc_scan.cu


def tc_stream_smem(d, k):
    return (4 * d + 15) // 16 * 16 + FIN_SEG * 4 + pool_cap(k) * 12 + 32


@gpu
@pytest.mark.parametrize("d", [24576, 24580, 32760, 32768])
@pytest.mark.parametrize("kind", [FLAT, IVF_FLAT], ids=["flat", "ivf"])
def test_largest_dimensions(oracle, kind, d):
    """d * 4 > 96 KB (d > 24576) skips tc_final_hybrid_kernel: tc_final_kernel finishes every query.  24576 is the last d
    with the hybrid kernel, 24580 the first without (TF32 rows, d % 8 == 4); 32760 with max_results 1024 is the largest
    tile-eligible range shape (the streaming finish needs exactly 160 KB); at 32768 range search takes the exact scan."""
    require_gpu()
    rng = np.random.default_rng(d)
    n, nq = (8300 if (kind, d) == (FLAT, 24580) else 2000), 16
    xb = rng.standard_normal((n, d)).astype(np.float32)
    ids = rng.permutation(np.arange(1, n + 1, dtype=np.int64))
    c = Built(oracle, kind, L2, xb, ids, cent=xb[:8] if kind == IVF_FLAT else None)
    xq = rng.standard_normal((nq, d)).astype(np.float32)
    # top-k on the tile path
    D, I = c.ix.search(xq, 10, **c.kw(0))
    st = c.ix.stats()
    assert st[1] == nq, f"top-k: expected the tile pass, stats {st}"
    De, Ie = c.ix.search(xq, 10, exact_only=True, **c.kw(0))
    assert_same_results(D, I, De, Ie)
    check_f64(c.X, c.ids, xq, L2, D, I, every_row=True, queries=[0, nq - 1])
    # range
    mr = 1024
    tile = tc_stream_smem(d, mr) <= 160 * 1024
    assert tile == (d < 32768) and (d != 32760 or tc_stream_smem(d, mr) == 160 * 1024), "premise: the finish's smem"
    radius = radius_for(raw_fp32(c.X, xq[0], L2), L2, 300)
    D, I, C = c.range(xq, radius, mr, "tile" if tile else "exact")
    if tile:
        assert c.stats[2] == 0, c.stats
    c.expect(D, I, C, xq, radius, mr, [0, nq - 1])
    if (kind, d) == (FLAT, 24580):  # every row a hit: more rows than the capture slots, the streaming kernel's overflow
        assert n > tc_cand_cap(16)
        D, I, C = c.range(xq, 1e30, 16, "tile")
        assert c.stats[2] == nq and (C == 16).all(), c.stats
        c.expect(D, I, C, xq, 1e30, 16, [0, nq - 1])
    if d == 32768:  # max_results 4096: the exact scan's shared memory (query row + probe prefix + select pool)
        nseg = 1 if kind == FLAT else c.nlist
        assert scan_smem(d, nseg, 4096) <= MAX_SMEM, "premise: the exact scan holds d = 32768 at max_results 4096"
        D, I, C = c.range(xq, radius, 4096, "exact")
        c.expect(D, I, C, xq, radius, 4096, [0])
    c.ix.close()


@gpu
def test_exact_scan_shared_memory_refusal(oracle):
    """IVF-Flat at d = 32768, max_results 4096 and 1024 probes: the query row, the probe prefix and the select pool need
    more than 227 KB, so the call is refused with EILLEGAL_PARAMETERS before any launch, and the index keeps answering."""
    require_gpu()
    rng = np.random.default_rng(5)
    d, nlist, n = 32768, 1024, 2048
    assert scan_smem(d, nlist, 4096) > MAX_SMEM and scan_smem(d, nlist, 1024) <= MAX_SMEM, "premise: the limit"
    xb = rng.standard_normal((n, d)).astype(np.float32)
    c = Built(oracle, IVF_FLAT, L2, xb, np.arange(1, n + 1, dtype=np.int64), cent=xb[:nlist])
    xq = rng.standard_normal((16, d)).astype(np.float32)
    radius = radius_for(raw_fp32(c.X, xq[0], L2), L2, 50)
    with pytest.raises(b200vs.B200VSError) as e:
        c.ix.range_search(xq, radius, 4096, nprobe=nlist)
    assert e.value.code == b200vs.EILLEGAL_PARAMETERS
    D, I, C = c.range(xq, radius, 1024, "exact")
    c.expect(D, I, C, xq, radius, 1024, [0])


# =====================================================================================================================
# 5. non-finite and extreme radii
# =====================================================================================================================
def f32_bits(b):
    return float(np.array([b], np.uint32).view(np.float32)[0])


RADII = {"+nan": f32_bits(0x7FC00000), "-nan": f32_bits(0xFFC00000), "+inf": float("inf"), "-inf": float("-inf"),
         "flt_max": FLT_MAX, "-flt_max": -FLT_MAX}


def every_row_passes(metric, radius):
    """The rule on finite, non-NaN values for these radii: all of them pass or none does."""
    r = np.float32(radius)
    if metric == L2:
        return bool(np.float32(0) < r) and bool(np.float32(1e30) < r)
    thr = np.float32(1) - r
    return bool(np.float32(-1e30) > thr)


def test_radii_are_what_they_claim():
    assert np.isnan(RADII["+nan"]) and not np.signbit(RADII["+nan"])
    assert np.isnan(RADII["-nan"]) and np.signbit(RADII["-nan"])
    for m in (L2, IP, COSINE):
        assert not every_row_passes(m, RADII["+nan"]) and not every_row_passes(m, RADII["-nan"])


@gpu
@pytest.mark.parametrize("metric", [L2, IP, COSINE], ids=["L2", "IP", "cos"])
@pytest.mark.parametrize("kind", [FLAT, IVF_FLAT], ids=["flat", "ivf"])
def test_extreme_radii(oracle, kind, metric):
    """Flat and IVF-Flat with 32 queries (tile pass, re-run) and 8 (exact scan), the sharded call at world 1 and the
    streaming range scan: each equals the restated rule; a NaN radius of either sign returns nothing and launches nothing."""
    require_gpu()
    rng = np.random.default_rng(60 + metric)
    d, n, mr = 32, 3000, 4096
    xb = rng.standard_normal((n, d)).astype(np.float32)
    ids = rng.permutation(np.arange(1, n + 1, dtype=np.int64))
    cent = prep(oracle, metric, xb[rng.choice(n, 16, replace=False)]) if kind == IVF_FLAT else None
    c = Built(oracle, kind, metric, xb, ids, cent=cent)
    xq = rng.standard_normal((32, d)).astype(np.float32)
    sh = b200vs.Shard(c.ix, 0, 1, None) if kind == IVF_FLAT else None
    for name, radius in RADII.items():
        nan = np.isnan(radius)
        for nq in (32, 8):
            D, I, C = c.range(xq[:nq], radius, mr, "exact" if nan or nq < 16 else "tile")
            if nan:
                assert c.ix.stats()[0] == 0, "a NaN radius launches nothing"
                assert (C == 0).all() and (I == -1).all() and (D == 0).all(), f"{name}: hits for a NaN radius"
            assert ((C == n) if every_row_passes(metric, radius) else (C == 0)).all(), f"{name}: counts {C[:4]}"
            c.expect(D, I, C, xq[:nq], radius, mr, range(3))
            if sh is not None:
                same(sh.range_search(xq[:nq], radius, mr, nprobe=c.nlist), (D, I, C))
        rs = b200vs.BruteForceRangeScan(metric, d, xq[:8], radius, max_results=mr)
        for a in range(0, n, 1024):
            rs.push(xb[a:a + 1024], ids[a:a + 1024])
        Ds, Is, Cs = rs.finish()
        Db, Ib, Cb = c.ix.range_search(xq[:8], radius, mr)
        assert np.array_equal(Cs, Cb), f"{name}: streaming range scan counts"
        for qi in range(8):
            assert sorted(zip(Is[qi, :Cs[qi]].tolist(), Ds[qi, :Cs[qi]].view(np.uint32).tolist())) == \
                sorted(zip(Ib[qi, :Cb[qi]].tolist(), Db[qi, :Cb[qi]].view(np.uint32).tolist())), f"{name}: streaming scan, query {qi}"
    if sh is not None:
        sh.close()


@gpu
@pytest.mark.parametrize("nbits", [8, 4])
@pytest.mark.parametrize("metric", [L2, IP, COSINE], ids=["L2", "IP", "cos"])
def test_extreme_radii_ivf_pq(metric, nbits):
    """IVF-PQ (thresholded LUT scan), plain and sharded at world 1, every list probed: all rows or none, by the rule;
    nothing for a NaN radius."""
    require_gpu()
    from test_gpu_shard_range import NLIST as PQ_NLIST, _ivf_pq, _rows
    n = 3000
    ix = _ivf_pq(metric, nbits, n=n)
    ix.coalescing(0)
    sh = b200vs.Shard(ix, 0, 1, None)
    xq = _rows(24, 31)
    for name, radius in RADII.items():
        for nq in (24, 5):
            D, I, C = ix.range_search(xq[:nq], radius, 4096, nprobe=PQ_NLIST)
            if every_row_passes(metric, radius):
                assert (C == n).all() and all(np.array_equal(np.sort(I[q, :n]), np.arange(1, n + 1)) for q in range(nq)), name
            else:
                assert (C == 0).all() and (I == -1).all() and (D == 0).all(), f"{name}: hits"
            same(sh.range_search(xq[:nq], radius, 4096, nprobe=PQ_NLIST), (D, I, C))
    sh.close()


@gpu
def test_nan_inner_products_are_never_hits(oracle):
    """The "inf" overflow rung on mixed-sign data: inner products overflow to +-inf and their sums to NaN.  A NaN value
    passes no range test, so IP range search (Flat tile and exact scans, the streaming scan) returns only the +inf rows."""
    require_gpu()
    from test_gpu_fp32_range import D as RD, N as RN, NQ as RNQ, dataset
    _, xb, xq = dataset("inf", "n", RN, RNQ, RD, seed=909)
    ids = np.arange(1, RN + 1, dtype=np.int64)
    c = Built(oracle, FLAT, IP, xb, ids)
    with np.errstate(all="ignore"):
        raw = np.stack([raw_fp32(c.X, q, IP) for q in xq])
    assert np.isnan(raw).any(axis=1).all(), "premise: every query has NaN inner products"
    pos = {int(i): r for r, i in enumerate(c.ids.tolist())}
    for radius in (0.5, FLT_MAX, float("inf")):
        D, I, C = c.ix.range_search(xq, radius, 4096)
        same(c.ix.range_search(xq, radius, 4096, exact_only=True), (D, I, C))
        with np.errstate(all="ignore"):
            c.expect(D, I, C, xq, radius, 4096, range(RNQ))
        for qi in range(RNQ):
            r = [pos[int(i)] for i in I[qi, :C[qi]]]
            assert not np.isnan(raw[qi, r]).any(), f"query {qi}: a NaN inner product came back as a hit"
        rs = b200vs.BruteForceRangeScan(IP, RD, xq, radius, max_results=4096)
        rs.push(xb, ids)
        Ds, Is, Cs = rs.finish()
        assert np.array_equal(Cs, C), "streaming range scan counts"
        for qi in range(RNQ):
            assert sorted(Is[qi, :Cs[qi]].tolist()) == sorted(I[qi, :C[qi]].tolist())
