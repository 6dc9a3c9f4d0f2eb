"""HNSW batched construction on the GPU (b200vs_hnsw_add_batched, DESIGN §4.4).

batch = 1 has no batch peers and at most one incoming link per target, so it must rebuild the host single-writer graph byte
for byte (and so the oracle's).  Larger batches give another graph, defined by the rule; it must be deterministic, a sound
HNSW graph with the host builder's levels and entry point, as good as the host graph, and searched exactly like the oracle
searches it once adopted."""

import json
import os
import sys

import numpy as np
import pytest

import b200vs
import oracle_lib
from b200vs import COSINE, FLAT, HNSW, IP, L2
from gpu_util import assert_same_results, recall, require_gpu

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))

import make_hnsw_batched_golden as golden  # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _gpu():
    require_gpu()


def parse_blob(blob, M):
    """(hdr, levels, link lists per level) of the export layout (hnsw.cu HnswIndex::get_state)."""
    b = np.asarray(blob, dtype=np.uint8)
    hdr = b[:64].view(np.int64)
    n = int(hdr[1])
    maxM0 = int(hdr[4])
    p = 64
    levels = b[p:p + 4 * n].view(np.int32)
    p = (p + 4 * n + 7) // 8 * 8
    off = b[p:p + 8 * (n + 1)].view(np.int64)
    p += 8 * (n + 1)
    link0 = b[p:p + 4 * n * (maxM0 + 1)].view(np.uint32).reshape(n, maxM0 + 1)
    p += 4 * n * (maxM0 + 1)
    up = b[p:p + 4 * int(off[n])].view(np.uint32)
    lists = []
    for i in range(n):
        ls = [link0[i, 1:1 + link0[i, 0]]]
        for lv in range(1, int(levels[i]) + 1):
            o = int(off[i]) + (lv - 1) * (M + 1)
            ls.append(up[o + 1:o + 1 + up[o]])
        lists.append(ls)
    return hdr, levels, lists


def data(n, d, seed):
    rng = np.random.default_rng(seed)
    return rng.random((n, d)).astype(np.float32), np.arange(1000, 1000 + n, dtype=np.int64)


def build(metric, d, xb, labels, M, efc, batch=None, calls=3, max_elements=None):
    """batch None: the host builder (b200vs_add_with_ids, one writer); else add_batched(batch)."""
    n = len(labels)
    ix = b200vs.Index(HNSW, metric, d, hnsw_m=M, hnsw_efc=efc, max_elements=max_elements or n * 2)
    step = (n + calls - 1) // calls
    for a in range(0, n, step):
        if batch is None:
            ix.add(xb[a:a + step], labels[a:a + step])
        else:
            ix.add_batched(xb[a:a + step], labels[a:a + step], batch=batch)
    return ix


@pytest.mark.parametrize("metric", [L2, IP, COSINE])
@pytest.mark.parametrize("n,d,M", [(10, 16, 2), (3000, 32, 16), (2000, 128, 8), (1500, 100, 16)])
def test_batch1_equals_host_builder(oracle, metric, n, d, M):
    xb, labels = data(n, d, n + d)
    dev = build(metric, d, xb, labels, M, 200, batch=1)
    host = build(metric, d, xb, labels, M, 200)
    h = oracle_lib.OracleHnsw(oracle, metric, d, n, M, 200)
    h.add(xb, labels)
    blob = dev.get_trained_state()
    assert np.array_equal(blob, host.get_trained_state())
    assert np.array_equal(blob, h.export())
    xq = np.random.default_rng(7).random((20, d)).astype(np.float32)
    Dg, Ig = dev.search(xq, 10, efsearch=64)
    Do, Io, _, _ = h.search(xq, 10, ef=64, nthreads=8)
    assert_same_results(Dg, Ig, Do, Io)


@pytest.mark.parametrize("metric", [L2, COSINE])
def test_batch1_wide_lists_equal_host_builder(metric):
    """M = 40: level-0 lists of up to 80 links, walked 32 at a time and shrunk by the heuristic over 81 rows."""
    xb, labels = data(2500, 48, 40)
    dev = build(metric, 48, xb, labels, 40, 120, batch=1, calls=2)
    host = build(metric, 48, xb, labels, 40, 120, calls=2)
    blob = dev.get_trained_state()
    assert np.array_equal(blob, host.get_trained_state())
    _, _, lists = parse_blob(blob, 40)
    assert max(len(ls[0]) for ls in lists) > 32


def write_sequence(ix, xb, labels, batched, batch=1):
    """add / delete / upsert live and deleted labels / add with a repeated label; the blob after every step."""
    add = (lambda x, i: ix.add_batched(x, i, batch=batch)) if batched else (lambda x, i: ix.add(x, i))
    rng = np.random.default_rng(11)
    out = []
    add(xb[:1200], labels[:1200])
    out.append(ix.get_trained_state())
    ix.delete(labels[:1200:7])
    out.append(ix.get_trained_state())
    ups = labels[3:1200:5]  # some of them deleted above
    add(rng.random((len(ups), xb.shape[1])).astype(np.float32), ups)
    out.append(ix.get_trained_state())
    rep = np.concatenate([labels[1200:1400], labels[1250:1260], labels[10:12]])  # repeats inside the call, and an upsert
    add(xb[1200:1200 + len(rep)], rep)
    out.append(ix.get_trained_state())
    return out


@pytest.mark.parametrize("metric", [L2, COSINE])
def test_batch1_tombstones_and_upserts_equal_host_builder(metric):
    xb, labels = data(1500, 24, 5)
    host = b200vs.Index(HNSW, metric, 24, hnsw_m=12, hnsw_efc=80, max_elements=10000)
    dev = b200vs.Index(HNSW, metric, 24, hnsw_m=12, hnsw_efc=80, max_elements=10000)
    for step, (a, b) in enumerate(zip(write_sequence(host, xb, labels, False), write_sequence(dev, xb, labels, True))):
        assert np.array_equal(a, b), f"blob differs after step {step}"
    assert dev.get_count() == host.get_count() and dev.get_deleted_count() == host.get_deleted_count()


def test_repeated_label_default_batch_last_row_wins():
    rng = np.random.default_rng(3)
    n, d = 3000, 16
    xb = rng.random((n, d)).astype(np.float32)
    ids = np.arange(n, dtype=np.int64)
    ids[2000] = 77  # repeats of a label the index already holds, and of one first seen in this call
    ids[2500] = 77
    ids[2600] = 1500
    ix = b200vs.Index(HNSW, L2, d, hnsw_m=8, hnsw_efc=64, max_elements=10000)
    ix.add_batched(xb[:1000], np.arange(1000, dtype=np.int64) + 10000)
    ix.add_batched(xb, ids)
    live = n - 3
    assert ix.get_count() == 1000 + live and ix.get_deleted_count() == 3
    _, _, _, out_ids = ix.export_lists(1, with_vectors=False)
    assert (out_ids == 77).sum() == 1 and (out_ids == 1500).sum() == 1
    vec, found = ix.reconstruct(np.array([77, 1500], dtype=np.int64))
    assert found.all()
    assert np.array_equal(vec[0], xb[2500]) and np.array_equal(vec[1], xb[2600])


def test_deterministic():
    xb, labels = data(20000, 32, 9)
    for batch in (0, 257):
        a = build(L2, 32, xb, labels, 16, 100, batch=batch, calls=2).get_trained_state()
        b = build(L2, 32, xb, labels, 16, 100, batch=batch, calls=2).get_trained_state()
        assert np.array_equal(a, b), f"batch {batch}: two builds differ"


def test_batched_graphs_match_frozen_hashes():
    """Graphs of batch > 1 builds, in both construction-search forms, are those of tests/golden/hnsw_batched_graphs.json."""
    want = json.load(open(os.path.join(HERE, "golden", "hnsw_batched_graphs.json")))
    assert sorted(want) == sorted(golden.CASES)
    for name in sorted(want):
        assert golden.graph_hash(name) == want[name], f"graph of case {name} changed"


@pytest.mark.parametrize("metric", [L2, IP])
def test_batched_graph_invariants(metric):
    M = 12
    xb, labels = data(12000, 40, 21)
    dev = build(metric, 40, xb, labels, M, 100, batch=0)
    host = build(metric, 40, xb, labels, M, 100)
    hdr, levels, lists = parse_blob(dev.get_trained_state(), M)
    hhdr, hlevels, _ = parse_blob(host.get_trained_state(), M)
    assert np.array_equal(levels, hlevels)
    assert hdr[5] == hhdr[5] and hdr[6] == hhdr[6]  # max level, entry point
    assert hdr[1] == 12000
    for i, ls in enumerate(lists):
        for lv, l in enumerate(ls):
            assert len(l) <= (2 * M if lv == 0 else M)
            assert i not in set(l.tolist()) and len(set(l.tolist())) == len(l)
            if len(l):
                assert (levels[l] >= lv).all()


@pytest.mark.parametrize("metric", [L2, COSINE])
def test_quality_against_host_graph(oracle, metric):
    n, d, M, efc = 50000, 64, 16, 100
    xb, labels = data(n, d, 50)
    dev = build(metric, d, xb, labels, M, efc, batch=0, calls=1)
    host = build(metric, d, xb, labels, M, efc, calls=1)
    xq = np.random.default_rng(51).random((400, d)).astype(np.float32)
    om = oracle_lib.L2 if metric == L2 else oracle_lib.COSINE
    _, If = oracle.flat_search(om, xb, labels, xq, 10, nthreads=8)
    for ef in (64, 128):
        rd = recall(dev.search(xq, 10, efsearch=ef)[1], If)
        rh = recall(host.search(xq, 10, efsearch=ef)[1], If)
        assert rd >= rh - 0.01, (ef, rd, rh)
    sd = (dev.search(xb[:2000], 1, efsearch=64)[1][:, 0] == labels[:2000]).mean()
    sh = (host.search(xb[:2000], 1, efsearch=64)[1][:, 0] == labels[:2000]).mean()
    assert sd >= sh - 0.01, (sd, sh)


def test_device_built_graph_searched_exactly(oracle):
    n, d = 8000, 48
    xb, labels = data(n, d, 60)
    ix = build(COSINE, d, xb, labels, 16, 150, batch=0, calls=2)
    h = oracle_lib.OracleHnsw(oracle, COSINE, d, n, 16, 150)
    h.load(ix.get_trained_state())
    xq = np.random.default_rng(61).random((48, d)).astype(np.float32)
    for kw in (dict(), dict(id_range=(1500, 6000)), dict(sorted_ids=np.arange(1000, 9000, 5))):
        Dg, Ig = ix.search(xq, 10, efsearch=96, **kw)
        Do, Io, _, _ = h.search(xq, 10, ef=96, nthreads=8, **kw)
        assert_same_results(Dg, Ig, Do, Io)
    dead = labels[::4]
    ix.delete(dead)
    # a tombstone is traversed but never returned, with the strict stop rule: the oracle's negated id filter
    Dg, Ig = ix.search(xq, 10, efsearch=96)
    Do, Io, _, _ = h.search(xq, 10, ef=96, nthreads=8, sorted_ids=dead, negate=True)
    assert_same_results(Dg, Ig, Do, Io)
    assert not (set(Ig.ravel()) & set(labels[::4].tolist()))


def test_mixed_writes_save_load(oracle, tmp_path):
    d, M, efc = 32, 16, 100
    xb, labels = data(9000, d, 70)
    ix = b200vs.Index(HNSW, L2, d, hnsw_m=M, hnsw_efc=efc, max_elements=20000)
    twin = b200vs.Index(HNSW, L2, d, hnsw_m=M, hnsw_efc=efc, max_elements=20000)
    ix.add_batched(xb[:4000], labels[:4000])
    ix.add(xb[4000:5000], labels[4000:5000])
    ix.delete(labels[100:300])
    ix.add_batched(xb[5000:9000], labels[5000:9000], batch=300)
    twin.add(xb[:5000], labels[:5000])
    twin.delete(labels[100:300])
    twin.add(xb[5000:9000], labels[5000:9000])
    assert ix.get_count() == twin.get_count() == 8800 and ix.get_deleted_count() == twin.get_deleted_count() == 200
    q = labels[::37]
    v1, f1 = ix.reconstruct(q)
    v2, f2 = twin.reconstruct(q)
    assert np.array_equal(f1, f2) and np.array_equal(v1, v2)
    _, lv, _ = parse_blob(ix.get_trained_state(), M)
    _, lt, _ = parse_blob(twin.get_trained_state(), M)
    assert np.array_equal(lv, lt)
    path = str(tmp_path / "hnsw.idx")
    ix.save(path)
    back = b200vs.Index(HNSW, L2, d, hnsw_m=M, hnsw_efc=efc, max_elements=20000)
    back.load(path)
    assert np.array_equal(back.get_trained_state(), ix.get_trained_state())
    assert back.get_count() == 8800 and back.get_deleted_count() == 200
    h = oracle_lib.OracleHnsw(oracle, L2, d, 20000, M, efc)
    h.load(ix.get_trained_state())
    xq = np.random.default_rng(71).random((40, d)).astype(np.float32)
    Do, Io, _, _ = h.search(xq, 10, ef=80, nthreads=8, sorted_ids=labels[100:300], negate=True)  # the tombstones
    for idx in (ix, back):
        Dg, Ig = idx.search(xq, 10, efsearch=80)
        assert_same_results(Dg, Ig, Do, Io)


def test_refusals_leave_the_index_unchanged():
    d = 16
    xb, labels = data(600, d, 80)
    ix = b200vs.Index(HNSW, L2, d, hnsw_m=8, hnsw_efc=50, max_elements=1000)
    ix.add_batched(xb[:500], labels[:500])
    blob = ix.get_trained_state()

    def refused(code, x, ids, batch=0, index=ix):
        with pytest.raises(b200vs.B200VSError) as e:
            index.add_batched(x, ids, batch=batch)
        assert e.value.code == code
        assert np.array_equal(ix.get_trained_state(), blob)

    refused(b200vs.EILLEGAL_PARAMETERS, np.zeros((0, d), np.float32), np.zeros(0, np.int64))
    refused(b200vs.EINTERNAL, np.zeros((501, d), np.float32), np.arange(5000, 5501, dtype=np.int64))
    fl = b200vs.Index(FLAT, L2, d)
    refused(b200vs.EILLEGAL_PARAMETERS, xb[:5], labels[:5], index=fl)
    big = b200vs.Index(HNSW, L2, d, hnsw_m=8, hnsw_efc=20000, max_elements=1000)
    big.add(xb[:300], labels[:300])
    big_blob = big.get_trained_state()
    with pytest.raises(b200vs.B200VSError) as e:
        big.add_batched(xb[300:400], labels[300:400])
    assert e.value.code == b200vs.EILLEGAL_PARAMETERS
    assert np.array_equal(big.get_trained_state(), big_blob) and big.get_count() == 300


def test_efc_above_merged_array_limit_runs_heap_form():
    """efc + 1 > 1024 candidates: the construction search takes the candidate-heap form; batch 1 still equals the host."""
    xb, labels = data(1500, 8, 90)
    dev = build(L2, 8, xb, labels, 6, 1100, batch=1, calls=2)
    host = build(L2, 8, xb, labels, 6, 1100, calls=2)
    assert np.array_equal(dev.get_trained_state(), host.get_trained_state())


def test_failed_call_leaves_the_index_unchanged():
    """A call that runs out of device scratch (capped with the diagnostics limit, at every size from the first allocation to
    the peer matrix of a late batch) changes nothing: blob, counts, the level generator and the search all stay those of an
    index that never saw the call.  The mirror, whose link lists earlier batches already wrote, is rebuilt before the next
    search."""
    d, M, efc = 16, 8, 64
    xb, labels = data(2100, d, 95)
    ix = b200vs.Index(HNSW, L2, d, hnsw_m=M, hnsw_efc=efc, max_elements=10000)
    twin = b200vs.Index(HNSW, L2, d, hnsw_m=M, hnsw_efc=efc, max_elements=10000)
    for idx in (ix, twin):
        idx.add(xb[:100], labels[:100])
    blob = twin.get_trained_state()
    xq = np.random.default_rng(96).random((16, d)).astype(np.float32)
    Dt, It = twin.search(xq, 10, efsearch=64)
    limit, failures = 1024, 0
    while True:
        ix.set_build_scratch_limit(limit)
        try:
            ix.add_batched(xb[100:], labels[100:], batch=2048)
            break
        except b200vs.B200VSError as e:
            assert e.code == b200vs.EINTERNAL, e
            failures += 1
        assert np.array_equal(ix.get_trained_state(), blob), f"blob changed by a call that failed at limit {limit}"
        assert ix.get_count() == 100 and ix.get_deleted_count() == 0
        Dg, Ig = ix.search(xq, 10, efsearch=64)
        assert np.array_equal(Ig, It) and np.array_equal(Dg.view(np.uint32), Dt.view(np.uint32))
        limit = int(limit * 1.5)
    assert failures >= 10
    ref = b200vs.Index(HNSW, L2, d, hnsw_m=M, hnsw_efc=efc, max_elements=10000)
    ref.add(xb[:100], labels[:100])
    ref.add_batched(xb[100:], labels[100:], batch=2048)
    assert np.array_equal(ix.get_trained_state(), ref.get_trained_state())
    # an upsert that fails tombstones nothing
    ix.set_build_scratch_limit(1024)
    blob = ix.get_trained_state()
    with pytest.raises(b200vs.B200VSError) as e:
        ix.add_batched(xb[:50] + 1.0, labels[:50])
    assert e.value.code == b200vs.EINTERNAL
    assert np.array_equal(ix.get_trained_state(), blob) and ix.get_deleted_count() == 0
    vec, found = ix.reconstruct(labels[:50])
    assert found.all() and np.array_equal(vec, xb[:50])
    ix.set_build_scratch_limit(0)
    ix.add_batched(xb[:50] + 1.0, labels[:50])
    assert ix.get_deleted_count() == 50
