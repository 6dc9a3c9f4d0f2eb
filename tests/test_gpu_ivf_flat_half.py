"""The IVF-Flat list scan on the FP16 mirror of the arena: decoys built against the FP16 rounding, and the mirror kept in
step with the FP32 rows through every way the arena is written (adds that relocate a list, delete + compaction, upsert,
reserve_lists, save / load, extreme scales).  Every case compares the tile path with exact_only=True (ids and distance
bits); an index with dim % 8 != 0 keeps no mirror and scans in TF32."""
import os

import numpy as np
import pytest

import b200vs
import fp16_emu as H
from b200vs import IVF_FLAT, L2
from gpu_util import assert_same_results, require_gpu
from test_gpu_tc_adversarial import far_centroids, run_both

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _gpu():
    require_gpu()


def arena_bytes(ix, d, nlist, mirror):
    """get_memory_size() of an IVF-Flat index split into its arena rows: (FP32 rows + ids + norms) = 4d + 12 B per row,
    the FP16 mirror adds 2d + 4.  Returns the arena capacity in rows."""
    per_row = 4 * d + 12 + (2 * d + 4 if mirror else 0)
    rest = ix.get_memory_size() - nlist * d * 4
    assert rest % per_row == 0, f"memory size {ix.get_memory_size()} is not a whole number of {per_row}-byte rows"
    return rest // per_row


def clustered(rng, nlist, per, d, scale=1.0):
    cent = far_centroids(nlist, d, 1000.0 * scale)
    xb = (np.repeat(cent, per, axis=0) + scale * rng.standard_normal((nlist * per, d))).astype(np.float32)
    return cent, xb


@pytest.mark.parametrize("k", [1, 10])
def test_half_decoys(oracle, k):
    """32 queries, each with its own FP16 decoy pair (fp16_emu.decoy_l2, more than half of the 2 eps window): the tile
    path returns R as the k-th neighbour, matches exact_only and the oracle, and certifies the decoy query."""
    d, npair = 128, 32
    pairs = [H.decoy_l2(np.random.default_rng(2000 * k + p), d, k, nfill=1500) for p in range(npair)]
    xq = np.concatenate([p[1] for p in pairs])
    for p in range(0, npair, 4):
        rows, _, r, dd = pairs[p]
        assert H.decoy_margin(rows, pairs[p][1], r, dd) > 0.5
        ids = np.arange(rows.shape[0], dtype=np.int64) * 7 + 3
        cent = np.zeros((4, d), np.float32)
        cent[1:, d // 2:d // 2 + 3] = -1000 * np.eye(3, dtype=np.float32)
        ix = b200vs.Index(IVF_FLAT, L2, d, nlist=4)
        ix.set_trained_state(b200vs.ivf_state_blob(cent, L2))
        ix.add(rows, ids)
        assert arena_bytes(ix, d, 4, True) > 0
        D, I, st = run_both(ix, xq, k, nprobe=4)
        assert st[1] == npair, st
        assert I[p, k - 1] == ids[r], f"pair {p}: the decoy displaced R (got id {I[p, k - 1]}, R {ids[r]}, D {ids[dd]})"
        _, Ic, stc = run_both(ix, np.repeat(xq[p:p + 1], 16, axis=0), k, nprobe=4)
        assert stc[1] == 16 and stc[2] == 0, f"pair {p}: the decoy query fell back to the exact scan: stats {stc}"
        assert np.all(Ic[:, k - 1] == ids[r])
        off, lx, _, lids = ix.export_lists(4)
        Do, Io = oracle.ivfflat_search(L2, cent, off, lx, lids, xq, k, 4, nthreads=8)
        assert_same_results(D, I, Do, Io)
        ix.close()


def test_mirror_follows_relocating_adds_delete_compaction_and_upsert():
    rng = np.random.default_rng(21)
    d, nlist, per = 64, 16, 300
    cent, xb = clustered(rng, nlist, per, d)
    ids = np.arange(xb.shape[0], dtype=np.int64) + 100
    ix = b200vs.Index(IVF_FLAT, L2, d, nlist=nlist)
    ix.set_trained_state(b200vs.ivf_state_blob(cent, L2))
    xq = (cent[rng.integers(0, nlist, 64)] + rng.standard_normal((64, d))).astype(np.float32)
    kw = dict(nprobe=4)
    for a in range(0, xb.shape[0], 700):  # small batches: every list outgrows its slot and is relocated several times
        ix.add(xb[a:a + 700], ids[a:a + 700])
        run_both(ix, xq, 10, **kw)
    assert arena_bytes(ix, d, nlist, True) > 0
    ix.delete(ids[: int(0.7 * ids.size)])  # more than half dead: compaction
    _, I, st = run_both(ix, xq, 10, **kw)
    assert st[1] == 64 and np.all(I[I >= 0] >= ids[int(0.7 * ids.size)])
    new = (xb[-500:] + 0.25).astype(np.float32)
    ix.upsert(new, ids[-500:])
    D, I, _ = run_both(ix, new[:64], 1, **kw)
    assert np.array_equal(I[:, 0], ids[-500:][:64]) and np.all(D == 0)


def test_reserved_arena_holds_the_mirror():
    """reserve_lists allocates the mirror with the arena: get_memory_size() is the FP32 arena plus the mirror right after
    the reservation and stays put while the rows arrive."""
    rng = np.random.default_rng(22)
    d, nlist, per = 64, 16, 500
    cent, xb = clustered(rng, nlist, per, d)
    ids = np.arange(xb.shape[0], dtype=np.int64)
    ix = b200vs.Index(IVF_FLAT, L2, d, nlist=nlist)
    ix.set_trained_state(b200vs.ivf_state_blob(cent, L2))
    ix.reserve_lists(np.full(nlist, per))
    mem0 = ix.get_memory_size()
    cap = arena_bytes(ix, d, nlist, True)
    assert cap >= nlist * per
    for a in range(0, xb.shape[0], 1500):
        ix.add(xb[a:a + 1500], ids[a:a + 1500])
    assert ix.get_memory_size() == mem0
    xq = (cent[rng.integers(0, nlist, 64)] + rng.standard_normal((64, d))).astype(np.float32)
    run_both(ix, xq, 10, nprobe=4)


def test_save_load_rebuilds_the_mirror(tmp_path):
    rng = np.random.default_rng(23)
    d, nlist = 96, 8
    cent, xb = clustered(rng, nlist, 400, d)
    ids = np.arange(xb.shape[0], dtype=np.int64) * 5
    a = b200vs.Index(IVF_FLAT, L2, d, nlist=nlist)
    a.set_trained_state(b200vs.ivf_state_blob(cent, L2))
    a.add(xb, ids)
    a.delete(ids[::7])
    xq = (cent[rng.integers(0, nlist, 48)] + rng.standard_normal((48, d))).astype(np.float32)
    Da, Ia, _ = run_both(a, xq, 10, nprobe=3)
    path = os.path.join(tmp_path, "idx.b2vs")
    a.save(path)
    b = b200vs.Index(IVF_FLAT, L2, d, nlist=nlist)
    b.load(path)
    assert arena_bytes(b, d, nlist, True) > 0
    Db, Ib, st = run_both(b, xq, 10, nprobe=3)
    assert st[1] == 48
    assert_same_results(Da, Ia, Db, Ib)


@pytest.mark.parametrize("e", [-40, 40])
def test_extreme_scales(e):
    """Data scaled by 2^+-40: the power-of-two scales keep the FP16 operands in range, so the scores (and the results)
    are those of the unscaled data scaled by 2^(2e)."""
    rng = np.random.default_rng(24)
    d, nlist = 128, 8
    cent, xb = clustered(rng, nlist, 500, d)
    xq = (cent[rng.integers(0, nlist, 32)] + rng.standard_normal((32, d))).astype(np.float32)
    f = np.float32(2.0 ** e)
    ids = np.arange(xb.shape[0], dtype=np.int64)
    out = []
    for s in (np.float32(1), f):
        ix = b200vs.Index(IVF_FLAT, L2, d, nlist=nlist)
        ix.set_trained_state(b200vs.ivf_state_blob(cent * s, L2))
        ix.add(xb * s, ids)
        D, I, st = run_both(ix, xq * s, 10, nprobe=3)
        assert st[1] == 32
        out.append((D, I))
        ix.close()
    assert np.array_equal(out[0][1], out[1][1])
    assert np.array_equal(out[0][0] * f * f, out[1][0])


def test_dim_not_multiple_of_8_keeps_tf32():
    rng = np.random.default_rng(25)
    d, nlist = 36, 8
    cent, xb = clustered(rng, nlist, 400, d)
    ix = b200vs.Index(IVF_FLAT, L2, d, nlist=nlist)
    ix.set_trained_state(b200vs.ivf_state_blob(cent, L2))
    ix.add(xb, np.arange(xb.shape[0], dtype=np.int64))
    assert arena_bytes(ix, d, nlist, False) > 0
    xq = (cent[rng.integers(0, nlist, 32)] + rng.standard_normal((32, d))).astype(np.float32)
    _, _, st = run_both(ix, xq, 10, nprobe=3)
    assert st[1] == 32
