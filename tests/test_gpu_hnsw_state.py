"""HNSW graph layout: the levels the concurrent host writers draw, and the validation of the state blob (DESIGN §5).

Every add lays out all of its nodes before the first insertion, node c with the level generator's c-th draw, so any
number of writers, the single writer and the batched device build draw the same levels for the same node slots.  A
state blob enters from outside (set_trained_state, a saved file, a shard snapshot): one whose graph the host builder or
the device walk could not traverse within its arrays is refused before the index changes."""
import numpy as np
import pytest

import b200vs
import oracle_lib
from b200vs import HNSW, L2
from gpu_util import require_gpu

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _gpu():
    require_gpu()


def sections(blob):
    """A writable copy of an HNSW state blob and views of its sections: hdr, levels, up_off, link0 [n, maxM0 + 1], linkup,
    the offset where the labels end, and the trailing tombstones (None when absent)."""
    b = np.array(blob, dtype=np.uint8, copy=True)
    hdr = b[:64].view(np.int64)
    n, d, maxM0 = int(hdr[1]), int(hdr[2]), int(hdr[4])
    pad8 = lambda v: (v + 7) // 8 * 8
    p = pad8(64 + 4 * n)
    up_off = b[p:p + 8 * (n + 1)].view(np.int64)
    p += 8 * (n + 1)
    link0 = b[p:p + 4 * n * (maxM0 + 1)].view(np.uint32).reshape(n, maxM0 + 1)
    p += 4 * n * (maxM0 + 1)
    linkup = b[p:p + 4 * int(up_off[n])].view(np.uint32)
    end = pad8(pad8(p + 4 * int(up_off[n])) + 4 * n * d) + 8 * n
    tomb = b[end:end + n] if b.size >= end + n else None
    return dict(b=b, hdr=hdr, n=n, levels=b[64:64 + 4 * n].view(np.int32), up_off=up_off, link0=link0, linkup=linkup,
                end=end, tomb=tomb)


def levels_of(ix):
    s = sections(ix.get_trained_state())
    return s["levels"].copy(), int(s["hdr"][5]), int(s["levels"][int(s["hdr"][6])])


def test_concurrent_writers_draw_the_single_writer_levels():
    """16 writers over several adds: the levels array, the max level and the entry point's level equal a single-writer build
    of the same rows; so do the levels of the one-row (single-writer) adds and the batched add that follow."""
    rng = np.random.default_rng(21)
    n, d, M = 6000, 16, 4
    xb = rng.random((n + 240, d)).astype(np.float32)
    labels = np.arange(1, n + 241, dtype=np.int64)
    one = b200vs.Index(HNSW, L2, d, hnsw_m=M, hnsw_efc=40, max_elements=2 * n)
    many = b200vs.Index(HNSW, L2, d, hnsw_m=M, hnsw_efc=40, max_elements=2 * n, hnsw_build_threads=16)
    for a in range(0, n, 1500):
        one.add(xb[a:a + 1500], labels[a:a + 1500])
        many.add(xb[a:a + 1500], labels[a:a + 1500])
    lev1, top1, ep1 = levels_of(one)
    levm, topm, epm = levels_of(many)
    assert top1 >= 2, "too few levels to pin anything"
    assert np.array_equal(lev1, levm) and top1 == topm and ep1 == top1 and epm == topm
    for i in range(n, n + 40):  # one row per call: the single writer on both indexes
        one.add(xb[i:i + 1], labels[i:i + 1])
        many.add(xb[i:i + 1], labels[i:i + 1])
    one.add_batched(xb[n + 40:], labels[n + 40:])
    many.add_batched(xb[n + 40:], labels[n + 40:])
    lev1, top1, ep1 = levels_of(one)
    levm, topm, epm = levels_of(many)
    assert lev1.size == n + 240
    assert np.array_equal(lev1, levm) and top1 == topm and ep1 == top1 and epm == topm


def corrupt(s, what):
    """Apply one corruption to the sections s (in place) and return the blob."""
    b, hdr, n, levels, up_off, link0 = s["b"], s["hdr"], s["n"], s["levels"], s["up_off"], s["link0"]
    maxM0 = int(hdr[4])
    maxM = maxM0 // 2
    ep, maxlevel = int(hdr[6]), int(hdr[5])
    low = next(i for i in range(n) if levels[i] == 0 and i != ep)  # a node on level 0 only
    linked0 = next(i for i in range(n) if link0[i, 0] > 0)
    up = next(i for i in range(n) if levels[i] >= 1 and s["linkup"][up_off[i]] > 0)  # a node with a level-1 link
    up1 = s["linkup"][int(up_off[up]):int(up_off[up]) + maxM + 1]  # its level-1 list
    if what == "maxM0":
        hdr[4] += 1
    elif what == "up_off[0]":
        up_off[0] = 1
    elif what == "up_off step":
        up_off[n // 2] += 1
    elif what == "up_off not monotone":
        up_off[n // 2] = up_off[n] + 100
    elif what == "level below 0":
        levels[low] = -1
    elif what == "level above maxlevel":
        levels[low] = maxlevel + 1
    elif what == "level-0 count":
        link0[linked0, 0] = maxM0 + 1
    elif what == "upper count":
        up1[0] = maxM + 1
    elif what == "level-0 target":
        link0[linked0, 1] = n
    elif what == "upper target":
        up1[1] = 0xFFFFFFFF
    elif what == "upper target below its level":
        up1[1] = low
    elif what == "entry point":
        hdr[6] = n
    elif what == "entry point below maxlevel":
        hdr[6] = low
    elif what == "maxlevel":
        hdr[5] = maxlevel + 1
    elif what == "tombstone":
        if s["tomb"] is None:
            t = np.zeros(n, np.uint8)
            t[low] = 2
            return np.concatenate([b, t])
        s["tomb"][low] = 2
    elif what == "truncated":
        return b[:s["end"] - 1]
    else:
        raise AssertionError(what)
    return b


CORRUPTIONS = ["maxM0", "up_off[0]", "up_off step", "up_off not monotone", "level below 0", "level above maxlevel", "level-0 count",
               "upper count", "level-0 target", "upper target", "upper target below its level", "entry point",
               "entry point below maxlevel", "maxlevel", "tombstone", "truncated"]


@pytest.fixture(scope="module")
def valid_blobs(oracle):
    """(engine blob with tombstones, oracle blob, empty blob) of one geometry: d = 8, M = 4, efConstruction 30."""
    rng = np.random.default_rng(5)
    d, M, efc, n = 8, 4, 30, 400
    ix = b200vs.Index(HNSW, L2, d, hnsw_m=M, hnsw_efc=efc, max_elements=n)
    ix.add(rng.random((n, d)).astype(np.float32), np.arange(n, dtype=np.int64))
    ix.delete(np.arange(0, n, 7, dtype=np.int64))
    h = oracle_lib.OracleHnsw(oracle, L2, d, n, M, efc)
    h.add(rng.random((n, d)).astype(np.float32), np.arange(1000, 1000 + n, dtype=np.int64))
    empty = b200vs.Index(HNSW, L2, d, hnsw_m=M, hnsw_efc=efc).get_trained_state()
    return dict(geometry=(d, M, efc), engine=ix.get_trained_state(), oracle=h.export(), empty=empty)


def target(valid_blobs):
    d, M, efc = valid_blobs["geometry"]
    tgt = b200vs.Index(HNSW, L2, d, hnsw_m=M, hnsw_efc=efc)
    tgt.set_trained_state(valid_blobs["engine"])
    return tgt


def refused(tgt, blob):
    before = tgt.get_trained_state()
    with pytest.raises(b200vs.B200VSError) as e:
        tgt.set_trained_state(blob)
    assert e.value.code == b200vs.EILLEGAL_PARAMETERS and "bad HNSW state blob" in str(e.value)
    assert np.array_equal(tgt.get_trained_state(), before), "a refused blob changed the index"


@pytest.mark.parametrize("what", CORRUPTIONS)
def test_corrupt_blob_is_refused(valid_blobs, what):
    tgt = target(valid_blobs)
    for base in ("engine", "oracle"):
        s = sections(valid_blobs[base])
        assert s["hdr"][5] >= 1, "the blob needs upper levels"
        refused(tgt, corrupt(s, what))


@pytest.mark.parametrize("field,value", [(5, 0), (6, 0)])
def test_empty_graph_with_an_entry_point_is_refused(valid_blobs, field, value):
    """An empty graph is maxlevel -1 and entry point 0xFFFFFFFF, as both writers emit it."""
    s = sections(valid_blobs["empty"])
    assert s["n"] == 0 and s["hdr"][5] == -1 and s["hdr"][6] == 0xFFFFFFFF
    s["hdr"][field] = value
    refused(target(valid_blobs), s["b"])


def test_valid_blobs_are_accepted(valid_blobs):
    tgt = target(valid_blobs)
    for base in ("oracle", "empty", "engine"):
        tgt.set_trained_state(valid_blobs[base])
        assert np.array_equal(tgt.get_trained_state(), valid_blobs[base]), base
