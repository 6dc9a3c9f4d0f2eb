"""Fork-based snapshots (b200vs_save_stage / b200vs_save_staged / b200vs_save_unstage): the staged file equals b200vs_save's
file at the moment of the stage, byte for byte, whatever is written to the index afterwards; a forked child writes it without
CUDA and without the library's locks, even while another parent thread holds the index's reader lock and a lane; and it
loads into an index that searches exactly like the staged one did."""
import os
import signal
import threading
import time
import warnings

import numpy as np
import pytest

import b200vs
from b200vs import BINARY_FLAT, BINARY_IVF_FLAT, COSINE, FLAT, HAMMING, HNSW, IP, IVF_FLAT, IVF_PQ, L2
from gpu_util import require_gpu

pytestmark = pytest.mark.gpu

CHILD_TIMEOUT_S = 120

# (name, type, metric, dim, rows, creation keywords).  The row formats cover every width of the pack kernel: FP32 rows of 48
# and 33 floats, PQ code rows of 8, 4 and 3 bytes (nbits 8, 4, 3), packed binary rows of 9, 16 and 32 bytes.
CASES = [
    ("flat_l2", FLAT, L2, 48, 3000, {}),
    ("flat_ip_d33", FLAT, IP, 33, 3000, {}),
    ("flat_cosine", FLAT, COSINE, 48, 3000, {}),
    ("ivf_flat_l2", IVF_FLAT, L2, 48, 6000, dict(nlist=16)),
    ("ivf_flat_ip", IVF_FLAT, IP, 48, 6000, dict(nlist=16)),
    ("ivf_flat_cosine", IVF_FLAT, COSINE, 48, 6000, dict(nlist=16)),
    ("ivf_pq_inner_flat", IVF_PQ, L2, 32, 2000, dict(nlist=16, pq_m=8, pq_nbits=8)),
    ("ivf_pq_inner_flat_cosine", IVF_PQ, COSINE, 32, 2000, dict(nlist=16, pq_m=8, pq_nbits=8)),
    ("ivf_pq_nbits8", IVF_PQ, L2, 16, 66000, dict(nlist=16, pq_m=8, pq_nbits=8)),
    ("ivf_pq_nbits4_ip", IVF_PQ, IP, 32, 6000, dict(nlist=16, pq_m=8, pq_nbits=4)),
    ("ivf_pq_nbits3", IVF_PQ, L2, 32, 6000, dict(nlist=16, pq_m=8, pq_nbits=3)),
    ("hnsw_l2", HNSW, L2, 32, 3000, dict(hnsw_m=16, hnsw_efc=100, max_elements=10000)),
    ("hnsw_ip", HNSW, IP, 32, 3000, dict(hnsw_m=16, hnsw_efc=100, max_elements=10000)),
    ("hnsw_cosine", HNSW, COSINE, 32, 3000, dict(hnsw_m=16, hnsw_efc=100, max_elements=10000)),
    ("binary_flat_72", BINARY_FLAT, HAMMING, 72, 3000, {}),
    ("binary_flat_256", BINARY_FLAT, HAMMING, 256, 3000, {}),
    ("binary_ivf_flat_128", BINARY_IVF_FLAT, HAMMING, 128, 6000, dict(nlist=16)),
]


def rows(kind, dim, n, rng):
    if kind in b200vs.BINARY_TYPES:
        return rng.integers(0, 256, (n, dim // 8), dtype=np.uint8)
    return (rng.random((n, dim), dtype=np.float32) - 0.5).astype(np.float32)


def build(case, seed=0):
    """An index of the case with tombstoned rows, its queries and its rng."""
    name, kind, metric, dim, n, kw = case
    rng = np.random.default_rng(seed + sum(map(ord, name)))
    ix = b200vs.Index(kind, metric, dim, **kw)
    x = rows(kind, dim, n, rng)
    ids = np.arange(1, n + 1, dtype=np.int64) * 3
    if kind in (IVF_FLAT, IVF_PQ, BINARY_IVF_FLAT):
        ix.train(x)
    ix.add(x, ids)
    ix.delete(ids[::5])
    return ix, rows(kind, dim, 20, rng), rng, ids


def search(ix, xq):
    return ix.search(xq, 10, nprobe=8, efsearch=64)


def same_search(a, b):
    (Da, Ia), (Db, Ib) = a, b
    return np.array_equal(Ia, Ib) and np.array_equal(Da.view(np.uint32), Db.view(np.uint32))


def file_bytes(path):
    with open(path, "rb") as f:
        return f.read()


def reap(pid):
    """waitpid with a timeout: a child still running at the timeout is killed and reaped, and the test fails."""
    deadline = time.monotonic() + CHILD_TIMEOUT_S
    while time.monotonic() < deadline:
        got, status = os.waitpid(pid, os.WNOHANG)
        if got == pid:
            return os.waitstatus_to_exitcode(status)
        time.sleep(0.005)
    os.kill(pid, signal.SIGKILL)
    os.waitpid(pid, 0)
    pytest.fail(f"the child's staged write did not finish within {CHILD_TIMEOUT_S} s")


def fork_staged_write(ix, path, parent_work=None):
    """Fork; the child calls only save_staged and _exits with its status (0 = written).  The parent runs parent_work while the
    child runs, and always reaps the child."""
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", DeprecationWarning)  # fork() of a multi-threaded process: what the snapshot path does
        pid = os.fork()
    if pid == 0:
        code = 1
        try:
            ix.save_staged(path)
            code = 0
        finally:
            os._exit(code)
    try:
        if parent_work:
            parent_work()
    finally:
        status = reap(pid)
    return status


def mutate(case, ix, rng, ids, base):
    """Adds (new ids from base), upserts and deletes (of live ids in ids) after the stage."""
    _, kind, _, dim, n, _ = case
    ix.add(rows(kind, dim, 300, rng), np.arange(base, base + 300, dtype=np.int64))
    live = ids[1::5][:50]
    ix.upsert(rows(kind, dim, live.size, rng), live)
    ix.delete(ids[2::5][:80])


def loaded(case, path):
    _, kind, metric, dim, _, kw = case
    ix = b200vs.Index(kind, metric, dim, **kw)
    ix.load(path)
    return ix


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_fork_staged_write_equals_save_at_stage(tmp_path, case):
    require_gpu()
    ix, xq, rng, ids = build(case)
    before = search(ix, xq)
    ref = str(tmp_path / "ref.b2vs")
    ix.save(ref)
    ix.save_stage()
    mutate(case, ix, rng, ids, 10**7)  # writes after the stage reach neither the image nor the child's file
    in_proc = str(tmp_path / "in_proc.b2vs")
    ix.save_staged(in_proc)
    child = str(tmp_path / "child.b2vs")
    assert fork_staged_write(ix, child, parent_work=lambda: mutate(case, ix, rng, ids[3::5], 2 * 10**7)) == 0
    ix.save_unstage()
    want = file_bytes(ref)
    assert file_bytes(in_proc) == want
    assert file_bytes(child) == want
    back, from_ref = loaded(case, child), loaded(case, ref)
    assert same_search(search(back, xq), before)
    assert back.get_count() == from_ref.get_count()
    assert back.get_deleted_count() == from_ref.get_deleted_count()
    assert back.sub_type() == from_ref.sub_type()


@pytest.mark.parametrize("kind", [IVF_FLAT, BINARY_IVF_FLAT, FLAT])
def test_staged_write_after_compaction(tmp_path, kind):
    """A freshly compacted index (IVF: the arena rebuilt list by list; Flat: rows moved down), then new tombstones."""
    require_gpu()
    dim = 128 if kind == BINARY_IVF_FLAT else 32
    case = ("compacted", kind, HAMMING if kind in b200vs.BINARY_TYPES else L2, dim, 12000, dict(nlist=32) if kind != FLAT else {})
    ix, xq, rng, ids = build(case)
    live = ids[np.arange(ids.size) % 5 != 0]
    ix.delete(live[:8000])  # dead rows outweigh live ones: compacted
    assert ix.get_deleted_count() == 0
    for path_name in ("clean", "tombstoned"):
        if path_name == "tombstoned":
            ix.delete(live[8000:8100])
        ref, staged = str(tmp_path / f"{path_name}.ref"), str(tmp_path / f"{path_name}.staged")
        ix.save(ref)
        ix.save_stage()
        ix.save_staged(staged)
        ix.save_unstage()
        assert file_bytes(staged) == file_bytes(ref)
    assert ix.get_deleted_count() == 100


@pytest.mark.parametrize("case", [c for c in CASES if c[0] in ("flat_l2", "ivf_flat_l2", "ivf_pq_nbits4_ip", "hnsw_l2",
                                                                "binary_ivf_flat_128")], ids=lambda c: c[0])
def test_empty_and_untrained_indexes_stage_save_bytes(tmp_path, case):
    require_gpu()
    _, kind, metric, dim, _, kw = case
    ix = b200vs.Index(kind, metric, dim, **kw)
    ref, staged = str(tmp_path / "ref"), str(tmp_path / "staged")
    ix.save(ref)
    ix.save_stage()
    ix.save_staged(staged)
    assert file_bytes(staged) == file_bytes(ref)


def test_fork_while_another_thread_holds_the_reader_lock_and_a_lane(tmp_path):
    """One thread searches back to back, so at the fork it most likely holds the index's reader lock and a lane; the child's
    staged write takes neither and still completes."""
    require_gpu()
    case = CASES[3]  # ivf_flat_l2
    ix, xq, _, _ = build(case)
    ref = str(tmp_path / "ref.b2vs")
    ix.save(ref)
    ix.save_stage()
    stop = threading.Event()
    searches = [0]

    def reader():
        while not stop.is_set():
            ix.search(xq[:1], 10, nprobe=8)
            searches[0] += 1

    t = threading.Thread(target=reader)
    t.start()
    try:
        while searches[0] < 20:
            time.sleep(0.001)
        for i in range(3):
            path = str(tmp_path / f"child{i}.b2vs")
            assert fork_staged_write(ix, path) == 0
            assert file_bytes(path) == file_bytes(ref)
    finally:
        stop.set()
        t.join()
    ix.save_unstage()


def test_refusals_and_image_lifetime(tmp_path):
    require_gpu()
    case = CASES[3]  # ivf_flat_l2
    ix, _, rng, _ = build(case)
    good = str(tmp_path / "good.b2vs")
    with pytest.raises(b200vs.B200VSError) as e:
        ix.save_staged(good)  # no image
    assert e.value.code == b200vs.EILLEGAL_PARAMETERS
    ix.save_unstage()  # no image: a no-op
    ref1 = str(tmp_path / "ref1")
    ix.save(ref1)
    ix.save_stage()
    with pytest.raises(b200vs.B200VSError) as e:
        ix.save_staged("")
    assert e.value.code == b200vs.EILLEGAL_PARAMETERS
    with pytest.raises(b200vs.B200VSError) as e:
        ix.save_staged(str(tmp_path / "missing_dir" / "x.b2vs"))  # unwritable
    assert e.value.code == b200vs.EINTERNAL and "missing_dir" in e.value.msg
    ix.save_staged(good)  # the image was kept: the retry writes it
    assert file_bytes(good) == file_bytes(ref1)
    # a second stage replaces the first
    ix.add(rows(IVF_FLAT, case[3], 100, rng), np.arange(10**8, 10**8 + 100, dtype=np.int64))
    ref2 = str(tmp_path / "ref2")
    ix.save(ref2)
    ix.save_stage()
    ix.save_staged(good)
    assert file_bytes(good) == file_bytes(ref2) != file_bytes(ref1)
    ix.save_unstage()
    ix.save_unstage()
    with pytest.raises(b200vs.B200VSError) as e:
        ix.save_staged(good)  # unstaged
    assert e.value.code == b200vs.EILLEGAL_PARAMETERS
    ix.save_stage()
    ix.close()  # b200vs_destroy frees a held image
