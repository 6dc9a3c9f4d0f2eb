"""The tile kernel's passes must agree score for score wherever their work overlaps.

* The threshold sample pass runs its own configuration of tc_scan_kernel (one consumer warpgroup, a 3-stage ring of
  32-row boxes, several CTAs per SM).  The capture threshold's argument (DESIGN.md 4.2: A_k <= tau because the sample is
  a subset of the captured scores) needs each sampled score to be bit for bit the score the capture-shaped kernel
  computes for that (row, query).  b200vs_debug_tc_scores with split = 3 / 4 returns the sample configuration's scores,
  split = 0 / 2 the capture-shaped kernel's dense scores, in the TF32 and FP16 arithmetic.
* The coarse pass picks its query-group width (the wgmma N) from the batch size, so the same centroid scores must come
  out of one large call and of many small ones."""
import numpy as np
import pytest

import b200vs
from b200vs import FLAT, IP, L2
from gpu_util import require_gpu

pytestmark = pytest.mark.gpu

SPAN, SAMPLE = 2048, 32  # TC_SPAN, TC_SAMPLE: the first 32 rows of every 2048-row span are sampled


@pytest.fixture(autouse=True)
def _gpu():
    require_gpu()


def sampled_rows(n):
    return np.array([r for s in range(0, n, SPAN) for r in range(s, min(s + SAMPLE, n))], np.int64)


@pytest.mark.parametrize("half", [False, True], ids=["tf32", "fp16"])
@pytest.mark.parametrize("metric", [L2, IP], ids=["L2", "IP"])
@pytest.mark.parametrize("n", [31, 32, 33, 2047, 2048, 2049, 4097])
def test_sample_scores_equal_capture_scores(n, metric, half):
    d = 96  # TF32: 3 K blocks; FP16: 2 K blocks, the second half past the row end
    rng = np.random.default_rng(1000 * n + 10 * metric + half)
    xb = rng.standard_normal((n, d)).astype(np.float32)
    ix = b200vs.Index(FLAT, metric, d)
    ix.add(xb, np.arange(n, dtype=np.int64))
    ix.delete(np.arange(3, n, 11))  # tombstoned rows: +inf in both passes
    rows = sampled_rows(n)
    # query groups of 5 / 20 / 40 / 150 queries: B tiles of N = 16 / 32 / 64 / 128 + 32
    for nq in (5, 20, 40, 150):
        xq = rng.standard_normal((nq, d)).astype(np.float32)
        S, Es = ix.tc_scores(xq, half=half, sample=True)
        D, Ed = ix.tc_scores(xq, half=half)
        assert np.array_equal(Es, Ed)
        assert np.all(np.isnan(np.delete(S, rows, axis=1))), "a row outside the sample was written"
        got, want = S[:, rows], D[:, rows]
        assert np.isfinite(want).any() and not np.isnan(want).any()
        bad = np.argwhere(got.view(np.uint32) != want.view(np.uint32))
        assert bad.size == 0, (f"n={n} nq={nq}: sample score differs at (q, sampled row) {bad[0].tolist()}: "
                               f"{got[tuple(bad[0])]!r} vs capture-shaped {want[tuple(bad[0])]!r}")
    ix.close()


def test_sample_scores_argument_checks():
    L = b200vs.lib()
    ix = b200vs.Index(FLAT, L2, 36)
    ix.add(np.ones((4, 36), np.float32), np.arange(4, dtype=np.int64))
    q = np.zeros((16, 36), np.float32)
    out = np.zeros((16, 4), np.float32)
    eps = np.zeros(16, np.float32)
    assert L.b200vs_debug_tc_scores(ix.h, 16, q.ctypes.data, 3, out.ctypes.data, eps.ctypes.data) == b200vs.OK
    for split in (-1, 5, 100):
        assert L.b200vs_debug_tc_scores(ix.h, 16, q.ctypes.data, split, out.ctypes.data, eps.ctypes.data) == b200vs.EILLEGAL_PARAMETERS
    assert L.b200vs_debug_tc_scores(ix.h, 16, q.ctypes.data, 4, out.ctypes.data, eps.ctypes.data) == b200vs.EILLEGAL_PARAMETERS  # dim % 8
    with pytest.raises(ValueError):
        ix.tc_scores(q, split=True, sample=True)
    ix.close()


@pytest.mark.parametrize("metric", [L2, IP], ids=["L2", "IP"])
@pytest.mark.parametrize("ncent", [1024, 4096])
def test_coarse_scores_do_not_depend_on_the_batch(ncent, metric):
    d, nq = 256, 1024
    rng = np.random.default_rng(ncent + metric)
    cent = rng.standard_normal((ncent, d)).astype(np.float32)
    xq = rng.standard_normal((nq, d)).astype(np.float32)
    ix = b200vs.Index(FLAT, metric, d)
    ix.add(cent, np.arange(ncent, dtype=np.int64))
    whole, eps = ix.tc_scores(xq, split=True)
    parts = [ix.tc_scores(xq[i:i + 16], split=True) for i in range(0, nq, 16)]
    assert np.all(np.isfinite(whole))
    assert np.array_equal(np.concatenate([p[1] for p in parts]), eps)
    split16 = np.concatenate([p[0] for p in parts])
    bad = np.argwhere(whole.view(np.uint32) != split16.view(np.uint32))
    assert bad.size == 0, f"ncent={ncent}: score at (q, centroid) {bad[0].tolist()} differs between one call and calls of 16"
    ix.close()
