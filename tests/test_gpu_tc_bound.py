"""The premise of the tile path's exactness proof (DESIGN.md 4.2), measured on the hardware: for every query q and row x

    |approx - s64| + |exact32 - e64| <= eps(q)

approx = the tile kernel's score (b200vs_debug_tc_scores runs the production tc_scan_kernel in dense mode), s64 / e64 =
float64 score / distance of the FP32 operands, exact32 = the engine's exact reference-order distance (the oracle's
primitives return the same bits), eps(q) = the device's tc_eps().  Both the list-scan arithmetic (single pass) and the
coarse quantiser's hi / lo arithmetic (split) are checked.  The coherent family also sets a tightness floor, so the test
fails against an eps much looser than the one the kernels claim."""
import numpy as np
import pytest

import b200vs
import tf32_emu as E
from b200vs import COSINE, FLAT, IP, L2
from gpu_util import require_gpu

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _gpu():
    require_gpu()


METRICS = {L2: "L2", IP: "IP", COSINE: "cosine"}


def exact_scores(oracle, metric, xb, xq):
    """(s64 [nq, n], |exact32 - e64| [nq, n]) for the operands the kernel sees."""
    x64, q64 = xb.astype(np.float64), xq.astype(np.float64)
    if metric == L2:
        e64 = np.stack([np.sum((q[None, :] - x64) ** 2, axis=1) for q in q64])  # not the expansion: exact against an offset
        e32 = np.array([[oracle.l2sqr(q, x) for x in xb] for q in xq], np.float64)
        s64 = e64 - np.einsum("qd,qd->q", q64, q64)[:, None]
    else:
        e64 = q64 @ x64.T
        e32 = np.array([[oracle.ip(q, x) for x in xb] for q in xq], np.float64)
        s64 = -e64
    return s64, np.abs(e32 - e64)


@pytest.mark.parametrize("d", [32, 36, 100, 768, 1536, 4096])
@pytest.mark.parametrize("family", sorted(E.FAMILIES))
def test_tc_score_error_within_eps(oracle, family, d):
    n, nq = 512, 16
    rng = np.random.default_rng(d * 7 + len(family))
    xb, xq = E.FAMILIES[family](rng, n, nq, d)
    report = []
    for metric in (L2, IP, COSINE):
        ix = b200vs.Index(FLAT, metric, d)
        ix.add(xb, np.arange(n, dtype=np.int64))
        b, q = (oracle.normalize_faiss(xb), oracle.normalize_faiss(xq)) if metric == COSINE else (xb, xq)
        s64, rerr = exact_scores(oracle, metric, b, q)
        for split in (False, True):
            approx, eps = ix.tc_scores(xq, split=split)
            assert approx.shape == (nq, n) and np.all(np.isfinite(approx))
            assert np.all(eps >= 0)
            lhs = np.abs(approx.astype(np.float64) - s64) + rerr
            ratio = np.divide(lhs, eps[:, None].astype(np.float64), out=np.zeros_like(lhs), where=lhs > 0)
            worst = float(ratio.max())
            report.append(f"{METRICS[metric]}/{'split' if split else 'single'}={worst:.3f}")
            bad = np.argwhere(lhs > eps[:, None])
            assert bad.size == 0, (f"{family} d={d} {METRICS[metric]} split={split}: bound violated at (q, row) "
                                   f"{bad[0].tolist()}: |err| {lhs[tuple(bad[0])]:.6g} > eps {eps[bad[0][0]]:.6g}")
            if family == "coherent" and metric != COSINE:
                # tightness: the hardware reaches what the operand model predicts, so eps is not loose by more than ~25 %
                emu = E.emulated_ratio(b, q, metric == L2, split)
                assert worst >= 0.8 * emu, f"d={d} {METRICS[metric]} split={split}: measured {worst:.4f}, emulated {emu:.4f}"
                if not split and d == 32:
                    assert worst >= 0.7
        ix.close()
    print(f"\n[tc bound] {family:9s} d={d:5d} max |err|/eps: " + " ".join(report))


def test_tc_scores_rejects_what_the_tile_kernel_cannot_run():
    for t, d in ((FLAT, 30), (FLAT, 28), (b200vs.IVF_FLAT, 64)):
        ix = b200vs.Index(t, L2, d, nlist=4) if t != FLAT else b200vs.Index(t, L2, d)
        with pytest.raises(b200vs.B200VSError) as e:
            ix.tc_scores(np.zeros((16, d), np.float32))
        assert e.value.code == b200vs.EILLEGAL_PARAMETERS


def test_tc_scores_tombstones_are_inf():
    rng = np.random.default_rng(3)
    xb = rng.random((300, 64), dtype=np.float32)
    ix = b200vs.Index(FLAT, L2, 64)
    ix.add(xb, np.arange(300, dtype=np.int64))
    ix.delete(np.arange(0, 300, 5))
    s, eps = ix.tc_scores(rng.random((16, 64), dtype=np.float32))
    assert s.shape == (16, 300)
    assert np.all(np.isinf(s[:, ::5])) and np.all(np.isfinite(np.delete(s, np.s_[::5], axis=1)))
