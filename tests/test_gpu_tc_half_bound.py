"""The premise of the FP16 list scan's exactness (DESIGN.md 4.2), measured on the hardware: for every query q and row x

    |approx - s64| + |exact32 - e64| <= eps(q)

approx = the tile kernel's score in its FP16 arithmetic (b200vs_debug_tc_scores with split = 2 runs the production
tc_scan_kernel on a scaled FP16 copy of the rows, made as an IVF-Flat index makes its mirror), s64 / e64 = float64 score /
distance of the FP32 operands, exact32 = the engine's exact reference-order distance, eps(q) = the device's FP16 tc_eps().
The coherent FP16 family also sets a tightness floor: a kernel whose eps were 0.9 of the one it claims fails there."""
import numpy as np
import pytest

import b200vs
import fp16_emu as H
from b200vs import COSINE, FLAT, IP, L2
from gpu_util import require_gpu
from test_gpu_tc_bound import METRICS, exact_scores

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _gpu():
    require_gpu()


@pytest.mark.parametrize("d", [32, 40, 768, 1536, 4096])
@pytest.mark.parametrize("family", sorted(H.FAMILIES))
def test_tc_half_score_error_within_eps(oracle, family, d):
    n, nq = 512, 16
    rng = np.random.default_rng(d * 11 + len(family))
    xb, xq = H.FAMILIES[family](rng, n, nq, d)
    report = []
    for metric in (L2, IP, COSINE):
        ix = b200vs.Index(FLAT, metric, d)
        ix.add(xb, np.arange(n, dtype=np.int64))
        b, q = (oracle.normalize_faiss(xb), oracle.normalize_faiss(xq)) if metric == COSINE else (xb, xq)
        s64, rerr = exact_scores(oracle, metric, b, q)
        approx, eps = ix.tc_scores(xq, half=True)
        assert approx.shape == (nq, n) and np.all(np.isfinite(approx))
        assert np.all(eps >= 0)
        lhs = np.abs(approx.astype(np.float64) - s64) + rerr
        ratio = np.divide(lhs, eps[:, None].astype(np.float64), out=np.zeros_like(lhs), where=lhs > 0)
        worst = float(ratio.max())
        report.append(f"{METRICS[metric]}={worst:.3f}")
        bad = np.argwhere(lhs > eps[:, None])
        assert bad.size == 0, (f"{family} d={d} {METRICS[metric]}: bound violated at (q, row) {bad[0].tolist()}: "
                               f"|err| {lhs[tuple(bad[0])]:.6g} > eps {eps[bad[0][0]]:.6g}")
        if family == "coherent_half" and metric != COSINE:
            emu = H.emulated_ratio(b, q, metric == L2)
            assert worst >= 0.8 * emu, f"d={d} {METRICS[metric]}: measured {worst:.4f}, emulated {emu:.4f}"
            if d <= 40:
                assert worst > 0.92, f"d={d} {METRICS[metric]}: eps is looser than the arithmetic needs ({worst:.4f})"
        ix.close()
    print(f"\n[tc half bound] {family:13s} d={d:5d} max |err|/eps: " + " ".join(report))


def test_tc_half_scores_need_dim_multiple_of_8():
    ix = b200vs.Index(FLAT, L2, 36)
    ix.add(np.ones((4, 36), np.float32), np.arange(4, dtype=np.int64))
    with pytest.raises(b200vs.B200VSError) as e:
        ix.tc_scores(np.zeros((16, 36), np.float32), half=True)
    assert e.value.code == b200vs.EILLEGAL_PARAMETERS
