"""CPU checks of the FP16 emulator and the adversarial generators in fp16_emu.py: the GPU tests rely on the coherent family
reaching the bound (its tightness floor) and on the decoys using up more than half of the 2 eps window."""
import numpy as np
import pytest

import fp16_emu as H
import tf32_emu as E


def test_half_rounding():
    x = np.float32([[3.0, -1.0, 0.5], [0.0, 0.0, 0.0], [2.0 ** -40, 3 * 2.0 ** -41, 0.0]])
    assert np.array_equal(H.half_exp(x), [1 - 14, 0, -40 - 14])
    assert np.array_equal(H.half_round(x), x.astype(np.float64))  # exactly representable after scaling
    one = E.with_low_bits(np.float32(1.0), H.BELOW_MID)
    assert H.half_round(np.float32([[one]]))[0, 0] == 1.0  # below the FP16 midpoint: down
    tie = E.with_low_bits(np.float32(1.0), 0x1000)
    assert H.half_round(np.float32([[tie]]))[0, 0] == 1.0  # tie: to even
    x = np.random.default_rng(0).standard_normal((64, 100)).astype(np.float32) * np.exp2(np.arange(-32, 32))[:, None]
    r = np.abs(H.half_round(x) - x) / np.abs(x)
    assert np.all(r <= 2.0 ** -11)


@pytest.mark.parametrize("family", sorted(H.FAMILIES))
@pytest.mark.parametrize("d", [32, 40, 768])
def test_emulated_error_within_eps(family, d):
    xb, xq = H.FAMILIES[family](np.random.default_rng(d), 256, 16, d)
    for l2 in (True, False):
        assert H.emulated_ratio(xb, xq, l2) < 1.0


def test_coherent_half_family_reaches_the_bound():
    """The evidence for the tightness floor of test_gpu_tc_half_bound.py: at d = 32 the operand error alone reaches more
    than 0.95 of eps, so a kernel whose eps were 0.9 of the one it claims would violate the bound there."""
    for d in (32, 40):
        xb, xq = H.fam_coherent_half(np.random.default_rng(1), 256, 16, d)
        for l2 in (True, False):
            assert H.emulated_ratio(xb, xq, l2) > 0.95
    # the TF32 coherent family and the easy families stay well below it
    for fam in ("coherent", "uniform", "normal"):
        xb, xq = H.FAMILIES[fam](np.random.default_rng(2), 256, 16, 32)
        assert H.emulated_ratio(xb, xq, True) < 0.6


@pytest.mark.parametrize("k", [1, 10])
@pytest.mark.parametrize("d", [64, 128])
def test_half_decoys(k, d):
    rows, q, r, dd = H.decoy_l2(np.random.default_rng(k * d), d, k)
    score = E.true_scores(rows, q, True)[0]
    order = np.argsort(score, kind="stable")
    assert order[k - 1] == r and order[k] == dd, "R must be the exact k-th neighbour and D the next"
    assert score[dd] - score[r] < 1e-4 * abs(score[r]), "D must lie just above R"
    approx = H.approx_scores(rows, q, True)[0]
    assert approx[dd] < approx[r], "D's approximate score must lie below R's"
    m = H.decoy_margin(rows, q, r, dd)
    assert 0.6 < m < 1.0, m  # more than half of the 2 eps window
