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


@pytest.mark.parametrize("k", [1, 10])
@pytest.mark.parametrize("d", [64, 128, 768])
@pytest.mark.parametrize("gen", ["decoy_ip", "decoy_cos"])
def test_half_ip_and_cos_decoys(gen, k, d):
    """The IP and cosine pairs on the FP16 mirror: R the exact k-th neighbour, D the next, and more than half of the 2 eps
    window used up (IP 0.64 to 0.68, cosine 0.51 to 0.55), so a kernel whose window were half as wide returns D.  The
    cosine pair is at unit norm, within the 1e-5 under which the index's normalisation leaves a vector as it is."""
    rows, q, r, dd = getattr(H, gen)(np.random.default_rng(k * d + 5), d, k)
    score = E.true_scores(rows, q, False)[0]
    order = np.argsort(score, kind="stable")
    assert order[k - 1] == r and order[k] == dd, "R must be the exact k-th neighbour and D the next"
    assert score[dd] - score[r] < 1e-4 * abs(score[r]), "D must lie just above R"
    if gen == "decoy_cos":
        n2 = np.einsum("ij,ij->i", rows.astype(np.float64), rows.astype(np.float64))
        assert np.all(np.abs(1 - n2) < 1e-6) and abs(1 - float(np.sum(q.astype(np.float64) ** 2))) < 1e-6
    m = H.decoy_margin(rows, q, r, dd, l2=False)
    assert (0.6 if gen == "decoy_ip" else 0.5) < m < 1.0, m
