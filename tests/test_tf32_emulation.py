"""CPU checks of the TF32 emulator and the adversarial generators in tf32_emu.py.  The GPU tests use these generators to
pin tc_eps(): the bound test needs data that actually reaches its premise, the end-to-end tests need decoys that only a
correct eps survives.  These tests show, without a GPU, that the data does what it is meant to."""
import numpy as np
import pytest

import tf32_emu as E


def test_tf32_rounding_modes():
    one = np.float32(1.0)
    assert E.tf32_trunc(E.with_low_bits(one, 0x1FFF)) == one
    assert E.tf32_rna(E.with_low_bits(one, 0x0FFF)) == one                       # below half an ulp: down
    assert E.tf32_rna(E.with_low_bits(one, 0x1000)) == np.float32(1 + 2 ** -10)  # tie: away from zero
    assert E.tf32_rna(-E.with_low_bits(one, 0x1000)) == np.float32(-(1 + 2 ** -10))
    x = np.random.default_rng(0).standard_normal(10000).astype(np.float32)
    assert np.all(np.abs(E.tf32_trunc(x)) <= np.abs(x))
    assert np.all(np.abs(x - E.tf32_trunc(x)) < np.abs(x) * 2.0 ** -10)
    assert np.all(np.abs(x - E.tf32_rna(x)) <= np.abs(x) * 2.0 ** -11)


@pytest.mark.parametrize("family", sorted(E.FAMILIES))
@pytest.mark.parametrize("d", [32, 100, 768])
def test_emulated_error_within_eps(family, d):
    """In exact arithmetic the operand error alone stays below eps in both modes, for every family: the rest of eps is
    the accumulation budget the GPU test checks on the hardware."""
    xb, xq = E.FAMILIES[family](np.random.default_rng(d), 256, 16, d)
    for l2 in (True, False):
        for split in (False, True):
            assert E.emulated_ratio(xb, xq, l2, split) < 1.0


def test_coherent_family_reaches_the_bound():
    """The coherent family is the evidence for the tightness floors of test_gpu_tc_bound.py: single pass within 3 % of eps
    at d = 32 (floor there: 0.7), and a split-pass ratio far enough above 0 that 0.8 of it is a real floor."""
    xb, xq = E.fam_coherent(np.random.default_rng(1), 256, 16, 32)
    for l2 in (True, False):
        assert E.emulated_ratio(xb, xq, l2, False) > 0.97
        assert E.emulated_ratio(xb, xq, l2, True) > 0.025
    # the easy families stay far from it: a suite built on them would not notice a halved eps
    for fam in ("uniform", "normal"):
        xb, xq = E.FAMILIES[fam](np.random.default_rng(2), 256, 16, 32)
        assert E.emulated_ratio(xb, xq, True, False) < 0.3


@pytest.mark.parametrize("k", [1, 10])
@pytest.mark.parametrize("d", [64, 128])
def test_decoys(k, d):
    for gen, l2, floor in ((E.decoy_l2, True, 0.6), (E.decoy_ip, False, 0.4)):
        rows, q, r, dd = gen(np.random.default_rng(k * d), d, k)
        score = E.true_scores(rows, q, l2)[0]
        order = np.argsort(score, kind="stable")
        assert order[k - 1] == r and order[k] == dd, "R must be the exact k-th neighbour and D the next"
        assert score[dd] - score[r] < 1e-4 * abs(score[r]), "D must lie just above R"
        approx = E.approx_scores(rows, q, l2, False)[0]
        assert approx[dd] < approx[r], "D's approximate score must lie below R's"
        m = E.decoy_margin(rows, q, r, dd, l2)
        # L2: more than half of the 2 eps window, so halving eps drops R from the window
        assert floor < m < 1.0, m


@pytest.mark.parametrize("k", [1, 10])
def test_list_form_decoys(k):
    """The TF32 list form at d = 132 (16-byte rows, d % 8 != 0: IVF-Flat keeps no FP16 mirror).  L2 uses more than half of
    the 2 eps window; IP and cosine (unit norm) only about 0.45 and 0.37, because truncation lowers |D| as well, so D's
    side gains from the query's rounding alone: the GPU tests hold them to these emulated floors."""
    d = 132
    assert (4 * d) % 16 == 0 and d % 8 != 0
    for gen, l2, floor in ((E.decoy_l2, True, 0.6), (E.decoy_ip, False, 0.4), (E.decoy_cos, False, 0.35)):
        rows, q, r, dd = gen(np.random.default_rng(k * d), d, k)
        score = E.true_scores(rows, q, l2)[0]
        order = np.argsort(score, kind="stable")
        assert order[k - 1] == r and order[k] == dd, "R must be the exact k-th neighbour and D the next"
        approx = E.approx_scores(rows, q, l2, False)[0]
        assert approx[dd] < approx[r], "D's approximate score must lie below R's"
        if gen is E.decoy_cos:
            n2 = np.einsum("ij,ij->i", rows.astype(np.float64), rows.astype(np.float64))
            assert np.all(np.abs(1 - n2) < 1e-6)
        assert floor < E.decoy_margin(rows, q, r, dd, l2) < 1.0
