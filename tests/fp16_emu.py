"""numpy model of the tile kernel's FP16 arithmetic (the IVF-Flat list scan on the FP16 mirror, tc_scan.cu) and the
adversarial data that stresses it.

TEST INFRASTRUCTURE, shared by test_fp16_emulation.py (CPU), test_gpu_tc_half_bound.py and test_gpu_ivf_flat_half.py.

Model of one approximate score (DESIGN.md 4.2):
  * every row and every query is scaled by 2^-e, e chosen so that its largest |coordinate| lands in [2^14, 2^15), and
    rounded to FP16 to nearest (ties to even); np.float16 performs the same rounding, subnormals included;
  * products and sums exact (float64), then scaled back by 2^(e_x + e_q), so the emulated error is the operand error alone.
Score: L2 = ||x||^2 - 2 <q, x>, IP / cosine = -<q, x>.
"""
import numpy as np

import tf32_emu as E


def half_exp(x):
    """Per-row e with max |x_i| * 2^-e in [2^14, 2^15); 0 for a zero row."""
    m = np.max(np.abs(np.asarray(x, np.float32)), axis=1)
    _, ex = np.frexp(m)  # m = f 2^ex, f in [0.5, 1)
    return np.where(m > 0, ex - 1 - 14, 0).astype(np.int64)


def half_round(x):
    """The operand the tensor core sees, scaled back to the original units (float64)."""
    x = np.asarray(x, np.float32)
    e = half_exp(x)[:, None]
    h = np.ldexp(x, -e).astype(np.float16)  # the scaling is exact in FP32; the one rounding is to FP16
    return np.ldexp(h.astype(np.float64), e)


def approx_scores(xb, xq, l2):
    """Emulated tile-kernel scores [nq, n] (float64)."""
    dot = half_round(xq) @ half_round(xb).T
    if not l2:
        return -dot
    x64 = np.asarray(xb, np.float64)
    return np.einsum("ij,ij->i", x64, x64)[None, :] - 2.0 * dot


def tc_eps(l2, qnorm_sq, max_norm, d):
    """Restatement of tc_eps(..., TC_ARITH_FP16) in float64, for the emulation test only: the GPU tests read the
    device's value."""
    qn = np.sqrt(np.asarray(qnorm_sq, np.float64))
    delta = 2.0 ** -11 + np.sqrt(d) * 2.0 ** -39
    operand = (2.0 if l2 else 1.0) * delta * (2 + delta) * qn * max_norm
    accum = 2.0 * (d + 64) * 2.0 ** -24 * ((max_norm + qn) ** 2 if l2 else qn * max_norm)
    return operand + accum


def emulated_eps(xb, xq, l2):
    xb64, xq64 = np.asarray(xb, np.float64), np.asarray(xq, np.float64)
    max_norm = np.sqrt(np.max(np.einsum("ij,ij->i", xb64, xb64))) if xb64.size else 0.0
    return tc_eps(l2, np.einsum("ij,ij->i", xq64, xq64), max_norm, xb.shape[1])


def emulated_ratio(xb, xq, l2):
    """max over (query, row) of |emulated approx - true| / eps (0 where both are 0)."""
    err = np.abs(approx_scores(xb, xq, l2) - E.true_scores(xb, xq, l2))
    eps = np.broadcast_to(emulated_eps(xb, xq, l2)[:, None], err.shape)
    return float(np.max(np.divide(err, eps, out=np.zeros_like(err), where=err > 0)))


# one FP32 mantissa pattern below the FP16 midpoint: 0x0FFF in the low 13 bits rounds down by almost half an FP16 ulp
BELOW_MID = 0x0FFF


def fam_coherent_half(rng, n, nq, d):
    """Every row and query coordinate is +-2^e (1 + 0x0FFF FP32 ulp), the bottom of a binade: after the power-of-two
    scale it lies just below the midpoint between two FP16 neighbours, so RN drops almost 2^-11 of it, towards zero.
    Query i has the signs (and exponents) of row i, so every product of that pair is positive and the operand errors of
    both sides add up."""
    e = np.exp2(rng.integers(-1, 2, d)).astype(np.float32)
    sx = rng.choice(np.float32([-1, 1]), (n, d))
    v = E.with_low_bits(e, BELOW_MID)[None, :]
    return (sx * v).astype(np.float32), (sx[np.arange(nq) % n] * v).astype(np.float32)


FAMILIES = dict(E.FAMILIES, coherent_half=fam_coherent_half)


def decoy_l2(rng, d, k=1, nfill=1000):
    """L2 decoy against the FP16 rounding (layout of tf32_emu.decoy_l2).  q has support S, every coordinate rounding
    down by almost 2^-11.  R points along q, its coordinates rounding down too, so <q, R> comes out low and R's
    approximate score too high.  D is the same pattern negated at 0.75 of R's size, so <q, D> comes out less negative and
    D's approximate score too low; an orthogonal part on the query's zero coordinates is bisected so that D's exact
    distance lies just above R's.  k - 1 scaled copies of R are strictly closer.  Returns (rows, query [1, d], row of R,
    row of D)."""
    h = d // 2
    perm = rng.permutation(h)
    S, T = perm[: h // 2], perm[h // 2:]
    sg = rng.choice(np.float32([-1, 1]), S.size)
    q = np.zeros(d, np.float32)
    q[S] = sg * E.with_low_bits(np.float32(0.125), BELOW_MID)
    R = np.zeros(d, np.float32)
    R[S] = sg * E.with_low_bits(np.float32(1.0), BELOW_MID)
    u = rng.standard_normal(T.size)
    u /= np.linalg.norm(u)

    def make_d(t):
        D = np.zeros(d, np.float32)
        D[S] = -sg * E.with_low_bits(np.float32(0.75), BELOW_MID)
        D[T] = (t * u).astype(np.float32)
        return D

    def dist(x):
        return float(np.sum((q.astype(np.float64) - x.astype(np.float64)) ** 2))

    target = dist(R) * (1 + 2.0 ** -20)
    lo, hi = 0.0, float(np.linalg.norm(R.astype(np.float64)))
    for _ in range(80):
        mid = 0.5 * (lo + hi)
        lo, hi = (mid, hi) if dist(make_d(mid)) < target else (lo, mid)
    D = make_d(hi)
    assert dist(D) > dist(R)
    closer = [(R * np.float32(1 - 0.002 * m)).astype(np.float32) for m in range(1, k)]
    mR = float(np.linalg.norm(R.astype(np.float64)))
    rows = np.concatenate([E._filler(rng, nfill, d, 0.93 * mR, 0.99 * mR), np.array(closer + [R, D], np.float32).reshape(-1, d)])
    return rows, q[None, :], rows.shape[0] - 2, rows.shape[0] - 1


# one FP32 mantissa pattern above the FP16 midpoint: 0x1001 in the low 13 bits rounds up by almost half an FP16 ulp
ABOVE_MID = 0x1001


def decoy_ip(rng, d, k=1, nfill=1000):
    """IP decoy against the FP16 rounding.  The query support is split into S1 and S2.  On S1 the query's coordinates are
    +-1 with low bits 0x0FFF, so RN takes almost 2^-11 off each, and R is aligned with the same pattern: both operands
    of <q, R> come out low, so R's approximate score comes out too high.  On S2 the query's coordinates carry 0x1001,
    which rounds up, and D lies on S2 with the same round-up pattern: <q, D> comes out high, so D's approximate score
    comes out too low.  D's magnitudes are lowered one FP16 step at a time until <q, D> lies just below <q, R>.  k - 1
    rows rotated from R towards the query's S2 part are strictly closer.  Returns (rows, query [1, d], row of R, row of
    D)."""
    h = d // 2
    perm = rng.permutation(h)
    S1, S2 = perm[: h // 2], perm[h // 2:]
    s1 = rng.choice(np.float32([-1, 1]), S1.size)
    s2 = rng.choice(np.float32([-1, 1]), S2.size)
    one_lo, one_hi = E.with_low_bits(np.float32(1.0), BELOW_MID)[0], E.with_low_bits(np.float32(1.0), ABOVE_MID)[0]
    q = np.zeros(d, np.float32)
    q[S1], q[S2] = s1 * one_lo, s2 * one_hi
    R = np.zeros(d, np.float32)
    R[S1] = s1 * one_lo
    D = np.zeros(d, np.float32)
    D[S2] = s2 * one_hi
    D = E.lower_until_below(q, D, S2, float(q.astype(np.float64) @ R.astype(np.float64)))
    t = np.zeros(d)
    t[S2] = s2 / np.sqrt(S2.size)
    mR = float(np.linalg.norm(R.astype(np.float64)))
    rows = np.concatenate([E._filler(rng, nfill, d, 0.5 * mR, mR), np.array(E.closer_ip(R, t, k) + [R, D], np.float32).reshape(-1, d)])
    return rows, q[None, :], rows.shape[0] - 2, rows.shape[0] - 1


def decoy_cos(rng, d, k=1, nfill=1000):
    """Cosine decoy against the FP16 rounding: decoy_ip's rounding patterns (query 0x0FFF on S1, 0x1001 on S2; R 0x0FFF,
    D 0x1001) at unit norm, laid out by tf32_emu.unit_decoy.  The pair uses 0.51 to 0.55 of the 2 eps window at d = 64
    to 768, less than decoy_ip's 0.64 to 0.68: at unit norm the query's half-mass coordinates and R's whole-mass
    coordinates differ by sqrt 2, so the power-of-two scale cannot put both at mantissa 1, where the rounding is largest
    relative to the value.  Returns (rows, query [1, d], row of R, row of D)."""
    return E.unit_decoy(rng, d, k, nfill, (BELOW_MID, ABOVE_MID, BELOW_MID, ABOVE_MID))


def decoy_margin(rows, q, r, dd, l2=True):
    """(emulated approx score of R - that of D) / (2 eps): the share of the finish kernel's window the decoy uses up."""
    s = approx_scores(rows[[r, dd]], q, l2)[0]
    return float((s[0] - s[1]) / (2 * emulated_eps(rows, q, l2)[0]))
