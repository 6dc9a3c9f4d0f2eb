"""numpy model of the tile kernel's TF32 arithmetic (tc_scan.cu) and the adversarial data that stresses it.

TEST INFRASTRUCTURE, shared by test_tf32_emulation.py (CPU), test_gpu_tc_bound.py and test_gpu_tc_adversarial.py.

Model of one approximate score (DESIGN.md 4.2):
  * single pass: the tensor core truncates the row operand to TF32 (low 13 mantissa bits dropped); the query was rounded
    to TF32 by cvt.rna (nearest, ties away from zero);
  * split pass (coarse quantiser): rows hi = truncated, lo = x - hi (the tensor core truncates lo); queries hi = rna(q),
    lo = rna(q - hi); the sum hi*hi + lo*hi + hi*lo;
  * products and sums exact (float64), so the emulated error is the operand error alone.
Score: L2 = ||x||^2 - 2 <q, x>, IP / cosine = -<q, x>.
"""
import numpy as np


def _bits(x):
    return np.ascontiguousarray(x, dtype=np.float32).view(np.uint32)


def tf32_trunc(x):
    return (_bits(x) & np.uint32(0xFFFFE000)).view(np.float32)


def tf32_rna(x):
    """cvt.rna.tf32.f32 on finite inputs: add half a TF32 ulp to the magnitude, then truncate (ties away from zero)."""
    return ((_bits(x) + np.uint32(0x1000)) & np.uint32(0xFFFFE000)).view(np.float32)


def with_low_bits(v, low):
    """v (float32) with its low 13 mantissa bits replaced by `low`."""
    return ((_bits(v) & np.uint32(0xFFFFE000)) | np.uint32(low)).view(np.float32)


def approx_scores(xb, xq, l2, split):
    """Emulated tile-kernel scores [nq, n] (float64)."""
    xb, xq = np.asarray(xb, np.float32), np.asarray(xq, np.float32)
    if split:
        xh = tf32_trunc(xb)
        xl = tf32_trunc(xb - xh)  # xb - xh is exact in FP32
        qh = tf32_rna(xq)
        ql = tf32_rna(xq - qh)
        xh, xl, qh, ql = (a.astype(np.float64) for a in (xh, xl, qh, ql))
        dot = qh @ xh.T + qh @ xl.T + ql @ xh.T
    else:
        dot = tf32_rna(xq).astype(np.float64) @ tf32_trunc(xb).astype(np.float64).T
    if not l2:
        return -dot
    x64 = xb.astype(np.float64)
    return np.einsum("ij,ij->i", x64, x64)[None, :] - 2.0 * dot


def true_scores(xb, xq, l2):
    """float64 scores of the FP32 operands: L2 = ||x||^2 - 2 <q, x> (= distance - ||q||^2), IP = -<q, x>."""
    x64, q64 = np.asarray(xb, np.float64), np.asarray(xq, np.float64)
    dot = q64 @ x64.T
    if not l2:
        return -dot
    return np.einsum("ij,ij->i", x64, x64)[None, :] - 2.0 * dot


def tc_eps(l2, qnorm_sq, max_norm, d, split):
    """Restatement of tc_eps() (tc_scan.cu) in FP32, for the emulation test only: the GPU tests read the device's value."""
    f = np.float32
    qn = np.sqrt(np.asarray(qnorm_sq, f))
    m = f(max_norm)
    operand = f(2.0 if l2 else 1.0) * (f(1.9073486e-6) if split else f(0.0014648438)) * qn * m
    accum = f(2.0) * f(d + 64) * f(5.9604645e-8) * ((m + qn) * (m + qn) if l2 else qn * m)
    return (operand + accum).astype(f)


def emulated_eps(xb, xq, l2, split):
    xb64, xq64 = np.asarray(xb, np.float64), np.asarray(xq, np.float64)
    max_norm = np.sqrt(np.max(np.einsum("ij,ij->i", xb64, xb64))) if xb64.size else 0.0
    return tc_eps(l2, np.einsum("ij,ij->i", xq64, xq64), max_norm, xb.shape[1], split).astype(np.float64)


def emulated_ratio(xb, xq, l2, split):
    """max over (query, row) of |emulated approx - true| / eps (0 where both are 0: IP against a zero query)."""
    err = np.abs(approx_scores(xb, xq, l2, split) - true_scores(xb, xq, l2))
    eps = np.broadcast_to(emulated_eps(xb, xq, l2, split)[:, None], err.shape)
    return float(np.max(np.divide(err, eps, out=np.zeros_like(err), where=err > 0)))


def normalize(x):
    """Cosine: the rows and queries the kernel sees (faiss normalisation; zero rows stay zero)."""
    x = np.asarray(x, np.float32)
    n = np.sqrt(np.einsum("ij,ij->i", x.astype(np.float64), x.astype(np.float64)))
    out = x.copy()
    nz = n > 0
    out[nz] = (x[nz] / n[nz, None]).astype(np.float32)
    return out


# ---------------------------------------------------------------------------------------------------------------------
# data families for the bound test: (rows [n, d], queries [nq, d]), float32
# ---------------------------------------------------------------------------------------------------------------------
def fam_uniform(rng, n, nq, d):
    return rng.random((n, d), dtype=np.float32), rng.random((nq, d), dtype=np.float32)


def fam_normal(rng, n, nq, d):  # mixed signs: cancellation in the dot product
    return rng.standard_normal((n, d)).astype(np.float32), rng.standard_normal((nq, d)).astype(np.float32)


def fam_offset(rng, n, nq, d):  # a large common offset: every distance is a small difference of large terms
    return (1000 + 1e-3 * rng.random((n, d))).astype(np.float32), (1000 + 1e-3 * rng.random((nq, d))).astype(np.float32)


def fam_norm_span(rng, n, nq, d):  # row norms spread over 2^-20 .. 2^20 within one index
    xb = rng.standard_normal((n, d)) * np.exp2(rng.integers(-20, 21, n))[:, None]
    xq = rng.standard_normal((nq, d)) * np.exp2(rng.integers(-20, 21, nq))[:, None]
    return xb.astype(np.float32), xq.astype(np.float32)


def fam_zeros(rng, n, nq, d):  # all-zero rows and all-zero queries among ordinary ones
    xb, xq = fam_normal(rng, n, nq, d)
    xb[::3] = 0
    xq[::4] = 0
    return xb, xq


def fam_coherent(rng, n, nq, d):
    """Every row coordinate is +-2^e (1 + 0x1FFF ulp): truncation drops almost 2^-10 of it, always towards zero.  Every
    query coordinate is +-2^e (1 + 0x0FFF ulp): RN rounds it down by almost 2^-11.  Query i has the signs (and exponents)
    of row i, so every product of that pair is positive and all the operand errors add up."""
    e = np.exp2(rng.integers(-1, 2, d)).astype(np.float32)  # one exponent pattern: every row has the largest norm
    sx = rng.choice(np.float32([-1, 1]), (n, d))
    xb = sx * with_low_bits(e, 0x1FFF)[None, :]
    xq = sx[np.arange(nq) % n] * with_low_bits(e, 0x0FFF)[None, :]
    return xb.astype(np.float32), xq.astype(np.float32)


FAMILIES = {"uniform": fam_uniform, "normal": fam_normal, "offset": fam_offset, "norm_span": fam_norm_span,
            "zeros": fam_zeros, "coherent": fam_coherent}


# ---------------------------------------------------------------------------------------------------------------------
# decoys for the end-to-end tests: one query, its true k-th neighbour R and a decoy D whose exact distance lies just
# above R's while its approximate score lies well below R's.  The decoy margin is (approx R - approx D) / (2 eps): the
# finish kernel keeps R only while that margin is below 1, so a generator with margin m > 0.5 breaks any kernel whose
# eps is half of what it claims.  Coordinates [0, d/2) hold the query and its structure; filler rows live in [d/2, d),
# orthogonal to the query, so their scores never compete.
# ---------------------------------------------------------------------------------------------------------------------
def _filler(rng, nfill, d, lo, hi):
    f = np.zeros((nfill, d))
    g = rng.standard_normal((nfill, d - d // 2))
    f[:, d // 2:] = g / np.linalg.norm(g, axis=1, keepdims=True) * rng.uniform(lo, hi, (nfill, 1))
    return f.astype(np.float32)


def decoy_l2(rng, d, k=1, nfill=1000):
    """L2.  q has support S (half of the query coordinates), norm ~ M / 8.  R points along q with maximal truncation, so
    its approximate score is too high.  D is the same pattern negated, with 0.75 of R's norm and maximal truncation, so
    its approximate score is too low, plus an orthogonal part on the query's zero coordinates, bisected so that D's exact
    distance lies just above R's.  k - 1 scaled copies of R are strictly closer than R and than D's approximate score.
    Returns (rows, query [1, d], row of R, row of D)."""
    h = d // 2
    perm = rng.permutation(h)
    S, T = perm[: h // 2], perm[h // 2:]
    sg = rng.choice(np.float32([-1, 1]), S.size)
    q = np.zeros(d, np.float32)
    q[S] = sg * with_low_bits(np.float32(0.125), 0x0FFF)
    R = np.zeros(d, np.float32)
    R[S] = sg * with_low_bits(np.float32(1.0), 0x1FFF)
    u = rng.standard_normal(T.size)
    u /= np.linalg.norm(u)

    def make_d(t):
        D = np.zeros(d, np.float32)
        D[S] = -sg * with_low_bits(np.float32(0.75), 0x1FFF)
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
    rows = np.concatenate([_filler(rng, nfill, d, 0.93 * mR, 0.99 * mR), np.array(closer + [R, D], np.float32).reshape(-1, d)])
    return rows, q[None, :], rows.shape[0] - 2, rows.shape[0] - 1


def decoy_ip(rng, d, k=1, nfill=1000):
    """IP.  The query support is split in halves: on S1 the query rounds down by almost 2^-11 and R (aligned, maximal
    truncation) loses almost 2^-10, so R's approximate score is too high; on S2 the query rounds UP by almost 2^-11 and D
    (aligned, coordinates exact in TF32) loses nothing, so D's approximate score is too low.  D's coordinates are TF32
    steps above 1 chosen so that <q, D> lies just below <q, R>.  k - 1 copies of R scaled up by up to 4 % are strictly
    closer.  Returns (rows, query [1, d], row of R, row of D)."""
    h = d // 2
    perm = rng.permutation(h)
    S1, S2 = perm[: h // 2], perm[h // 2:]
    s1 = rng.choice(np.float32([-1, 1]), S1.size)
    s2 = rng.choice(np.float32([-1, 1]), S2.size)
    q = np.zeros(d, np.float32)
    q[S1] = s1 * with_low_bits(np.float32(1.0), 0x0FFF)
    q[S2] = s2 * with_low_bits(np.float32(1.0), 0x1001)
    R = np.zeros(d, np.float32)
    R[S1] = s1 * with_low_bits(np.float32(1.0), 0x1FFF)
    P = float(q.astype(np.float64) @ R.astype(np.float64))
    qa = np.abs(q[S2].astype(np.float64))
    step = 2.0 ** -10  # one TF32 ulp of a coordinate in [1, 2)
    n_steps = int(np.floor((P - qa.sum()) / (step * qa[0])))
    while True:
        mag = 1.0 + step * (n_steps // S2.size + (np.arange(S2.size) < n_steps % S2.size))
        D = np.zeros(d, np.float32)
        D[S2] = s2 * mag.astype(np.float32)
        if float(q.astype(np.float64) @ D.astype(np.float64)) < P:
            break
        n_steps -= 1
    assert np.array_equal(tf32_trunc(D), D)
    closer = [(R * np.float32(1 + 0.004 * m)).astype(np.float32) for m in range(1, k)]
    mR = float(np.linalg.norm(R.astype(np.float64)))
    rows = np.concatenate([_filler(rng, nfill, d, 0.5 * mR, mR), np.array(closer + [R, D], np.float32).reshape(-1, d)])
    return rows, q[None, :], rows.shape[0] - 2, rows.shape[0] - 1


def closer_ip(R, toward, k):
    """k - 1 rows strictly closer than R by inner product, at R's norm: R rotated towards the unit vector `toward`
    (orthogonal to R, positive against the query) by 0.05 m rad, so they never raise max ||x|| (eps) above the pair's."""
    nR = float(np.linalg.norm(R.astype(np.float64)))
    return [(np.cos(0.05 * m) * R + np.sin(0.05 * m) * nR * toward).astype(np.float32) for m in range(1, k)]


def lower_until_below(q, D, S, P):
    """Lower D's magnitudes on S one step of the 10-bit mantissa grid (TF32 and FP16 alike) at a time, coordinate after coordinate, keeping their low 13 bits, until
    <q, D> < P.  Returns D."""
    D = D.copy()
    i = 0
    while float(q.astype(np.float64) @ D.astype(np.float64)) >= P:
        j = S[i % S.size]
        low = int(_bits(D[j])[0]) & 0x1FFF
        g = np.float32(np.nextafter(np.float16(abs(tf32_trunc(D[j])[0])), np.float16(0)))
        D[j] = np.sign(D[j]) * with_low_bits(g, low)[0]
        i += 1
    return D


def _coord(target, low):
    """The largest FP32 value <= target whose top 10 mantissa bits lie on the TF32 / FP16 grid and whose low 13 bits are `low`."""
    g = np.float16(target)
    while with_low_bits(np.float32(g), low)[0] > target:
        g = np.nextafter(g, np.float16(0))
    return with_low_bits(np.float32(g), low)[0]


def _unit(x, axis):
    """x completed to unit norm by one coordinate on `axis` (which x leaves zero): |1 - ||x||^2| stays far below the
    1e-5 under which the index's cosine normalisation leaves a vector bit for bit as it is."""
    n2 = float(x.astype(np.float64) @ x.astype(np.float64))
    assert x[axis] == 0 and n2 < 1
    x = x.copy()
    x[axis] = np.float32(np.sqrt(1.0 - n2))
    return x


def unit_decoy(rng, d, k, nfill, pats):
    """An IP pair at unit norm (the cosine decoys), so the index's cosine normalisation leaves the query, R and D bit for
    bit as they are.  pats = low 13 bits of (query on S1, query on S2, R, D).  The query puts half of its mass on S1 and
    half on S2 (n coordinates each), R all of its mass on S1 and D on S2; every coordinate is the largest value within
    its share of the norm that carries its pattern, and every vector is completed to unit norm by one coordinate on an
    axis its partner leaves zero.  D's magnitudes are lowered one grid step at a time until <q, D> lies just below
    <q, R>; k - 1 rows rotated from R towards the query's S2 part are strictly closer; filler rows are unit vectors on
    [d/2, d).  n = 15 puts R's coordinates near mantissa 1 and the query's near sqrt 2 (their values differ by sqrt 2).
    Returns (rows, query [1, d], row of R, row of D)."""
    h = d // 2
    n = min(15, (h - 3) // 2)
    perm = rng.permutation(h)
    S1, S2, (cq, cr, cd) = perm[:n], perm[n:2 * n], perm[2 * n:2 * n + 3]
    s1 = rng.choice(np.float32([-1, 1]), n)
    s2 = rng.choice(np.float32([-1, 1]), n)
    q = np.zeros(d, np.float32)
    q[S1] = s1 * _coord(np.sqrt(0.5 / n), pats[0])
    q[S2] = s2 * _coord(np.sqrt(0.5 / n), pats[1])
    R = np.zeros(d, np.float32)
    R[S1] = s1 * _coord(np.sqrt(1.0 / n), pats[2])
    D = np.zeros(d, np.float32)
    D[S2] = s2 * _coord(np.sqrt(1.0 / n), pats[3])
    D = lower_until_below(q, D, S2, float(q.astype(np.float64) @ R.astype(np.float64)))
    q, R, D = _unit(q, cq), _unit(R, cr), _unit(D, cd)
    t = np.zeros(d)
    t[S2] = s2 / np.sqrt(n)
    rows = np.concatenate([_filler(rng, nfill, d, 1.0, 1.0), np.array(closer_ip(R, t, k) + [R, D], np.float32).reshape(-1, d)])
    return rows, q[None, :], rows.shape[0] - 2, rows.shape[0] - 1


def decoy_cos(rng, d, k=1, nfill=1000):
    """Cosine decoy against the TF32 list scan: decoy_ip's patterns (query 0x0FFF on S1, rounding down, 0x1001 on S2,
    rounding up; R 0x1FFF, losing almost a TF32 ulp to truncation; D exact in TF32) at unit norm (unit_decoy).  Like
    decoy_ip it uses less than half of the 2 eps window (about 0.37): truncation only ever lowers |D|, so D's side gains
    from the query's rounding alone.  Returns (rows, query [1, d], row of R, row of D)."""
    return unit_decoy(rng, d, k, nfill, (0x0FFF, 0x1001, 0x1FFF, 0x0000))


def decoy_margin(rows, q, r, dd, l2):
    """(emulated approx score of R - that of D) / (2 eps): the share of the finish kernel's window the decoy uses up."""
    s = approx_scores(rows[[r, dd]], q, l2, False)[0]
    eps = emulated_eps(rows, q, l2, False)[0]
    return float((s[0] - s[1]) / (2 * eps))
