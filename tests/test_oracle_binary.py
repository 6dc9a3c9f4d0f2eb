"""The binary oracle (tests/binary_oracle.py) against plain restatements: np.unpackbits distances, hand-made ties, the
range-search radius rule and the binary_to_real / real_to_binary bit order.  Also the create-time refusals of the binary
types, which the library checks before it touches a device."""
import numpy as np
import pytest

import b200vs
import binary_oracle as bo


def brute(xq, xb):
    a = np.unpackbits(xq, axis=1)[:, None, :]
    b = np.unpackbits(xb, axis=1)[None, :, :]
    return (a != b).sum(-1)


def test_hamming_matches_unpackbits():
    rng = np.random.default_rng(0)
    xb = rng.integers(0, 256, (300, 65), dtype=np.uint8)
    xq = rng.integers(0, 256, (7, 65), dtype=np.uint8)
    assert np.array_equal(bo.hamming(xq, xb), brute(xq, xb))


def test_flat_mass_ties_ordered_by_id():
    rng = np.random.default_rng(1)
    xb = bo.tie_heavy(rng, 500, 8, patterns=2, flips=1)
    ids = rng.permutation(np.arange(500, dtype=np.int64) * 3 + (1 << 62))
    xq = xb[:4].copy()
    D, I = bo.flat_search(xb, ids, xq, 50)
    dist = brute(xq, xb)
    for i in range(4):
        ref = sorted(zip(dist[i].tolist(), ids.tolist()))[:50]
        assert D[i].tolist() == [float(d) for d, _ in ref] and I[i].tolist() == [j for _, j in ref]
    assert (np.diff(D, axis=1) == 0).sum() > 40  # the cut falls inside a block of equal distances


def test_probe_ties_pick_smaller_list_ids():
    c = np.zeros((6, 2), np.uint8)
    c[[0, 2, 3, 5]] = [0b11, 0]  # lists 0, 2, 3, 5 at distance 0 from q; lists 1, 4 at distance 2
    q = np.zeros((1, 2), np.uint8)
    q[0, 0] = 0b11
    assert bo.probes(c, q, 4)[0].tolist() == [0, 2, 3, 5]
    assert bo.probes(c, q, 3)[0].tolist() == [0, 2, 3]  # the tie at the boundary goes to the smaller list id
    z = np.zeros((1, 2), np.uint8)
    assert bo.probes(c, z, 3)[0].tolist() == [1, 4, 0]
    assert bo.assign(z, c).tolist() == [1] and bo.assign(q, c).tolist() == [0]


@pytest.mark.parametrize("radius,limit", [(3.0, 3), (2.5, 2), (0.0, 0), (-1.0, -1), (17.0, 17), (2.99, 2), (-0.5, 0)])
def test_range_radius_truncated_and_strict(radius, limit):
    rng = np.random.default_rng(2)
    xb = rng.integers(0, 256, (400, 2), dtype=np.uint8)
    ids = np.arange(400, dtype=np.int64)
    xq = xb[:3]
    D, I, C = bo.range_search(xb, ids, xq, radius, 1000)
    dist = brute(xq, xb)
    for i in range(3):
        want = sorted((d, j) for d, j in zip(dist[i].tolist(), ids.tolist()) if d < limit)
        assert C[i] == len(want)
        assert I[i, :C[i]].tolist() == [j for _, j in want]


def test_range_max_results_keeps_closest():
    xb = np.array([[0], [1], [3], [7], [1]], np.uint8)
    ids = np.array([50, 40, 30, 20, 10], np.int64)
    D, I, C = bo.range_search(xb, ids, np.zeros((1, 1), np.uint8), 3, 3)
    assert C.tolist() == [3] and I[0].tolist() == [50, 10, 40] and D[0].tolist() == [0, 1, 1]


def test_bit_order_lsb_first():
    x = np.array([[0b00000101, 0b10000000]], np.uint8)
    r = bo.binary_to_real(x, 16)
    want = -np.ones(16, np.float32)
    want[[0, 2, 15]] = 1
    assert np.array_equal(r[0], want)
    assert np.array_equal(bo.real_to_binary(r), x)
    assert np.array_equal(bo.real_to_binary(np.zeros((1, 8), np.float32)), [[0]])  # > 0, not >= 0


@pytest.mark.parametrize("index_type,metric,dim", [
    (b200vs.BINARY_FLAT, b200vs.HAMMING, 0), (b200vs.BINARY_FLAT, b200vs.HAMMING, 12), (b200vs.BINARY_FLAT, b200vs.HAMMING, 32776),
    (b200vs.BINARY_IVF_FLAT, b200vs.HAMMING, 12), (b200vs.BINARY_FLAT, b200vs.L2, 64), (b200vs.BINARY_IVF_FLAT, b200vs.IP, 64),
    (b200vs.FLAT, b200vs.HAMMING, 64), (b200vs.IVF_FLAT, b200vs.HAMMING, 64)])
def test_create_refusals(index_type, metric, dim):
    with pytest.raises(b200vs.B200VSError) as e:
        b200vs.Index(index_type, metric, dim)
    assert e.value.code == b200vs.EILLEGAL_PARAMETERS
