"""Ownership rule of row-sharded FLAT / HNSW indexes: b200vs_row_owner (a pure host function, no GPU) equals the numpy
mirror b200vs.shard.row_owner, and sequential ids spread evenly over the ranks."""
import numpy as np
import pytest

import b200vs
from b200vs import shard


def _id_sets():
    rng = np.random.default_rng(7)
    return {
        "sequential": np.arange(0, 20000, dtype=np.int64),
        "strided": np.arange(0, 64 * 20000, 64, dtype=np.int64),
        "negative": -np.arange(1, 20001, dtype=np.int64),
        "random": rng.integers(np.iinfo(np.int64).min, np.iinfo(np.int64).max, size=20000, dtype=np.int64),
        "edges": np.array([0, 1, -1, np.iinfo(np.int64).min, np.iinfo(np.int64).max], dtype=np.int64),
    }


@pytest.mark.parametrize("world", [1, 2, 3, 4, 7, 8, 1000, 1023, 1024])
@pytest.mark.parametrize("kind", ["sequential", "strided", "negative", "random", "edges"])
def test_library_equals_mirror(kind, world):
    ids = _id_sets()[kind]
    got = b200vs.row_owner(ids, world)
    assert got.dtype == np.int32
    assert np.array_equal(got, shard.row_owner(ids, world))
    assert got.min() >= 0 and got.max() < world


def test_known_values():
    # splitmix64's finalizer of 1 is 0x5692161d100b05e5 (the constants of the standard finalizer)
    z = np.uint64(0x5692161d100b05e5)
    assert shard.row_owner([1], 1000)[0] == int(z % np.uint64(1000))
    assert shard.row_owner([0], 7)[0] == 0


@pytest.mark.parametrize("world", [2, 4, 8])
def test_sequential_ids_spread_evenly(world):
    n = 1 << 16
    counts = np.bincount(b200vs.row_owner(np.arange(n, dtype=np.int64), world), minlength=world)
    expect = n / world
    # a uniform multinomial stays within 5 standard deviations of n / world
    assert np.all(np.abs(counts - expect) < 5 * np.sqrt(expect))


@pytest.mark.parametrize("world", [0, -1, 1025])
def test_bad_arguments(world):
    """A row-sharded index has 1 to 1024 ranks."""
    with pytest.raises(b200vs.B200VSError) as e:
        b200vs.row_owner(np.arange(4), world)
    assert e.value.code == b200vs.EILLEGAL_PARAMETERS
