"""b200vs_shard_rebuild_from_range without a GPU: the library exports it, and Shard.rebuild_from_range refuses the argument
errors the library refuses before any collective (1 to 16 sources, none of them None or closed, dst not among them, no source
listed twice) without calling the library, so one rank's bad list never reaches a collective."""
import subprocess

import pytest

import b200vs


class _Shard(b200vs.Shard):
    """A shard handle that never reached the library: the refusals below must come before any call into it."""

    def __init__(self, h):
        self.h = h

    def close(self):
        self.h = None


def test_library_exports_the_entry_point():
    out = subprocess.run(["nm", "-D", "--defined-only", b200vs.LIB_PATH], capture_output=True, text=True, check=True).stdout
    assert "b200vs_shard_rebuild_from_range" in {line.split()[-1] for line in out.splitlines() if line.strip()}
    assert "b200vs_shard_rebuild_from_range" in b200vs.ABI_SYMBOLS


@pytest.fixture
def no_library(monkeypatch):
    """Any call into the library fails the test."""
    def refuse():
        raise AssertionError("the binding called the library")
    monkeypatch.setattr(b200vs, "lib", refuse)


def _code(fn):
    with pytest.raises(b200vs.B200VSError) as e:
        fn()
    return e.value.code


def test_binding_refuses_bad_source_lists(no_library):
    dst, a, b = _Shard(1), _Shard(2), _Shard(3)
    closed = _Shard(4)
    closed.close()
    bad = {
        "no sources": [],
        "17 sources": [_Shard(10 + i) for i in range(17)],
        "a None entry": [a, None],
        "a closed source": [a, closed],
        "dst among the sources": [a, dst],
        "a source listed twice": [a, b, a],
    }
    for what, srcs in bad.items():
        assert _code(lambda: dst.rebuild_from_range(srcs, 0, 100)) == b200vs.EILLEGAL_PARAMETERS, what


def test_binding_passes_range_refusals_to_the_library(no_library):
    """id_min > id_max is agreed over the ranks by the library, so the binding leaves it to the call."""
    dst, a = _Shard(1), _Shard(2)
    with pytest.raises(AssertionError, match="called the library"):
        dst.rebuild_from_range([a], 10, 5)
