"""The fork-based snapshot entry points, without a GPU: the library exports them, and the staged write, the call a forked child
makes, is built so that it cannot reach CUDA: its object file has no undefined CUDA runtime or driver symbol."""
import os
import re
import subprocess

import b200vs

SNAPSHOT_ENTRY_POINTS = ("b200vs_save_stage", "b200vs_save_staged", "b200vs_save_unstage")
STAGED_WRITE_OBJ = os.path.join(b200vs.PKG_ROOT, "_build", "snapshot_write.o")


def _nm(*args):
    r = subprocess.run(["nm", *args], capture_output=True, text=True, check=True)
    return r.stdout


def test_library_exports_the_snapshot_entry_points():
    exported = {line.split()[-1] for line in _nm("-D", "--defined-only", b200vs.LIB_PATH).splitlines() if line.strip()}
    for name in SNAPSHOT_ENTRY_POINTS:
        assert name in exported, name
    b200vs.lib()  # and the binding resolves them


def test_staged_write_is_in_the_library_from_the_host_only_object():
    assert os.path.exists(STAGED_WRITE_OBJ), "build the library first (make -C dingo-store_b200)"
    defined = _nm("--defined-only", STAGED_WRITE_OBJ).split()
    assert "b200vs_save_staged" in defined


def test_staged_write_object_calls_no_cuda():
    undefined = [line.split()[-1] for line in _nm("-u", STAGED_WRITE_OBJ).splitlines() if line.strip()]
    assert "write" in undefined and "open" in undefined  # the list is the object's real imports
    cuda = [s for s in undefined if re.match(r"_*cu", s) or "cuda" in s.lower()]
    assert not cuda, cuda
    # nor any library lock or thread: a lock another parent thread held at fork() stays held in the child
    blocking = [s for s in undefined if re.search(r"pthread_(mutex|rwlock|cond|create)|mtx_|std.*mutex", s)]
    assert not blocking, blocking


def test_staged_write_source_includes_no_cuda_header():
    src = open(os.path.join(b200vs.PKG_ROOT, "csrc", "snapshot_write.cc")).read()
    headers = re.findall(r'#include\s+[<"]([^>"]+)[>"]', src)
    assert "snapshot.h" in headers
    hdr = open(os.path.join(b200vs.PKG_ROOT, "csrc", "snapshot.h")).read()
    for text in (src, hdr):
        assert not re.search(r'#include\s+[<"](cuda|cu_|cuda_runtime|.*\.cuh)', text)
