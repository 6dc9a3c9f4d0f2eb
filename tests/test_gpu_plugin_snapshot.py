"""Runs the C++ test of the plugin's fork-based snapshots (dingo-store_b200/host/test_plugin_snapshot.cc): the snapshot flow of
SaveVectorIndexSnapshot replayed for every plugin type, the non-fork branch, the switch's default and NeedToSave."""
import os
import subprocess

import pytest

import b200vs
from gpu_util import require_gpu

pytestmark = pytest.mark.gpu


def test_cpp_plugin_snapshot_contract(tmp_path):
    require_gpu()
    exe = os.path.join(b200vs.PKG_ROOT, "host", "test_plugin_snapshot")
    assert os.path.exists(exe), "build it with: make -C dingo-store_b200/host"
    r = subprocess.run([exe, str(tmp_path)], capture_output=True, text=True, timeout=600)
    print(r.stdout[-3000:])
    assert r.returncode == 0 and "PLUGIN SNAPSHOT TESTS OK" in r.stdout, r.stdout[-3000:] + r.stderr[-1000:]
