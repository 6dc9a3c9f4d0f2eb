"""Runs the C++ test of the plugin's index-served brute-force search (dingo-store_b200/host/test_plugin_index_brute_force.cc)."""
import os
import subprocess

import pytest

import b200vs
from gpu_util import require_gpu

pytestmark = pytest.mark.gpu


def test_cpp_plugin_index_brute_force_contract():
    require_gpu()
    exe = os.path.join(b200vs.PKG_ROOT, "host", "test_plugin_index_brute_force")
    assert os.path.exists(exe), "build it with: make -C dingo-store_b200/host"
    r = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    print(r.stdout[-3000:])
    assert r.returncode == 0 and "PLUGIN INDEX BRUTE FORCE TESTS OK" in r.stdout, r.stdout[-3000:] + r.stderr[-1000:]
