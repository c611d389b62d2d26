"""The wavefront profiling tool builds its own library: it must never build a variant over the in-tree one."""
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def test_wavex_profile_help_runs_without_a_gpu():
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "wavex_profile.py"), "--help"],
                       capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, r.stderr
    assert "--out" in r.stdout


def test_variant_build_needs_its_own_output_path():
    from isaac_ros_nvblox_b200 import build_ext
    with pytest.raises(ValueError):
        build_ext.build(defines=["NVB_WAVEX_PROF=1"])


def test_lib_path_override_is_refused_once_another_library_is_loaded(monkeypatch):
    from isaac_ros_nvblox_b200 import _lib
    monkeypatch.setattr(_lib, "_lib", object())
    with pytest.raises(RuntimeError):
        _lib.load(os.path.join(ROOT, "elsewhere", "libnvblox_b200.so"))
