"""The C-ABI library loads and exports every symbol include/pvn3d_b200.h declares (no compute)."""
import ctypes
import os
import re

from pvn3d_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def declared_symbols():
    src = open(os.path.join(ROOT, "include", "pvn3d_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(pvn3d_[a-z0-9_]+)\s*\(", src)))


def test_library_exports_every_declared_symbol():
    lib = _lib.load()
    names = declared_symbols()
    assert len(names) >= 20
    for n in names:
        assert hasattr(lib, n), f"{n} declared in include/pvn3d_b200.h but not exported"


def test_binding_table_matches_header():
    # every declared symbol has ctypes argtypes (so a signature drift is caught at load time)
    assert set(declared_symbols()) == set(_lib.EXPORTED_SYMBOLS)


def test_version_and_strerror():
    lib = _lib.load()
    assert lib.pvn3d_version() == 2
    assert lib.pvn3d_strerror(0) == b"ok"
    assert lib.pvn3d_strerror(-2) == b"unsupported size"


def test_no_torch_dependency_in_library():
    # the boundary is a C ABI: the shared object must not link against torch / ATen
    import subprocess

    out = subprocess.run(["ldd", _lib.LIB_PATH], capture_output=True, text=True).stdout
    assert "torch" not in out and "c10" not in out


def test_workspace_queries_are_host_only():
    lib = _lib.load()
    assert lib.pvn3d_meanshift_workspace_bytes(12288, 9, 300) > 12288 * 32
    assert lib.pvn3d_meanshift_workspace_bytes(12288, 9, 100000) == 0      # max_iter cap
    assert lib.pvn3d_frame_poses_workspace_bytes(2, 2048, 8, 22, 300) > 0
    assert lib.pvn3d_frame_poses_workspace_bytes(0, 2048, 8, 22, 300) == 0
