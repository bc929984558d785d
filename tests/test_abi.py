"""The C-ABI shared library builds for sm_90a, loads, and exports exactly the entry points that
include/cfm_b200.h declares (no compute is launched: this runs without a GPU)."""
import ctypes
import os
import re

import pytest

from conftest import ROOT


def _declared_symbols():
    text = open(os.path.join(ROOT, "include", "cfm_b200.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(cfm_[a-z0-9_]+)\s*\(", text)))


def test_header_and_binding_agree():
    from cfm_b200 import _ffi
    declared = _declared_symbols()
    assert len(declared) >= 25
    assert sorted(_ffi.SIGNATURES) == declared


def test_library_loads_exports_every_symbol_and_reports_the_header_abi_version(lib_built):
    from cfm_b200 import _ffi
    assert os.path.exists(lib_built)
    lib = _ffi.load_library(lib_built)  # binds every name in SIGNATURES or raises
    header = open(os.path.join(ROOT, "include", "cfm_b200.h")).read()
    declared_version = int(re.search(r"#define\s+CFM_ABI_VERSION\s+(\d+)", header).group(1))
    assert declared_version == 2  # 2: the stage-variant and unused dopri5 / MLP entry points were removed
    assert lib.cfm_abi_version() == declared_version
    raw = ctypes.CDLL(lib_built)
    for name in _declared_symbols():
        assert hasattr(raw, name), name


def test_library_holds_sm90a_code_only(lib_built):
    import subprocess
    out = subprocess.run(["/usr/local/cuda/bin/cuobjdump", "-lelf", lib_built], capture_output=True,
                         text=True).stdout
    arches = set(re.findall(r"sm_(\d+a?)", out))
    assert arches == {"90a"}, arches


def test_sqdist_refuses_algo_2(lib_built):
    """cfm_sqdist_f32 checks algo before any CUDA call; 2 (the retired 3xTF32 path) is an argument error.  The
    pointers are dummies that are never dereferenced, and the workspace is declared too small as well, so no build
    of the library gets as far as a launch."""
    from cfm_b200 import _ffi
    lib = _ffi.load_library(lib_built)
    buf = ctypes.create_string_buffer(256)
    p = ctypes.addressof(buf)
    rc = lib.cfm_sqdist_f32(p, p, p, 4, 4, 4, 4, 1, None, 2, p, 0, None)
    assert rc == -1  # CFM_ERR_ARG
    assert b"unknown algo" in lib.cfm_last_error()


def test_rk_state_struct_layout_matches_header():
    from cfm_b200 import _ffi
    assert ctypes.sizeof(_ffi.RkState) == 72
    assert _ffi.RkState.err_acc.offset == 64


def test_missing_library_fails_loudly(tmp_path):
    from cfm_b200 import _ffi
    with pytest.raises(_ffi.CfmLibraryError):
        _ffi.load_library(str(tmp_path / "nope.so"))


def test_no_product_module_imports_the_oracle():
    pkg = os.path.join(ROOT, "cfm_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                src = open(os.path.join(dirpath, f)).read()
                assert not re.search(r"^\s*(from|import)\s+oracle\b", src, flags=re.M), f
                assert not re.search(r"^\s*(from|import)\s+(scipy|ot)\b", src, flags=re.M), f
