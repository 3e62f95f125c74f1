"""CPU tests of the drop-in boundary: the C-ABI library builds, loads and exports every symbol include/vgicp_b200.h
declares; without a GPU, creating a handle fails loudly (no CPU fallback)."""
import ctypes
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared_symbols():
    src = open(os.path.join(ROOT, "include", "vgicp_b200.h")).read()
    return sorted(set(re.findall(r"VGICP_API\s+[\w\s\*]+?\b(vgicp_\w+)\s*\(", src)))


def test_header_symbols_all_exported():
    from fast_gicp_b200 import core

    lib = core.load_library()
    declared = _declared_symbols()
    assert len(declared) >= 38
    assert sorted(core.EXPORTED_SYMBOLS) == declared  # the binding knows exactly the header's surface
    for name in declared:
        assert hasattr(lib, name), name
    assert b"sm_90a" in lib.vgicp_version()


def test_library_is_sm90a_only():
    """The fatbin carries exactly one image: sm_90a (no PTX fallback for other architectures)."""
    import subprocess

    from fast_gicp_b200 import core

    out = subprocess.run(["cuobjdump", "--list-elf", core.LIB_PATH], capture_output=True, text=True)
    if out.returncode != 0:
        pytest.skip("cuobjdump unavailable")
    archs = set(re.findall(r"sm_\d+a?", out.stdout))
    assert archs == {"sm_90a"}, out.stdout


def test_no_cpu_fallback_without_gpu():
    import torch

    from fast_gicp_b200 import core

    if torch.cuda.is_available():
        pytest.skip("GPU present")
    with pytest.raises(core.VgicpError) as e:
        core.Core(0)
    assert e.value.code == core.ERR_NO_DEVICE
    h = ctypes.c_void_p()
    assert core.load_library().vgicp_create(0, ctypes.byref(h)) == core.ERR_NO_DEVICE


def test_product_never_imports_oracle():
    """The oracle is test infrastructure: nothing under fast_gicp_b200/ may reference it."""
    pkg = os.path.join(ROOT, "fast_gicp_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".hpp", ".h", ".cpp")):
                text = open(os.path.join(dirpath, f), errors="replace").read()
                assert not re.search(r"^\s*(import|from)\s+oracle\b", text, re.M), f
                assert "vgicp_oracle" not in text and not re.search(r"\borc_\w+\s*\(", text), f


def test_null_handle_is_rejected():
    from fast_gicp_b200 import core

    lib = core.load_library()
    assert lib.vgicp_set_resolution(None, 1.0) == core.ERR_INVALID_ARGUMENT
    assert lib.vgicp_destroy(None) == core.OK
