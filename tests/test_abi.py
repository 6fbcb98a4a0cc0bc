"""CPU checks of the drop-in boundary: libstarway_b200.so loads without a GPU, exports every
symbol include/starway_b200.h declares, and refuses to run without a CUDA device (no fallback)."""
import ctypes
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def header_symbols():
    text = open(os.path.join(ROOT, "include", "starway_b200.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(sw_[a-z_0-9]+)\s*\(", text)))


def test_header_and_python_table_agree():
    from starway_b200._core import C_ABI

    assert header_symbols() == sorted(C_ABI)


def test_product_library_exports_the_abi():
    import starway_b200 as sw

    lib = ctypes.CDLL(sw.LIB_PATH)
    for name in header_symbols():
        assert hasattr(lib, name), name
    assert sw._api.lib.sw_abi_version() == 1
    assert sw.backend_name() == "cuda-sm_90a"
    assert sw.status_string(-16) == "Request canceled"
    assert sw.status_string(-24) == "Endpoint is not connected"
    assert sw.status_string(-9) == "Message truncated"


def test_product_library_exports_nothing_else():
    import subprocess

    import starway_b200 as sw

    out = subprocess.check_output(["nm", "-D", "--defined-only", sw.LIB_PATH], text=True)
    syms = [l.split()[-1] for l in out.splitlines() if " T " in l]
    assert sorted(syms) == header_symbols()


def test_no_cpu_fallback_without_gpu():
    import starway_b200 as sw

    if sw.device_count() > 0:
        pytest.skip("a GPU is visible")
    with pytest.raises(RuntimeError, match="no CUDA device|no CPU fallback"):
        sw.Context(0)


def test_product_package_never_references_test_infrastructure():
    pkg = os.path.join(ROOT, "starway_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cpp", ".cu", ".cuh", ".h")):
                text = open(os.path.join(dirpath, f)).read()
                assert "hostsim" not in text.replace("tests/hostsim", "") or f in ("gpu.h", "_core.py"), f
                assert "import oracle" not in text and "from oracle" not in text, f
                assert "tagmatch" not in text, f
