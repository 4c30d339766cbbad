"""CPU test: the ctypes prototype of gsb_set_deterministic agrees with include/gs_b200.h, the header lists the switch among the
per-thread state, and the ABI version is unchanged."""
import ctypes
import os
import re
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _header_raw():
    return open(os.path.join(ROOT, "include", "gs_b200.h")).read()


def _dgr():
    sys.path.insert(0, os.path.join(ROOT, "gaussian-splatting_b200"))
    import diff_gaussian_rasterization as dgr
    return dgr


def test_prototype_matches_the_header():
    dgr = _dgr()
    code = re.sub(r"/\*.*?\*/", "", _header_raw(), flags=re.S)
    m = re.search(r"int32_t\s+gsb_set_deterministic\s*\(([^;]*)\)\s*;", code)
    assert m
    assert " ".join(m.group(1).split()) == "int32_t on"
    fn = dgr._C.gsb_set_deterministic
    assert fn.restype is ctypes.c_int32 and fn.argtypes == [ctypes.c_int32]


def test_switch_is_documented_as_per_thread_and_abi_version_is_unchanged():
    dgr = _dgr()
    head = _header_raw().split("*/", 1)[0]
    assert "deterministic switch" in head and "Per host thread" in head
    assert int(re.search(r"#define GSB_ABI_VERSION (\d+)", _header_raw()).group(1)) == dgr.ABI_VERSION == 6
