"""CPU test: the ctypes mirror of GsbCameraGrads agrees with include/gs_b200.h as gcc lays it out (the companion of
test_abi.py::test_ctypes_mirrors_agree_with_the_c_compiler for the camera gradient outputs)."""
import ctypes
import os
import shutil
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_camera_grads_mirror_agrees_with_the_c_compiler(tmp_path):
    gcc = shutil.which("gcc", path="/usr/bin") or shutil.which("gcc")
    if gcc is None:
        pytest.skip("no C compiler")
    sys.path.insert(0, os.path.join(ROOT, "gaussian-splatting_b200"))
    import diff_gaussian_rasterization as dgr
    fields = ["dL_d" + k for k in dgr.CAMERA_KEYS]
    assert [f for f, _ in dgr._CameraGrads._fields_] == fields
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "gs_b200.h"', 'int main(void) {',
             'printf("GSB_ABI_VERSION %d\\n", GSB_ABI_VERSION);', 'printf("GsbCameraGrads %zu\\n", sizeof(GsbCameraGrads));']
    lines += [f'printf("{f} %zu\\n", offsetof(GsbCameraGrads, {f}));' for f in fields]
    lines.append("return 0; }")
    src = tmp_path / "probe.c"
    src.write_text("\n".join(lines))
    exe = tmp_path / "probe"
    subprocess.run([gcc, "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    got = dict(l.split() for l in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.splitlines())
    assert int(got["GSB_ABI_VERSION"]) == dgr.ABI_VERSION == 6
    assert int(got["GsbCameraGrads"]) == ctypes.sizeof(dgr._CameraGrads)
    for f in fields:
        assert int(got[f]) == getattr(dgr._CameraGrads, f).offset, f
