"""CPU test: the ctypes mirrors of GsbSplitSH and GsbSparseAdamGroup agree with include/gs_b200.h as gcc lays it out (the
companion of test_abi.py::test_ctypes_mirrors_agree_with_the_c_compiler for the structs of the split SH input and the
sparse optimizer)."""
import ctypes
import os
import shutil
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_split_sh_and_sparse_adam_mirrors_agree_with_the_c_compiler(tmp_path):
    gcc = shutil.which("gcc", path="/usr/bin") or shutil.which("gcc")
    if gcc is None:
        pytest.skip("no C compiler")
    sys.path.insert(0, os.path.join(ROOT, "gaussian-splatting_b200"))
    import diff_gaussian_rasterization as dgr
    probes = {"GsbSplitSH": (dgr._SplitSH, ["dc", "rest", "dL_ddc", "dL_drest"]),
              "GsbSparseAdamGroup": (dgr._SparseAdamGroup, ["param", "grad", "exp_avg", "exp_avg_sq", "width", "lr", "eps"])}
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "gs_b200.h"', 'int main(void) {',
             'printf("GSB_MAX_SPARSE_GROUPS %d\\n", GSB_MAX_SPARSE_GROUPS);']
    for cname, (_, fields) in probes.items():
        lines.append(f'printf("{cname} %zu\\n", sizeof({cname}));')
        for f in fields:
            lines.append(f'printf("{cname}.{f} %zu\\n", offsetof({cname}, {f}));')
    lines.append("return 0; }")
    src = tmp_path / "probe.c"
    src.write_text("\n".join(lines))
    exe = tmp_path / "probe"
    subprocess.run([gcc, "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    got = dict(l.split() for l in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.splitlines())
    assert int(got["GSB_MAX_SPARSE_GROUPS"]) == dgr.MAX_SPARSE_GROUPS
    for cname, (ct, fields) in probes.items():
        assert int(got[cname]) == ctypes.sizeof(ct), cname
        for f in fields:
            assert int(got[f"{cname}.{f}"]) == getattr(ct, f).offset, (cname, f)
