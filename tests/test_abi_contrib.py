"""CPU test: the ctypes prototypes of gsb_contribution, gsb_prune_plan and gsb_prune_apply agree with include/gs_b200.h, the
ABI version is unchanged, and ContributionStats holds what the header documents."""
import ctypes
import os
import re
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAMES = ("gsb_contribution", "gsb_prune_plan", "gsb_prune_apply")


def _header():
    return re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "gs_b200.h")).read(), flags=re.S)


def _dgr():
    sys.path.insert(0, os.path.join(ROOT, "gaussian-splatting_b200"))
    import diff_gaussian_rasterization as dgr
    return dgr


def _expected(param, dgr):
    if re.search(r"\bGsbState\s*\*", param):
        return ctypes.POINTER(dgr._State)
    if re.search(r"\bint64_t\s*\*\s*P_new", param):
        return ctypes.POINTER(ctypes.c_int64)
    if "*" in param:
        return ctypes.c_void_p
    if param.startswith("int64_t"):
        return ctypes.c_int64
    assert param.startswith("int32_t"), param
    return ctypes.c_int32


def test_prototypes_match_the_header():
    dgr = _dgr()
    for name in NAMES:
        m = re.search(r"int32_t\s+" + name + r"\s*\(([^;]*)\)\s*;", _header())
        assert m, name
        params = [" ".join(p.split()) for p in m.group(1).split(",")]
        fn = getattr(dgr._C, name)
        assert fn.restype is ctypes.c_int32, name
        assert len(fn.argtypes) == len(params), (name, params)
        for i, (p, t) in enumerate(zip(params, fn.argtypes)):
            assert t is _expected(p, dgr), (name, i, p, t)


def test_abi_version_is_unchanged_and_stats_layout():
    import torch
    dgr = _dgr()
    assert int(re.search(r"#define GSB_ABI_VERSION (\d+)", _header()).group(1)) == dgr.ABI_VERSION == 6
    st = dgr.ContributionStats(5, "cpu")
    assert st.count.dtype == torch.int64 and st.weight_sum.dtype == torch.float32 and st.weight_max.dtype == torch.float32
    assert st.count.shape == st.weight_sum.shape == st.weight_max.shape == (5,)
    assert "ContributionStats" in dgr.__all__
