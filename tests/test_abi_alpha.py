"""CPU test: the ctypes prototypes of the rendered-alpha entry points (gsb_alpha, gsb_backward_alpha,
gsb_backward_batch_alpha) agree with include/gs_b200.h, parameter by parameter."""
import ctypes
import os
import re
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAMES = ("gsb_alpha", "gsb_backward_alpha", "gsb_backward_batch_alpha")


def _header_params(name):
    src = open(os.path.join(ROOT, "include", "gs_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    m = re.search(r"int32_t\s+" + name + r"\s*\(([^;]*)\)\s*;", src)
    assert m, name
    return [" ".join(p.split()) for p in m.group(1).split(",")]


def _expected(param, dgr):
    """ctypes type a header parameter must be declared with."""
    structs = {"GsbSettings": dgr._Settings, "GsbInputs": dgr._Inputs, "GsbState": dgr._State, "GsbSplitSH": dgr._SplitSH,
               "GsbGrads": dgr._Grads, "GsbCameraGrads": dgr._CameraGrads, "GsbPeerTable": dgr._PeerTable}
    if param.startswith("gsb_alloc_fn"):
        return dgr._ALLOC_FN
    if param.startswith("gsb_chunk_fn"):
        return dgr._CHUNK_FN
    for s, cls in structs.items():
        if re.search(r"\b" + s + r"\s*\*", param):
            return ctypes.POINTER(cls)
    if "*" in param:
        return ctypes.c_void_p
    assert param.startswith("int32_t"), param
    return ctypes.c_int32


def test_alpha_prototypes_match_the_header():
    sys.path.insert(0, os.path.join(ROOT, "gaussian-splatting_b200"))
    import diff_gaussian_rasterization as dgr
    for name in NAMES:
        params = _header_params(name)
        fn = getattr(dgr._C, name)
        assert fn.restype is ctypes.c_int32, name
        assert len(fn.argtypes) == len(params), (name, params)
        for i, (p, t) in enumerate(zip(params, fn.argtypes)):
            assert t is _expected(p, dgr), (name, i, p, t)
