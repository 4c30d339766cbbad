"""CPU test: the ctypes prototypes of the feature-map entry points (gsb_render_features, gsb_backward_features,
gsb_backward_batch_features) and the GsbFeatures mirror agree with include/gs_b200.h."""
import ctypes
import os
import re
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAMES = ("gsb_render_features", "gsb_backward_features", "gsb_backward_batch_features")


def _header():
    return re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "gs_b200.h")).read(), flags=re.S)


def _header_params(name):
    m = re.search(r"int32_t\s+" + name + r"\s*\(([^;]*)\)\s*;", _header())
    assert m, name
    return [" ".join(p.split()) for p in m.group(1).split(",")]


def _dgr():
    sys.path.insert(0, os.path.join(ROOT, "gaussian-splatting_b200"))
    import diff_gaussian_rasterization as dgr
    return dgr


def _expected(param, dgr):
    structs = {"GsbSettings": dgr._Settings, "GsbInputs": dgr._Inputs, "GsbState": dgr._State, "GsbSplitSH": dgr._SplitSH,
               "GsbGrads": dgr._Grads, "GsbCameraGrads": dgr._CameraGrads, "GsbPeerTable": dgr._PeerTable,
               "GsbFeatures": dgr._Features}
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


def test_feature_prototypes_match_the_header():
    dgr = _dgr()
    for name in NAMES:
        params = _header_params(name)
        fn = getattr(dgr._C, name)
        assert fn.restype is ctypes.c_int32, name
        assert len(fn.argtypes) == len(params), (name, params)
        for i, (p, t) in enumerate(zip(params, fn.argtypes)):
            assert t is _expected(p, dgr), (name, i, p, t)


def test_gsb_features_struct_matches_the_header():
    dgr = _dgr()
    m = re.search(r"typedef struct GsbFeatures \{(.*?)\} GsbFeatures;", _header(), flags=re.S)
    assert m
    fields = [re.match(r"\s*(.*?)\s*\**(\w+)$", f.strip()).groups() for f in m.group(1).split(";") if f.strip()]
    assert [name for _, name in fields] == [name for name, _ in dgr._Features._fields_]
    for (ctype, name), (_, t) in zip(fields, dgr._Features._fields_):
        assert t is (ctypes.c_int32 if ctype == "int32_t" else ctypes.c_void_p), (name, ctype, t)
    assert dgr.MAX_FEATURE_CHANNELS == int(re.search(r"#define GSB_MAX_FEATURE_CHANNELS (\d+)", _header()).group(1))
