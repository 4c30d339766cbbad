"""Drop-in ``diff_gaussian_rasterization`` package backed by libgs_b200.so (sm_90a CUDA, C ABI).

Mirrors the surface the reference imports at /root/reference/gaussian_renderer/__init__.py:14
(``GaussianRasterizationSettings``, ``GaussianRasterizer``) and calls at :36-52 / :91-110, plus the
``rasterize_gaussians`` autograd.Function named in BASELINE.json north_star.  ``GaussianRasterizer.forward`` also
takes the split SH input of the accel branch (``dc=features_dc, shs=features_rest``).

``SparseGaussianAdam`` (sparse_adam.py, train.py --optimizer_type sparse_adam) is bound at package top level only
when ``GSB_SPARSE_ADAM=1`` is set at import.  Its presence makes the reference scripts pass ``separate_sh=True``
(train.py:38,111, render.py:24), and the reference render() then binds ``dc`` only on its SH branch
(gaussian_renderer/__init__.py:83): ``--convert_SHs_python`` and ``override_color`` raise UnboundLocalError there, as
they do with the accel rasterizer.  Without the variable those flags keep working and the optimizer stays importable
as ``diff_gaussian_rasterization.sparse_adam.SparseGaussianAdam``.

There is no CPU path and no fallback: importing this package without the built library raises.
Host code is plumbing only -- tensors in, raw device pointers across the C ABI (include/gs_b200.h).
"""
from __future__ import annotations

import ctypes
import os
import warnings
from ctypes import CFUNCTYPE, POINTER, Structure, byref, c_char_p, c_float, c_int32, c_int64, c_size_t, c_void_p
from typing import NamedTuple, Optional

import torch
import torch.nn as nn

__all__ = ["GaussianRasterizationSettings", "GaussianRasterizer", "rasterize_gaussians", "ContributionStats"]

_PKG_DIR = os.path.dirname(os.path.abspath(__file__))
# GSB_LIBRARY: an alternative build of the same sources (A/B of compile-time knobs); default = the in-tree library
_LIB_PATH = os.environ.get("GSB_LIBRARY") or os.path.join(os.path.dirname(_PKG_DIR), "libgs_b200.so")


# ---------------------------------------------------------------------------------------------
# C ABI mirror (include/gs_b200.h)
# ---------------------------------------------------------------------------------------------
class _Settings(Structure):
    _fields_ = [("image_height", c_int32), ("image_width", c_int32), ("tanfovx", c_float), ("tanfovy", c_float),
                ("bg", c_void_p), ("scale_modifier", c_float), ("viewmatrix", c_void_p), ("projmatrix", c_void_p),
                ("sh_degree", c_int32), ("campos", c_void_p), ("prefiltered", c_int32), ("debug", c_int32),
                ("antialiasing", c_int32), ("sh_coeffs", c_int32)]


class _Inputs(Structure):
    _fields_ = [("P", c_int32), ("means3D", c_void_p), ("shs", c_void_p), ("colors_precomp", c_void_p),
                ("opacities", c_void_p), ("scales", c_void_p), ("rotations", c_void_p), ("cov3D_precomp", c_void_p)]


class _State(Structure):
    _fields_ = [("P", c_int32), ("num_tiles", c_int32), ("num_rendered", c_int64), ("num_visible", c_int64),
                ("binning_capacity", c_int64), ("geom", c_void_p), ("geom_bytes", c_size_t), ("binning", c_void_p), ("binning_bytes", c_size_t),
                ("image", c_void_p), ("image_bytes", c_size_t), ("splat", c_void_p), ("point_list", c_void_p),
                ("ranges", c_void_p), ("final_T", c_void_p), ("n_contrib", c_void_p), ("tile_order", c_void_p)]


class _Grads(Structure):
    _fields_ = [("dL_dmeans3D", c_void_p), ("dL_dmeans2D", c_void_p), ("dL_dshs", c_void_p), ("dL_dcolors", c_void_p),
                ("dL_dopacities", c_void_p), ("dL_dscales", c_void_p), ("dL_drotations", c_void_p),
                ("dL_dcov3D", c_void_p)]


class _PeerTable(Structure):          # GsbPeerTable
    _fields_ = [("world", c_int32), ("rank", c_int32), ("rows_per_rank", c_int32), ("reserved", c_int32), ("base", c_void_p * 16)]


_ALLOC_FN = CFUNCTYPE(c_void_p, c_void_p, c_int32, c_size_t)
_CHUNK_FN = CFUNCTYPE(None, c_void_p, c_int32, c_int32, c_int32)     # gsb_chunk_fn(ctx, chunk, p_begin, p_end)
ABI_VERSION = 6
COUNT_SLOTS = 17        # gsb_forward_batch_async: V counts (up to 16) + their running maximum in slot 16
BUF_GEOM, BUF_BINNING, BUF_IMAGE = 0, 1, 2


class _AdamArgs(Structure):          # GsbAdamArgs (include/gs_b200.h)
    _fields_ = [("P", c_int64), ("sh_coeffs", c_int32), ("skip_groups", c_int32), ("params", c_void_p), ("grads", c_void_p),
                ("exp_avg", c_void_p), ("exp_avg_sq", c_void_p), ("act", c_void_p), ("visible", c_void_p),
                ("step_size", c_float * 6), ("bias2_sqrt", c_float * 6), ("beta1", c_float), ("beta2", c_float), ("eps", c_float)]


class _DensifyArgs(Structure):       # GsbDensifyArgs
    _fields_ = [("P", c_int64), ("sh_coeffs", c_int32), ("n_children", c_int32), ("params", c_void_p), ("exp_avg", c_void_p),
                ("exp_avg_sq", c_void_p), ("grad_accum", c_void_p), ("denom", c_void_p), ("grad_threshold", c_float),
                ("size_limit", c_float), ("min_opacity", c_float), ("world_limit", c_float), ("scratch", c_void_p)]


class _SplitSH(Structure):           # GsbSplitSH
    _fields_ = [("dc", c_void_p), ("rest", c_void_p), ("dL_ddc", c_void_p), ("dL_drest", c_void_p)]


class _CameraGrads(Structure):       # GsbCameraGrads
    _fields_ = [("dL_dviewmatrix", c_void_p), ("dL_dprojmatrix", c_void_p), ("dL_dcampos", c_void_p), ("dL_dbg", c_void_p)]


class _Features(Structure):          # GsbFeatures
    _fields_ = [("channels", c_int32), ("features", c_void_p), ("out_features", c_void_p), ("dL_dout_features", c_void_p),
                ("dL_dfeatures", c_void_p)]


MAX_FEATURE_CHANNELS = 128          # GSB_MAX_FEATURE_CHANNELS


class _SparseAdamGroup(Structure):   # GsbSparseAdamGroup
    _fields_ = [("param", c_void_p), ("grad", c_void_p), ("exp_avg", c_void_p), ("exp_avg_sq", c_void_p), ("width", c_int32),
                ("lr", c_float), ("eps", c_float)]


MAX_SPARSE_GROUPS = 8               # GSB_MAX_SPARSE_GROUPS: groups per gsb_sparse_adam_step launch


def _load(path: Optional[str] = None):
    """Loads libgs_b200.so (or another build of the same C ABI at ``path``) and declares the prototypes."""
    _LIB_PATH = path or globals()["_LIB_PATH"]
    if not os.path.exists(_LIB_PATH):
        raise ImportError(
            f"{_LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            f"(or `make -C gaussian-splatting_b200/csrc`).  There is no CPU fallback.")
    lib = ctypes.CDLL(_LIB_PATH)
    lib.gsb_forward.restype = c_int32
    lib.gsb_forward.argtypes = [POINTER(_Settings), POINTER(_Inputs), c_void_p, c_void_p, c_void_p, c_int64, _ALLOC_FN,
                                c_void_p, POINTER(_State), c_void_p]
    lib.gsb_backward.restype = c_int32
    lib.gsb_backward.argtypes = [POINTER(_Settings), POINTER(_Inputs), POINTER(_State), c_void_p, c_void_p, c_void_p,
                                 c_void_p, POINTER(_Grads), c_int32, _ALLOC_FN, c_void_p, c_void_p]
    lib.gsb_forward_split_sh.restype = c_int32
    lib.gsb_forward_split_sh.argtypes = [POINTER(_Settings), POINTER(_Inputs), POINTER(_SplitSH), c_void_p, c_void_p, c_void_p,
                                         c_int64, _ALLOC_FN, c_void_p, POINTER(_State), c_void_p]
    lib.gsb_backward_split_sh.restype = c_int32
    lib.gsb_backward_split_sh.argtypes = [POINTER(_Settings), POINTER(_Inputs), POINTER(_SplitSH), POINTER(_State), c_void_p,
                                          c_void_p, c_void_p, c_void_p, POINTER(_Grads), c_int32, _ALLOC_FN, c_void_p, c_void_p]
    lib.gsb_backward_camera.restype = c_int32
    lib.gsb_backward_camera.argtypes = [POINTER(_Settings), POINTER(_Inputs), POINTER(_SplitSH), POINTER(_State), c_void_p, c_void_p,
                                        c_void_p, c_void_p, POINTER(_Grads), POINTER(_CameraGrads), c_int32, _ALLOC_FN, c_void_p,
                                        c_void_p]
    lib.gsb_backward_batch_camera.restype = c_int32
    lib.gsb_backward_batch_camera.argtypes = [c_int32, POINTER(_Settings), POINTER(_Inputs), POINTER(_State), c_void_p, c_void_p,
                                              c_void_p, c_void_p, POINTER(_Grads), POINTER(_CameraGrads), c_int32, _ALLOC_FN,
                                              c_void_p, c_void_p]
    lib.gsb_alpha.restype = c_int32
    lib.gsb_alpha.argtypes = [c_int32, POINTER(_State), c_int32, c_int32, c_void_p, c_void_p]
    lib.gsb_backward_alpha.restype = c_int32
    lib.gsb_backward_alpha.argtypes = [POINTER(_Settings), POINTER(_Inputs), POINTER(_SplitSH), POINTER(_State), c_void_p, c_void_p,
                                       c_void_p, c_void_p, c_void_p, POINTER(_Grads), POINTER(_CameraGrads), c_int32, _ALLOC_FN,
                                       c_void_p, c_void_p]
    lib.gsb_backward_batch_alpha.restype = c_int32
    lib.gsb_backward_batch_alpha.argtypes = [c_int32, POINTER(_Settings), POINTER(_Inputs), POINTER(_State), c_void_p, c_void_p,
                                             c_void_p, c_void_p, c_void_p, POINTER(_Grads), POINTER(_CameraGrads),
                                             POINTER(_PeerTable), c_int32, c_int32, _CHUNK_FN, c_void_p, _ALLOC_FN, c_void_p,
                                             c_void_p]
    lib.gsb_render_features.restype = c_int32
    lib.gsb_render_features.argtypes = [c_int32, POINTER(_State), c_int32, c_int32, c_int32, c_int32, c_void_p, c_void_p, c_void_p]
    lib.gsb_contribution.restype = c_int32
    lib.gsb_contribution.argtypes = [c_int32, POINTER(_State), c_int32, c_int32, c_int32, c_void_p, c_void_p, c_void_p, c_void_p]
    lib.gsb_backward_features.restype = c_int32
    lib.gsb_backward_features.argtypes = [POINTER(_Settings), POINTER(_Inputs), POINTER(_SplitSH), POINTER(_State), c_void_p,
                                          c_void_p, c_void_p, c_void_p, c_void_p, POINTER(_Grads), POINTER(_CameraGrads),
                                          POINTER(_Features), c_int32, _ALLOC_FN, c_void_p, c_void_p]
    lib.gsb_backward_batch_features.restype = c_int32
    lib.gsb_backward_batch_features.argtypes = [c_int32, POINTER(_Settings), POINTER(_Inputs), POINTER(_State), c_void_p, c_void_p,
                                                c_void_p, c_void_p, c_void_p, POINTER(_Grads), POINTER(_CameraGrads),
                                                POINTER(_Features), POINTER(_PeerTable), c_int32, c_int32, _CHUNK_FN, c_void_p,
                                                _ALLOC_FN, c_void_p, c_void_p]
    lib.gsb_sparse_adam_step.restype = c_int32
    lib.gsb_sparse_adam_step.argtypes = [POINTER(_SparseAdamGroup), c_int32, c_void_p, c_int64, c_float, c_float, c_void_p]
    lib.gsb_forward_batch.restype = c_int32
    lib.gsb_forward_batch.argtypes = [c_int32, POINTER(_Settings), POINTER(_Inputs), c_void_p, c_void_p, c_void_p, c_int64,
                                      _ALLOC_FN, c_void_p, POINTER(_State), c_void_p]
    lib.gsb_backward_batch.restype = c_int32
    lib.gsb_backward_batch.argtypes = [c_int32, POINTER(_Settings), POINTER(_Inputs), POINTER(_State), c_void_p, c_void_p,
                                       c_void_p, c_void_p, POINTER(_Grads), c_int32, _ALLOC_FN, c_void_p, c_void_p]
    lib.gsb_forward_batch_async.restype = c_int32
    lib.gsb_forward_batch_async.argtypes = [c_int32, POINTER(_Settings), POINTER(_Inputs), c_void_p, c_void_p, c_void_p, c_int64,
                                            c_void_p, _ALLOC_FN, c_void_p, POINTER(_State), c_void_p]
    lib.gsb_backward_batch_chunked.restype = c_int32
    lib.gsb_backward_batch_chunked.argtypes = [c_int32, POINTER(_Settings), POINTER(_Inputs), POINTER(_State), c_void_p, c_void_p,
                                               c_void_p, c_void_p, POINTER(_Grads), c_int32, c_int32, _CHUNK_FN, c_void_p,
                                               _ALLOC_FN, c_void_p, c_void_p]
    lib.gsb_backward_batch_peer.restype = c_int32
    lib.gsb_backward_batch_peer.argtypes = [c_int32, POINTER(_Settings), POINTER(_Inputs), POINTER(_State), c_void_p, c_void_p,
                                            c_void_p, c_void_p, POINTER(_Grads), POINTER(_PeerTable), _ALLOC_FN, c_void_p, c_void_p]
    lib.gsb_enable_peer_access.restype = c_int32
    lib.gsb_enable_peer_access.argtypes = [c_int32]
    lib.gsb_peer_alloc.restype = c_int32
    lib.gsb_peer_alloc.argtypes = [c_size_t, POINTER(c_void_p), c_void_p]
    lib.gsb_peer_open.restype = c_int32
    lib.gsb_peer_open.argtypes = [c_void_p, POINTER(c_void_p)]
    lib.gsb_peer_close.restype = c_int32
    lib.gsb_peer_close.argtypes = [c_void_p]
    lib.gsb_peer_free.restype = c_int32
    lib.gsb_peer_free.argtypes = [c_void_p]
    lib.gsb_mark_visible.restype = c_int32
    lib.gsb_mark_visible.argtypes = [c_int32, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]
    lib.gsb_sort_pairs.restype = c_int32
    lib.gsb_sort_pairs.argtypes = [c_void_p, c_void_p, c_int64, c_int32, c_int32, _ALLOC_FN, c_void_p, c_void_p]
    lib.gsb_l1_loss_grad.restype = c_int32
    lib.gsb_l1_loss_grad.argtypes = [c_void_p, c_void_p, c_int64, c_float, c_void_p, c_void_p, c_void_p]
    lib.gsb_photometric_loss_grad.restype = c_int32
    lib.gsb_photometric_loss_grad.argtypes = [c_void_p, c_void_p, c_int32, c_int32, c_int32, c_float, c_int32, c_void_p, c_void_p,
                                              _ALLOC_FN, c_void_p, c_void_p]
    lib.gsb_last_error.restype = c_char_p
    lib.gsb_abi_version.restype = c_int32
    lib.gsb_launch_count.restype = c_int64
    lib.gsb_reset_launch_count.restype = None
    lib.gsb_kernel_time.restype = c_int32
    lib.gsb_kernel_time.argtypes = [c_char_p, POINTER(ctypes.c_double), POINTER(c_int64), c_int32]
    lib.gsb_set_option.restype = c_int32
    lib.gsb_set_option.argtypes = [c_char_p, c_int32]
    lib.gsb_set_deterministic.restype = c_int32
    lib.gsb_set_deterministic.argtypes = [c_int32]
    lib.gsb_adam_step.restype = c_int32
    lib.gsb_adam_step.argtypes = [POINTER(_AdamArgs), c_void_p]
    lib.gsb_activate.restype = c_int32
    lib.gsb_activate.argtypes = [c_int64, c_int32, c_void_p, c_void_p, c_void_p]
    lib.gsb_densify_scratch_bytes.restype = ctypes.c_size_t
    lib.gsb_densify_scratch_bytes.argtypes = [c_int64, c_int32]
    lib.gsb_densify_plan.restype = c_int32
    lib.gsb_densify_plan.argtypes = [POINTER(_DensifyArgs), POINTER(c_int64 * 4), c_void_p]
    lib.gsb_densify_apply.restype = c_int32
    lib.gsb_densify_apply.argtypes = [POINTER(_DensifyArgs), c_void_p, c_int64, c_int64, c_void_p, c_void_p, c_void_p, c_void_p]
    lib.gsb_prune_plan.restype = c_int32
    lib.gsb_prune_plan.argtypes = [c_int64, c_void_p, c_void_p, POINTER(c_int64), c_void_p]
    lib.gsb_prune_apply.restype = c_int32
    lib.gsb_prune_apply.argtypes = [c_int64, c_int32, c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_void_p, c_void_p, c_void_p,
                                    c_void_p]
    lib.gsb_knn_mean_dist2.restype = c_int32
    lib.gsb_knn_mean_dist2.argtypes = [c_void_p, c_int64, c_void_p, _ALLOC_FN, c_void_p, c_void_p]
    if lib.gsb_abi_version() != ABI_VERSION:
        raise ImportError(f"{_LIB_PATH}: ABI version {lib.gsb_abi_version()} != {ABI_VERSION} (rebuild: make -C gaussian-splatting_b200/csrc)")
    return lib


_C = _load()


def enable_peer_access(device, peer_device_index: int) -> None:
    """Kernels on `device` may dereference pointers into GPU `peer_device_index` afterwards (gsb_enable_peer_access)."""
    with _device_ctx(device):
        _check(_C.gsb_enable_peer_access(int(peer_device_index)))


def peer_alloc(device, nbytes: int):
    """(device pointer, 64-byte IPC handle) of a fresh zero-filled allocation on `device` (gsb_peer_alloc)."""
    ptr, handle = c_void_p(), ctypes.create_string_buffer(64)
    with _device_ctx(device):
        _check(_C.gsb_peer_alloc(int(nbytes), byref(ptr), handle))
    return int(ptr.value), bytes(handle.raw)


def peer_open(device, handle: bytes) -> int:
    """Maps another process's gsb_peer_alloc allocation for kernels running on `device`; returns the local address."""
    ptr, buf = c_void_p(), ctypes.create_string_buffer(handle, 64)
    with _device_ctx(device):
        _check(_C.gsb_peer_open(buf, byref(ptr)))
    return int(ptr.value)


def peer_close(device, ptr: int) -> None:
    with _device_ctx(device):
        _check(_C.gsb_peer_close(c_void_p(ptr)))


def peer_free(device, ptr: int) -> None:
    with _device_ctx(device):
        _check(_C.gsb_peer_free(c_void_p(ptr)))


def launch_count() -> int:
    """Kernels launched by libgs_b200.so in this process since the last reset."""
    return int(_C.gsb_launch_count())


def reset_launch_count() -> None:
    _C.gsb_reset_launch_count()


def set_option(name: str, value: int) -> None:
    if _C.gsb_set_option(name.encode(), int(value)) != 0:
        raise KeyError(name)


def kernel_time(name: str = "", reset: bool = False):
    """(total_ms, launches) of kernel `name` ("" = all) timed with CUDA events on the launching stream while
    option time_kernels was on."""
    ms, n = ctypes.c_double(0.0), c_int64(0)
    _C.gsb_kernel_time(name.encode(), byref(ms), byref(n), int(reset))
    return float(ms.value), int(n.value)


def state_views(pack: dict, height: int, width: int):
    """Typed views over the forward state buffers (layout: csrc/abi.cu carve_image / carve_binning); for tests
    and the benchmark's instance statistics."""
    npix = height * width
    al = lambda v: (v + 255) // 256 * 256
    img, binning, D = pack["image"], pack["binning"], pack["num_rendered"]
    final_T = img[:npix * 4].view(torch.float32).view(height, width)
    n_contrib = img[al(npix * 4):al(npix * 4) + npix * 4].view(torch.int32).view(height, width)
    pl_bytes = max(int(pack["state"].binning_capacity), 1) * 4
    point_list = binning[:D * 4].view(torch.int32)
    num_tiles = int(pack["state"].num_tiles)
    ranges = binning[al(pl_bytes):al(pl_bytes) + num_tiles * 8].view(torch.int32).view(num_tiles, 2)
    return dict(final_T=final_T, n_contrib=n_contrib, point_list=point_list, ranges=ranges)


def l1_loss_and_grad(image: torch.Tensor, target: torch.Tensor, loss_accum: Optional[torch.Tensor] = None,
                     grad_out: Optional[torch.Tensor] = None):
    """mean |clamp(image,0,1) - target| and its gradient w.r.t. `image`, in one kernel.  Returns (loss, grad);
    `loss` is `loss_accum` (a 1-element float32 tensor that is ADDED to) or a fresh scalar tensor; the gradient is written
    into `grad_out` when given (contiguous float32 of the image's shape: e.g. the slot render_views_backward offers)."""
    _require_cuda(image)
    img, gt = _f32c(image), _f32c(target)
    n = img.numel()
    if grad_out is not None and (grad_out.dtype != torch.float32 or not grad_out.is_contiguous() or grad_out.shape != img.shape):
        grad_out = None
    grad = grad_out if grad_out is not None else torch.empty_like(img)
    if loss_accum is None:
        loss_accum = torch.zeros(1, dtype=torch.float32, device=img.device)
    with _device_ctx(img.device):
        rc = _C.gsb_l1_loss_grad(img.data_ptr(), gt.data_ptr(), n, 1.0 / n, grad.data_ptr(), loss_accum.data_ptr(),
                                 _current_stream(img.device))
    _check(rc)
    return loss_accum, grad


def photometric_loss_and_grad(image: torch.Tensor, target: torch.Tensor, lambda_dssim: float = 0.2, clamp_input: bool = True,
                              grad_out: Optional[torch.Tensor] = None):
    """The reference training step's loss (train.py:120-126) fused with its gradient:
    ``(1 - lambda) * mean|x - y| + lambda * (1 - SSIM(x, y))`` with ``x = clamp(image, 0, 1)`` (render()'s clamp and its
    gradient mask; ``clamp_input=False``: x = image); image / target [C,H,W].
    Returns (loss[1], dloss/dimage, parts) with parts = tensor [loss, mean L1, mean SSIM] (device, no sync)."""
    _require_cuda(image)
    img, gt = _f32c(image), _f32c(target)
    C, H, W = (int(v) for v in img.shape[-3:])
    if grad_out is not None and (grad_out.dtype != torch.float32 or not grad_out.is_contiguous() or grad_out.shape != img.shape):
        grad_out = None
    grad = grad_out if grad_out is not None else torch.empty_like(img)
    # accumulators [loss - lambda, sum |x - y|, sum SSIM]: created on the device (a host-side tensor would be a pageable copy,
    # i.e. a host synchronisation in every training step)
    acc = torch.zeros(3, dtype=torch.float32, device=img.device)
    acc[:1] += float(lambda_dssim)
    with _device_ctx(img.device):
        stream = _current_stream(img.device)
        arena = _Arena(img.device, stream)
        rc = _C.gsb_photometric_loss_grad(img.data_ptr(), gt.data_ptr(), C, H, W, float(lambda_dssim), int(bool(clamp_input)),
                                          grad.data_ptr(), acc.data_ptr(), arena.cb, None, stream)
    _check(rc, arena)
    n = float(C * H * W)
    parts = torch.stack((acc[0], acc[1] / n, acc[2] / n))
    return acc[:1], grad, parts


# The three places where this layer touches the CUDA runtime.  The library has no CPU path: CPU tensors are refused here.
# (tests/host_emul swaps these three together with _C to drive a host build of the kernel SOURCES in the CPU test-suite.)
def _require_cuda(t: torch.Tensor) -> None:
    if not t.is_cuda:
        raise RuntimeError("diff_gaussian_rasterization (H100): tensors must live on a CUDA device; there is no CPU path "
                           "(no CPU fallback)")


def _current_stream(device) -> int:
    return torch.cuda.current_stream(device).cuda_stream


def _device_ctx(device):
    return torch.cuda.device(device)


def _stream_of(t: torch.Tensor):
    _require_cuda(t)
    return _current_stream(t.device)


def adam_step(params, grads, exp_avg, exp_avg_sq, act, P: int, sh_coeffs: int, step_size, beta1: float, beta2: float,
              eps: float, bias2_sqrt, visible: Optional[torch.Tensor] = None, skip_groups: int = 0) -> None:
    """gsb_adam_step over the flat store (layout: include/gs_b200.h); every tensor float32, contiguous, same device.
    ``step_size`` / ``bias2_sqrt``: six values (xyz, f_dc, f_rest, opacity, scaling, rotation; a scalar bias2_sqrt is
    broadcast); ``skip_groups``: bit mask of groups to leave untouched."""
    a = _AdamArgs()
    a.P, a.sh_coeffs, a.skip_groups = int(P), int(sh_coeffs), int(skip_groups)
    a.params, a.grads, a.exp_avg, a.exp_avg_sq = params.data_ptr(), grads.data_ptr(), exp_avg.data_ptr(), exp_avg_sq.data_ptr()
    a.act = act.data_ptr() if act is not None else None
    if visible is not None:
        visible = visible.to(torch.uint8).contiguous()
    a.visible = visible.data_ptr() if visible is not None else None
    a.step_size = (c_float * 6)(*[float(v) for v in step_size])
    b2 = [float(bias2_sqrt)] * 6 if isinstance(bias2_sqrt, (int, float)) else [float(v) for v in bias2_sqrt]
    a.bias2_sqrt = (c_float * 6)(*b2)
    a.beta1, a.beta2, a.eps = float(beta1), float(beta2), float(eps)
    stream = _stream_of(params)
    with _device_ctx(params.device):
        _check(_C.gsb_adam_step(byref(a), stream))


def sparse_adam_step(groups, visible: torch.Tensor, N: int, beta1: float = 0.9, beta2: float = 0.999) -> None:
    """gsb_sparse_adam_step: ONE launch over 1..MAX_SPARSE_GROUPS groups ``(param, grad, exp_avg, exp_avg_sq, lr, eps)``, each
    tensor [N, ...] float32 contiguous on the device of ``visible`` ([N] bool or uint8, contiguous).  Rows with visible == 0
    are left untouched.  No host synchronisation; the caller validates shapes (SparseGaussianAdam.step)."""
    if not 1 <= len(groups) <= MAX_SPARSE_GROUPS:
        raise ValueError(f"sparse_adam_step: {len(groups)} groups, 1..{MAX_SPARSE_GROUPS} per launch")
    N = int(N)
    if N == 0:
        return
    vis = visible.contiguous()
    vis = vis.view(torch.uint8) if vis.dtype == torch.bool else vis.to(torch.uint8)
    arr = (_SparseAdamGroup * len(groups))()
    for k, (p, g, m, v, lr, eps) in enumerate(groups):
        arr[k].param, arr[k].grad, arr[k].exp_avg, arr[k].exp_avg_sq = p.data_ptr(), g.data_ptr(), m.data_ptr(), v.data_ptr()
        arr[k].width, arr[k].lr, arr[k].eps = p.numel() // N, float(lr), float(eps)
    stream = _stream_of(vis)
    with _device_ctx(vis.device):
        _check(_C.gsb_sparse_adam_step(arr, len(groups), vis.data_ptr(), N, float(beta1), float(beta2), stream))


def activate(params: torch.Tensor, act: torch.Tensor, P: int, sh_coeffs: int) -> None:
    stream = _stream_of(params)
    with _device_ctx(params.device):
        _check(_C.gsb_activate(int(P), int(sh_coeffs), params.data_ptr(), act.data_ptr(), stream))


def densify_plan(params, exp_avg, exp_avg_sq, grad_accum, denom, P: int, sh_coeffs: int, n_children: int, grad_threshold: float,
                 size_limit: float, min_opacity: float, world_limit: float):
    """gsb_densify_plan: returns (args, scratch, (n_clone, n_split, n_pruned, P_new)); one stream synchronisation."""
    stream = _stream_of(params)
    a = _DensifyArgs()
    a.P, a.sh_coeffs, a.n_children = int(P), int(sh_coeffs), int(n_children)
    a.params, a.exp_avg, a.exp_avg_sq = params.data_ptr(), exp_avg.data_ptr(), exp_avg_sq.data_ptr()
    ga, dn = _f32c(grad_accum.reshape(-1)), _f32c(denom.reshape(-1))
    a.grad_accum, a.denom = ga.data_ptr(), dn.data_ptr()
    a.grad_threshold, a.size_limit = float(grad_threshold), float(size_limit)
    a.min_opacity, a.world_limit = float(min_opacity), float(world_limit)
    scratch = torch.empty(max(int(_C.gsb_densify_scratch_bytes(int(P), int(n_children))), 1), dtype=torch.uint8, device=params.device)
    a.scratch = scratch.data_ptr()
    counts = (c_int64 * 4)()
    with _device_ctx(params.device):
        _check(_C.gsb_densify_plan(byref(a), byref(counts), stream))
    return a, (scratch, ga, dn), tuple(int(v) for v in counts)


def densify_apply(args, unit_samples: Optional[torch.Tensor], n_split: int, P_new: int, new_params, new_exp_avg, new_exp_avg_sq) -> None:
    us = _f32c(unit_samples) if unit_samples is not None and unit_samples.numel() else None
    stream = _stream_of(new_params)
    with _device_ctx(new_params.device):
        _check(_C.gsb_densify_apply(byref(args), _ptr(us), int(n_split), int(P_new), new_params.data_ptr(), new_exp_avg.data_ptr(),
                                    new_exp_avg_sq.data_ptr(), stream))


def prune_plan(remove: torch.Tensor, P: int):
    """gsb_prune_plan: ``remove`` bool / uint8 [P] (True = the row goes).  Returns (scratch, P_new); one stream synchronisation."""
    stream = _stream_of(remove)
    rm = remove.reshape(-1)
    rm = (rm if rm.dtype == torch.uint8 else rm.to(torch.uint8)).contiguous()
    scratch = torch.empty(max(int(_C.gsb_densify_scratch_bytes(int(P), 1)), 1), dtype=torch.uint8, device=remove.device)
    P_new = c_int64(0)
    with _device_ctx(remove.device):
        _check(_C.gsb_prune_plan(int(P), rm.data_ptr() if P > 0 else None, scratch.data_ptr(), byref(P_new), stream))
    return scratch, int(P_new.value)


def prune_apply(scratch: torch.Tensor, P: int, sh_coeffs: int, params, exp_avg, exp_avg_sq, P_new: int, new_params, new_exp_avg,
                new_exp_avg_sq) -> None:
    """gsb_prune_apply: one gather of the rows gsb_prune_plan kept into the new store and both moments."""
    stream = _stream_of(params)
    with _device_ctx(params.device):
        _check(_C.gsb_prune_apply(int(P), int(sh_coeffs), params.data_ptr(), exp_avg.data_ptr(), exp_avg_sq.data_ptr(),
                                  scratch.data_ptr(), int(P_new), new_params.data_ptr(), new_exp_avg.data_ptr(),
                                  new_exp_avg_sq.data_ptr(), stream))


def knn_mean_dist2(points: torch.Tensor) -> torch.Tensor:
    """Mean squared distance of every point [P,3] to its three nearest other points (gsb_knn_mean_dist2; the replacement of
    simple_knn._C.distCUDA2, scene/gaussian_model.py:159)."""
    stream = _stream_of(points)
    if points.numel() == 0:
        return torch.empty(0, dtype=torch.float32, device=points.device)
    pts = _f32c(points.reshape(-1, 3))
    out = torch.empty(pts.shape[0], dtype=torch.float32, device=pts.device)
    with _device_ctx(pts.device):
        arena = _Arena(pts.device, stream)
        rc = _C.gsb_knn_mean_dist2(pts.data_ptr(), int(pts.shape[0]), out.data_ptr(), arena.cb, None, stream)
    _check(rc, arena)
    return out


class _Arena:
    """Hands torch-owned device memory to the library (torch caching allocator).

    State buffers (GEOM / BINNING / IMAGE) are fresh tensors: they live until the backward pass.  SCRATCH buffers
    are only used by kernels enqueued during the call, on the caller's stream, so one grow-only tensor per
    (device, stream, class) is reused across calls: stream order makes that safe, and it keeps the allocator out
    of the steady-state loop (view-dependent sizes otherwise keep triggering cudaMalloc for tens of steps)."""
    _scratch = {}

    def __init__(self, device, stream=None):
        self.device = device
        self.stream = stream
        self.bufs = {}
        self.error = None
        self.cb = _ALLOC_FN(self._alloc)

    def _alloc(self, _ctx, which, nbytes):
        try:
            which, nbytes = int(which), int(nbytes)
            if which >= 3 and self.stream is not None:
                key = (self.device.index, self.stream, which)
                t = _Arena._scratch.get(key)
                if t is None or t.numel() < nbytes:
                    t = torch.empty(max(nbytes, int(nbytes * 1.25)), dtype=torch.uint8, device=self.device)
                    _Arena._scratch[key] = t
            else:
                t = torch.empty(nbytes, dtype=torch.uint8, device=self.device)
            self.bufs[which] = t
            return t.data_ptr()
        except Exception as e:  # never let an exception cross the C ABI
            self.error = e
            return None


def release_scratch():
    """Drop the cached scratch buffers (e.g. before torch.cuda.empty_cache())."""
    _Arena._scratch.clear()


def _ptr(t: Optional[torch.Tensor]):
    return None if t is None else t.data_ptr()


def _f32c(t: Optional[torch.Tensor]) -> Optional[torch.Tensor]:
    if t is None or t.numel() == 0:
        return None
    if t.dtype != torch.float32:
        t = t.float()
    return t.contiguous()


def _check(rc: int, arena: Optional[_Arena] = None):
    if arena is not None:
        # The ctypes callback holds a bound method of the arena, the arena holds the callback: a reference cycle that would keep
        # every buffer of the call (hundreds of MB of state per step) alive until the cyclic garbage collector runs -- forcing
        # the caching allocator to cudaMalloc fresh segments meanwhile (a device-wide synchronisation, tens of ms).  The library
        # never calls back after the entry point has returned, so the cycle is cut here and everything frees by refcount.
        arena.cb = None
    if rc != 0:
        msg = _C.gsb_last_error().decode(errors="replace")
        if arena is not None and arena.error is not None:
            raise RuntimeError(f"libgs_b200: {msg}") from arena.error
        raise RuntimeError(f"libgs_b200 error {rc}: {msg}")


class GaussianRasterizationSettings(NamedTuple):
    image_height: int
    image_width: int
    tanfovx: float
    tanfovy: float
    bg: torch.Tensor
    scale_modifier: float
    viewmatrix: torch.Tensor
    projmatrix: torch.Tensor
    sh_degree: int
    campos: torch.Tensor
    prefiltered: bool
    debug: bool
    antialiasing: bool


def _c_settings(rs: GaussianRasterizationSettings, sh_coeffs: int, keep: list) -> _Settings:
    dev_t = [_f32c(rs.bg), _f32c(rs.viewmatrix), _f32c(rs.projmatrix), _f32c(rs.campos)]
    keep.extend(dev_t)
    s = _Settings()
    s.image_height = int(rs.image_height)
    s.image_width = int(rs.image_width)
    s.tanfovx = float(rs.tanfovx)
    s.tanfovy = float(rs.tanfovy)
    s.bg = _ptr(dev_t[0])
    s.scale_modifier = float(rs.scale_modifier)
    s.viewmatrix = _ptr(dev_t[1])
    s.projmatrix = _ptr(dev_t[2])
    s.sh_degree = int(rs.sh_degree)
    s.campos = _ptr(dev_t[3])
    s.prefiltered = int(bool(rs.prefiltered))
    s.debug = int(bool(rs.debug))
    s.antialiasing = int(bool(rs.antialiasing))
    s.sh_coeffs = int(sh_coeffs)
    return s


def _c_inputs(P, means3D, sh, colors, opac, scales, rots, cov) -> _Inputs:
    i = _Inputs()
    i.P = int(P)
    i.means3D, i.shs, i.colors_precomp, i.opacities = _ptr(means3D), _ptr(sh), _ptr(colors), _ptr(opac)
    i.scales, i.rotations, i.cov3D_precomp = _ptr(scales), _ptr(rots), _ptr(cov)
    return i


# instance-count estimate per (P, H, W): the previous call's count + 25 % (+64 Ki); see gsb_forward's capacity_hint
_capacity_hints = {}
speculative_binning = True


def _split_sh(dc, rest, grads: Optional[dict] = None) -> _SplitSH:
    sp = _SplitSH()
    sp.dc, sp.rest = _ptr(dc), _ptr(rest)
    if grads is not None:
        sp.dL_ddc, sp.dL_drest = _ptr(grads.get("dc")), _ptr(grads.get("shs"))
    return sp


def _forward_impl(means3D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp, rs, dc=None):
    """Returns (color, radii, invdepth, ctx_pack).  All tensor arguments already float32-contiguous or None.
    ``dc`` (split SH input, gsb_forward_split_sh): the DC rows [P,1,3]; ``sh`` is then the rest [P,M-1,3] or None."""
    _require_cuda(means3D)
    dev = means3D.device
    P = int(means3D.shape[0])
    H, W = int(rs.image_height), int(rs.image_width)
    M = int(sh.shape[1]) if sh is not None else 0
    if dc is not None:
        M += 1
    with _device_ctx(dev):
        keep = []
        cs = _c_settings(rs, M, keep)
        ci = _c_inputs(P, means3D, sh if dc is None else None, colors_precomp, opacities, scales, rotations, cov3Ds_precomp)
        color = torch.empty((3, H, W), dtype=torch.float32, device=dev)
        radii = torch.empty((P,), dtype=torch.int32, device=dev)
        invdepth = torch.empty((1, H, W), dtype=torch.float32, device=dev)
        stream = _current_stream(dev)
        arena = _Arena(dev, stream)
        st = _State()
        hkey = (P, H, W, dev.index)
        hint = _capacity_hints.get(hkey, 0) if speculative_binning else 0
        if dc is None:
            rc = _C.gsb_forward(byref(cs), byref(ci), color.data_ptr(), radii.data_ptr(), invdepth.data_ptr(), hint,
                                arena.cb, None, byref(st), stream)
        else:
            sp = _split_sh(dc, sh)
            rc = _C.gsb_forward_split_sh(byref(cs), byref(ci), byref(sp), color.data_ptr(), radii.data_ptr(), invdepth.data_ptr(),
                                         hint, arena.cb, None, byref(st), stream)
        _check(rc, arena)
        # next estimate: this count + 25 %, rounded up to 1 Mi instances and never shrinking, so that buffer sizes
        # settle after the first few views instead of following every view's own count
        _capacity_hints[hkey] = max(capacity_for(st.num_rendered), _capacity_hints.get(hkey, 0))
    pack = dict(state=st, geom=arena.bufs.get(BUF_GEOM), binning=arena.bufs.get(BUF_BINNING),
                image=arena.bufs.get(BUF_IMAGE), num_rendered=int(st.num_rendered), sh_coeffs=M)
    return color, radii, invdepth, pack


def _alpha_impl(states, height: int, width: int, device) -> torch.Tensor:
    """Rendered alpha (1 - final transmittance, gsb_alpha) of the forward states ``states`` (a ``_State`` or a ctypes array of
    them, e.g. a pack's "state" / "states"): [V,1,H,W] for an array, [1,H,W] for one state.  One launch, no synchronisation."""
    one = isinstance(states, _State)
    V = 1 if one else len(states)
    out = torch.empty((V, 1, int(height), int(width)), dtype=torch.float32, device=device)
    with _device_ctx(device):
        rc = _C.gsb_alpha(V, byref(states) if one else states, int(height), int(width), out.data_ptr(), _current_stream(device))
    _check(rc)
    return out[0] if one else out


def check_features(features, P: int, device) -> None:
    """Raises ValueError unless ``features`` is a [P, C] tensor with 1 <= C <= MAX_FEATURE_CHANNELS on ``device``."""
    if not isinstance(features, torch.Tensor) or features.dim() != 2:
        raise ValueError(f"features must be a 2-D tensor [P, C]; got {type(features).__name__} "
                         f"{tuple(features.shape) if isinstance(features, torch.Tensor) else ''}")
    if int(features.shape[0]) != int(P):
        raise ValueError(f"features has {int(features.shape[0])} rows, the gaussians number {int(P)}")
    if not 1 <= int(features.shape[1]) <= MAX_FEATURE_CHANNELS:
        raise ValueError(f"features has {int(features.shape[1])} channels, 1..{MAX_FEATURE_CHANNELS} are supported")
    if features.device != torch.device(device):
        raise ValueError(f"features live on {features.device}, the gaussians on {device}")


def _features_impl(states, height: int, width: int, features: torch.Tensor, device) -> torch.Tensor:
    """Rendered feature maps (gsb_render_features) of the forward states ``states`` (a ``_State`` or a ctypes array of them) for
    ``features`` [P, C] float32 contiguous: [V,C,H,W] for an array, [C,H,W] for one state.  One launch, no synchronisation."""
    one = isinstance(states, _State)
    V = 1 if one else len(states)
    P, C = int(features.shape[0]), int(features.shape[1])
    out = torch.empty((V, C, int(height), int(width)), dtype=torch.float32, device=device)
    with _device_ctx(device):
        rc = _C.gsb_render_features(V, byref(states) if one else states, int(height), int(width), P, C,
                                    features.data_ptr() if P > 0 else None, out.data_ptr(), _current_stream(device))
    _check(rc)
    return out[0] if one else out


class ContributionStats:
    """Per-gaussian contribution statistics of forward passes (gsb_contribution; definition in include/gs_b200.h), accumulated
    over every view and call they are handed to (``contrib=`` of rasterize_gaussians / GaussianRasterizer / render /
    render_views_backward):

    * ``count`` int64 [P]: the number of (pixel, gaussian) pairs the forward blended;
    * ``weight_sum`` float32 [P]: the sum of their blend weights alpha * T;
    * ``weight_max`` float32 [P]: the largest of those weights, 0 for a gaussian that was never blended.

    The usage scores of contribution-based pruning (sum of weights, max weight, pixel count).  Starts at zero; ``zero_()``
    starts over.  A ``prune_points`` makes the statistics stale: take a new object for the new gaussians."""

    def __init__(self, P: int, device):
        self.P = int(P)
        self.device = torch.device(device)
        self.count = torch.zeros(self.P, dtype=torch.int64, device=self.device)
        self.weight_sum = torch.zeros(self.P, dtype=torch.float32, device=self.device)
        self.weight_max = torch.zeros(self.P, dtype=torch.float32, device=self.device)

    def zero_(self):
        self.count.zero_()
        self.weight_sum.zero_()
        self.weight_max.zero_()
        return self


def check_contrib(contrib, P: int, device) -> None:
    """Raises ValueError unless ``contrib`` is a ContributionStats of P gaussians on ``device`` with intact tensors."""
    if not isinstance(contrib, ContributionStats):
        raise ValueError(f"contrib must be a ContributionStats; got {type(contrib).__name__}")
    want = {"count": torch.int64, "weight_sum": torch.float32, "weight_max": torch.float32}
    for name, dtype in want.items():
        t = getattr(contrib, name)
        if not isinstance(t, torch.Tensor) or t.dtype != dtype or t.dim() != 1 or not t.is_contiguous():
            raise ValueError(f"contrib.{name} must be a contiguous 1-D {dtype} tensor")
        if int(t.shape[0]) != int(P):
            raise ValueError(f"contrib.{name} has {int(t.shape[0])} entries, the gaussians number {int(P)}")
        if t.device != torch.device(device):
            raise ValueError(f"contrib.{name} lives on {t.device}, the gaussians on {device}")


def _contrib_impl(states, height: int, width: int, P: int, contrib: ContributionStats, device) -> None:
    """Adds the contribution statistics of the forward states ``states`` (a ``_State`` or a ctypes array of them) into
    ``contrib``.  One launch (none for P == 0), no synchronisation."""
    _deterministic("contrib= (the float-atomic weight_sum of gsb_contribution)")
    one = isinstance(states, _State)
    V = 1 if one else len(states)
    with _device_ctx(device):
        rc = _C.gsb_contribution(V, byref(states) if one else states, int(height), int(width), int(P),
                                 contrib.count.data_ptr(), contrib.weight_sum.data_ptr(), contrib.weight_max.data_ptr(),
                                 _current_stream(device))
    _check(rc)


def _deterministic(what: Optional[str] = None) -> bool:
    """Whether the backward that follows must be deterministic: torch's ``use_deterministic_algorithms`` flag.  ``what`` names
    a path with no deterministic implementation; under the flag it raises RuntimeError as torch's own such operations do, or
    warns and takes the default path (returns False) with ``warn_only=True``."""
    if not torch.are_deterministic_algorithms_enabled():
        return False
    if what is None:
        return True
    msg = (f"{what} does not have a deterministic implementation, but you set 'torch.use_deterministic_algorithms(True)'. "
           f"You can turn off determinism just for this operation, or you can use the 'warn_only=True' option, if that's "
           f"acceptable for your application.")
    if not torch.is_deterministic_algorithms_warn_only_enabled():
        raise RuntimeError(msg)
    warnings.warn(msg)
    return False


def _feature_term(feats: Optional[dict]):
    """GsbFeatures over ``feats`` = {"features": [P,C], "out": forward output, "grad": dL/d output or None, "dL_dfeatures":
    [P,C] or None}, all float32 contiguous; None for no feature term."""
    if feats is None:
        return None
    f = feats["features"]
    ft = _Features()
    ft.channels = int(f.shape[1])
    ft.features = f.data_ptr() if f.numel() > 0 else None
    ft.out_features = feats["out"].data_ptr()
    ft.dL_dout_features = _ptr(feats.get("grad"))
    d = feats.get("dL_dfeatures")
    ft.dL_dfeatures = d.data_ptr() if d is not None and d.numel() > 0 else None
    return ft


CAMERA_KEYS = ("viewmatrix", "projmatrix", "campos", "bg")     # GsbCameraGrads, in field order
_CAMERA_NUMEL = dict(viewmatrix=16, projmatrix=16, campos=3, bg=3)


def _camera_grads(cam_grads: Optional[dict], V: Optional[int] = None):
    """GsbCameraGrads over the float32 contiguous tensors of ``cam_grads`` (keys CAMERA_KEYS, missing / None = not requested),
    each [16] / [3] per view ([V,16] / [V,3] for the view batch); None when nothing is requested."""
    if not cam_grads or all(cam_grads.get(k) is None for k in CAMERA_KEYS):
        return None
    cg = _CameraGrads()
    for k in CAMERA_KEYS:
        t = cam_grads.get(k)
        if t is None:
            continue
        n = _CAMERA_NUMEL[k] * (1 if V is None else V)
        if t.dtype != torch.float32 or not t.is_contiguous() or t.numel() != n:
            raise ValueError(f"camera gradient '{k}': contiguous float32 tensor of {n} elements expected, got "
                             f"{t.dtype} {tuple(t.shape)}")
        setattr(cg, "dL_d" + k, t.data_ptr())
    return cg


def _backward_impl(pack, rs, means3D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp,
                   out_color, out_invdepth, grad_color, grad_invdepth, grads: dict, accumulate: bool,
                   accumulate_means2D: Optional[bool] = None, dc=None, cam_grads: Optional[dict] = None,
                   grad_alpha: Optional[torch.Tensor] = None, feats: Optional[dict] = None):
    """grads: tensors to fill (accumulate=False) or add into (accumulate=True).  The C ABI has one accumulate
    switch; a per-view means2D buffer (accumulate_means2D=False while the rest accumulates) is zeroed here.
    ``dc``: split SH input (gsb_backward_split_sh); ``sh`` is the rest, grads["dc"] / grads["shs"] receive their gradients.
    ``cam_grads``: {"viewmatrix": [16], "projmatrix": [16], "campos": [3], "bg": [3]} float32 tensors (any subset) that receive
    the camera gradient under the same accumulate switch (gsb_backward_camera).  ``grad_alpha``: dL/d rendered alpha [1,H,W]
    float32 contiguous, or None (gsb_backward_alpha; None takes the calls above).  ``feats``: the feature term (_feature_term;
    gsb_backward_features), or None."""
    if accumulate and accumulate_means2D is False and grads.get("means2D") is not None:
        grads["means2D"].zero_()
    dev = means3D.device
    P = int(means3D.shape[0])
    with _device_ctx(dev):
        keep = []
        cs = _c_settings(rs, pack["sh_coeffs"], keep)
        ci = _c_inputs(P, means3D, sh if dc is None else None, colors_precomp, opacities, scales, rotations, cov3Ds_precomp)
        g = _Grads()
        g.dL_dmeans3D, g.dL_dmeans2D = _ptr(grads.get("means3D")), _ptr(grads.get("means2D"))
        g.dL_dshs, g.dL_dcolors = _ptr(grads.get("shs")) if dc is None else None, _ptr(grads.get("colors_precomp"))
        g.dL_dopacities = _ptr(grads.get("opacities"))
        g.dL_dscales, g.dL_drotations = _ptr(grads.get("scales")), _ptr(grads.get("rotations"))
        g.dL_dcov3D = _ptr(grads.get("cov3D_precomp"))
        stream = _current_stream(dev)
        arena = _Arena(dev, stream)
        cg = _camera_grads(cam_grads)
        ft = _feature_term(feats)
        det = _deterministic("the feature-map backward (features= with a loss on the map)"
                             if ft is not None and ft.dL_dout_features and P > 0 else None)
        _C.gsb_set_deterministic(int(det))
        if ft is not None:
            sp = _split_sh(dc, sh, grads) if dc is not None else None
            rc = _C.gsb_backward_features(byref(cs), byref(ci), byref(sp) if sp is not None else None, byref(pack["state"]),
                                          out_color.data_ptr(), out_invdepth.data_ptr(), grad_color.data_ptr(), _ptr(grad_invdepth),
                                          _ptr(grad_alpha), byref(g), byref(cg) if cg is not None else None, byref(ft),
                                          int(bool(accumulate)), arena.cb, None, stream)
        elif grad_alpha is not None:
            sp = _split_sh(dc, sh, grads) if dc is not None else None
            rc = _C.gsb_backward_alpha(byref(cs), byref(ci), byref(sp) if sp is not None else None, byref(pack["state"]),
                                       out_color.data_ptr(), out_invdepth.data_ptr(), grad_color.data_ptr(), _ptr(grad_invdepth),
                                       grad_alpha.data_ptr(), byref(g), byref(cg) if cg is not None else None,
                                       int(bool(accumulate)), arena.cb, None, stream)
        elif cg is not None:
            sp = _split_sh(dc, sh, grads) if dc is not None else None
            rc = _C.gsb_backward_camera(byref(cs), byref(ci), byref(sp) if sp is not None else None, byref(pack["state"]),
                                        out_color.data_ptr(), out_invdepth.data_ptr(), grad_color.data_ptr(), _ptr(grad_invdepth),
                                        byref(g), byref(cg), int(bool(accumulate)), arena.cb, None, stream)
        elif dc is None:
            rc = _C.gsb_backward(byref(cs), byref(ci), byref(pack["state"]), out_color.data_ptr(), out_invdepth.data_ptr(),
                                 grad_color.data_ptr(), _ptr(grad_invdepth), byref(g), int(bool(accumulate)), arena.cb,
                                 None, stream)
        else:
            sp = _split_sh(dc, sh, grads)
            rc = _C.gsb_backward_split_sh(byref(cs), byref(ci), byref(sp), byref(pack["state"]), out_color.data_ptr(),
                                          out_invdepth.data_ptr(), grad_color.data_ptr(), _ptr(grad_invdepth), byref(g),
                                          int(bool(accumulate)), arena.cb, None, stream)
        _check(rc, arena)


MAX_BATCH_VIEWS = 16


def _forward_batch_impl(means3D, sh, opacities, scales, rotations, settings_list, async_counts: Optional[torch.Tensor] = None,
                        capacity: int = 0):
    """View-batch forward (gsb_forward_batch): returns (color[V,3,H,W], radii[V,P], invdepth[V,1,H,W], pack).

    ``async_counts`` (int64 device tensor of COUNT_SLOTS elements) switches to gsb_forward_batch_async: no host
    synchronisation; ``capacity`` instances per view are final, the counts and their running maximum stay on the device
    (the caller polls ``async_counts[16]`` later: gaussian_renderer.AsyncCapacity)."""
    _require_cuda(means3D)
    dev = means3D.device
    V, P = len(settings_list), int(means3D.shape[0])
    H, W = int(settings_list[0].image_height), int(settings_list[0].image_width)
    M = int(sh.shape[1])
    with _device_ctx(dev):
        keep = []
        cs = (_Settings * V)(*[_c_settings(rs, M, keep) for rs in settings_list])
        ci = _c_inputs(P, means3D, sh, None, opacities, scales, rotations, None)
        color = torch.empty((V, 3, H, W), dtype=torch.float32, device=dev)
        radii = torch.empty((V, P), dtype=torch.int32, device=dev)
        invdepth = torch.empty((V, 1, H, W), dtype=torch.float32, device=dev)
        stream = _current_stream(dev)
        arena = _Arena(dev, stream)
        states = (_State * V)()
        if async_counts is not None:
            if async_counts.dtype != torch.int64 or async_counts.numel() < COUNT_SLOTS or not async_counts.is_contiguous():
                raise ValueError("async_counts: contiguous int64 tensor of COUNT_SLOTS elements on the gaussians' device")
            rc = _C.gsb_forward_batch_async(V, cs, byref(ci), color.data_ptr(), radii.data_ptr(), invdepth.data_ptr(), int(capacity),
                                            async_counts.data_ptr(), arena.cb, None, states, stream)
            _check(rc, arena)
        else:
            hkey = (P, H, W, dev.index, "batch")
            hint = _capacity_hints.get(hkey, 0) if speculative_binning else 0
            rc = _C.gsb_forward_batch(V, cs, byref(ci), color.data_ptr(), radii.data_ptr(), invdepth.data_ptr(), hint, arena.cb,
                                      None, states, stream)
            _check(rc, arena)
            dmax = max(int(states[v].num_rendered) for v in range(V))
            _capacity_hints[hkey] = max(capacity_for(dmax), _capacity_hints.get(hkey, 0))
    pack = dict(states=states, V=V, geom=arena.bufs.get(BUF_GEOM), binning=arena.bufs.get(BUF_BINNING),
                image=arena.bufs.get(BUF_IMAGE), num_rendered=[int(states[v].num_rendered) for v in range(V)], sh_coeffs=M,
                keep=keep)
    return color, radii, invdepth, pack


def capacity_for(count: int) -> int:
    """Instance capacity for an observed per-view count: + 25 %, + 64 Ki, rounded up to 1 Mi."""
    return ((int(count * 1.25) + 65536 + (1 << 20) - 1) >> 20) << 20


def _backward_batch_impl(pack, settings_list, means3D, sh, opacities, scales, rotations, out_color, out_invdepth,
                         grad_color, grad_invdepth, grads: dict, accumulate: bool, n_chunks: int = 1, on_chunk=None, peers=None,
                         cam_grads: Optional[dict] = None, grad_alpha: Optional[torch.Tensor] = None,
                         feats: Optional[dict] = None):
    """View-batch backward (gsb_backward_batch).  grads: tensors holding / receiving the gradient SUMMED over the views
    (means2D, if present, is [V,P,3] and per view).  ``n_chunks`` > 1: gsb_backward_batch_chunked -- the last kernel runs in
    gaussian-range chunks and ``on_chunk(chunk, p_begin, p_end)`` is called after each chunk has been enqueued (rows
    [p_begin, p_end) of every gradient are final in stream order from there on).  ``peers`` = (world, rank, rows_per_rank,
    [base pointers]): gsb_backward_batch_peer -- the gradients are ADDED into the owner ranks' buffers (fused reduce-scatter;
    gaussian_renderer.peer.PeerGradientBucket drives the protocol around it).  ``cam_grads``: {"viewmatrix": [V,16],
    "projmatrix": [V,16], "campos": [V,3], "bg": [V,3]} float32 tensors (any subset) receiving each view's camera gradient
    (gsb_backward_batch_camera); not with ``n_chunks`` > 1, ``on_chunk`` or ``peers``.  ``grad_alpha``: dL/d rendered alpha
    [V,1,H,W] float32 contiguous, or None; with it every mode goes through gsb_backward_batch_alpha.  ``feats``: the feature
    term (_feature_term over [V,C,H,W] maps; gsb_backward_batch_features), plain and camera modes only."""
    dev = means3D.device
    V, P = pack["V"], int(means3D.shape[0])
    cg = _camera_grads(cam_grads, V)
    if cg is not None and (peers is not None or n_chunks > 1 or on_chunk is not None):
        raise ValueError("camera gradients are not available on the chunked or peer view-batch backward: the per-view sum "
                         "would have to span gaussian chunks or ranks")
    ft = _feature_term(feats)
    if ft is not None and (peers is not None or n_chunks > 1 or on_chunk is not None):
        raise ValueError("features are not available on the chunked or peer view-batch backward")
    with _device_ctx(dev):
        keep = []
        cs = (_Settings * V)(*[_c_settings(rs, pack["sh_coeffs"], keep) for rs in settings_list])
        ci = _c_inputs(P, means3D, sh, None, opacities, scales, rotations, None)
        g = _Grads()
        g.dL_dmeans3D, g.dL_dmeans2D = _ptr(grads.get("means3D")), _ptr(grads.get("means2D"))
        g.dL_dshs, g.dL_dopacities = _ptr(grads.get("shs")), _ptr(grads.get("opacities"))
        g.dL_dscales, g.dL_drotations = _ptr(grads.get("scales")), _ptr(grads.get("rotations"))
        stream = _current_stream(dev)
        arena = _Arena(dev, stream)
        pt = None
        if peers is not None:
            world, rank, rows_per_rank, bases = peers
            pt = _PeerTable()
            pt.world, pt.rank, pt.rows_per_rank, pt.reserved = int(world), int(rank), int(rows_per_rank), 0
            pt.base = (c_void_p * 16)(*([int(b) for b in bases] + [None] * (16 - len(bases))))
        if ft is not None and ft.dL_dout_features:
            det = _deterministic("the feature-map backward (features= with a loss on the map)")
        elif pt is not None:
            det = _deterministic("the peer gradient reduce-scatter (peers=)")
        else:
            det = _deterministic()
        _C.gsb_set_deterministic(int(det))
        err = []

        def _cb(_ctx, chunk, p0, p1):
            try:
                if on_chunk is not None and not err:
                    on_chunk(int(chunk), int(p0), int(p1))
            except Exception as e:  # never let an exception cross the C ABI
                err.append(e)
        if ft is not None:
            rc = _C.gsb_backward_batch_features(V, cs, byref(ci), pack["states"], out_color.data_ptr(), out_invdepth.data_ptr(),
                                                grad_color.data_ptr(), _ptr(grad_invdepth), _ptr(grad_alpha), byref(g),
                                                byref(cg) if cg is not None else None, byref(ft), None, int(bool(accumulate)), 1,
                                                _CHUNK_FN(), None, arena.cb, None, stream)
            _check(rc, arena)
        elif grad_alpha is not None:
            chunked = pt is None and (n_chunks > 1 or on_chunk is not None)
            cb = _CHUNK_FN(_cb) if chunked else _CHUNK_FN()     # NULL callback
            rc = _C.gsb_backward_batch_alpha(V, cs, byref(ci), pack["states"], out_color.data_ptr(), out_invdepth.data_ptr(),
                                             grad_color.data_ptr(), _ptr(grad_invdepth), grad_alpha.data_ptr(), byref(g),
                                             byref(cg) if cg is not None else None, byref(pt) if pt is not None else None,
                                             int(bool(accumulate)), int(n_chunks) if chunked else 1, cb, None, arena.cb, None, stream)
            _check(rc, arena)
            if err:
                raise err[0]
        elif pt is not None:
            rc = _C.gsb_backward_batch_peer(V, cs, byref(ci), pack["states"], out_color.data_ptr(), out_invdepth.data_ptr(),
                                            grad_color.data_ptr(), _ptr(grad_invdepth), byref(g), byref(pt), arena.cb, None, stream)
            _check(rc, arena)
        elif n_chunks > 1 or on_chunk is not None:
            cb = _CHUNK_FN(_cb)
            rc = _C.gsb_backward_batch_chunked(V, cs, byref(ci), pack["states"], out_color.data_ptr(), out_invdepth.data_ptr(),
                                               grad_color.data_ptr(), _ptr(grad_invdepth), byref(g), int(bool(accumulate)),
                                               int(n_chunks), cb, None, arena.cb, None, stream)
            _check(rc, arena)
            if err:
                raise err[0]
        elif cg is not None:
            rc = _C.gsb_backward_batch_camera(V, cs, byref(ci), pack["states"], out_color.data_ptr(), out_invdepth.data_ptr(),
                                              grad_color.data_ptr(), _ptr(grad_invdepth), byref(g), byref(cg),
                                              int(bool(accumulate)), arena.cb, None, stream)
            _check(rc, arena)
        else:
            rc = _C.gsb_backward_batch(V, cs, byref(ci), pack["states"], out_color.data_ptr(), out_invdepth.data_ptr(),
                                       grad_color.data_ptr(), _ptr(grad_invdepth), byref(g), int(bool(accumulate)), arena.cb, None,
                                       stream)
            _check(rc, arena)


def rasterize_gaussians(means3D, means2D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp,
                        raster_settings, dc=None, return_alpha=False, features=None, contrib=None):
    """``dc`` (optional): split SH input -- ``dc`` [P,1,3] holds the DC coefficient and ``sh`` [P,M-1,3] the others (M-1 may
    be 0); the result equals that of ``sh = cat((dc, sh), 1)`` without the concatenation.

    Camera gradients: when grad mode is on and any of ``raster_settings.viewmatrix`` / ``.projmatrix`` / ``.campos`` / ``.bg``
    requires grad, the four tensors become trailing inputs of the autograd function and those that require grad receive
    their gradient (gsb_backward_camera; conventions in include/gs_b200.h).  Otherwise the call is exactly the plain one.

    ``return_alpha=True``: the result is (color, radii, invdepth, alpha[1,H,W]) with alpha = 1 - final transmittance (gsb_alpha;
    definition in include/gs_b200.h), differentiable w.r.t. every gaussian input and the camera tensors.  One extra launch in the
    forward; a backward in which alpha's gradient is unused (None) is the plain one.

    ``features`` [P, C] (1 <= C <= MAX_FEATURE_CHANNELS, view-independent): one more trailing output, the feature map [C,H,W]
    = sum_k alpha_k T_k features[k] with the forward's blend weights and background 0 (gsb_render_features; definition in
    include/gs_b200.h).  Its gradient reaches ``features`` and every gaussian and camera input.  One extra launch in the forward,
    one in a backward that uses the map's gradient; without ``features`` the call is unchanged.  Bad shapes raise ValueError.

    ``contrib`` (a ContributionStats of P gaussians on the gaussians' device): the forward's per-gaussian contribution
    statistics are added into it (gsb_contribution; one extra launch in the forward, outputs and gradients unchanged; also under
    torch.no_grad()).  A wrong P, device or dtype raises ValueError."""
    if features is not None:
        check_features(features, int(means3D.shape[0]), means3D.device)
    if contrib is not None:
        check_contrib(contrib, int(means3D.shape[0]), means3D.device)
    return _RasterizeGaussians.apply(means3D, means2D, sh, colors_precomp, opacities, scales, rotations,
                                     cov3Ds_precomp, raster_settings, dc, bool(return_alpha), features, contrib,
                                     *_camera_inputs(raster_settings))


def _camera_inputs(rs) -> tuple:
    """(viewmatrix, projmatrix, campos, bg) of the settings if grad mode is on and one of them requires grad, else ()."""
    cams = tuple(getattr(rs, k) for k in CAMERA_KEYS)
    if torch.is_grad_enabled() and any(isinstance(t, torch.Tensor) and t.requires_grad for t in cams):
        return cams
    return ()


class _RasterizeGaussians(torch.autograd.Function):
    @staticmethod
    def forward(ctx, means3D, means2D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp,
                raster_settings, dc=None, return_alpha=False, features=None, contrib=None, *camera):
        # camera: the settings' (viewmatrix, projmatrix, campos, bg) as inputs of their own (rasterize_gaussians), or ()
        args = [_f32c(means3D), _f32c(sh), _f32c(colors_precomp), _f32c(opacities), _f32c(scales), _f32c(rotations),
                _f32c(cov3Ds_precomp)]
        if args[0] is None:  # P == 0
            args[0] = means3D.float().contiguous()
        dcc = _f32c(dc)       # None also when P == 0: nothing to stage, the joint call renders the background
        if dcc is not None and dcc.numel() != 3 * int(args[0].shape[0]):
            raise ValueError(f"dc must hold one RGB coefficient per gaussian ([P,1,3]); got shape {tuple(dc.shape)}")
        try:
            color, radii, invdepth, pack = _forward_impl(*args, raster_settings, dc=dcc)
        except Exception:
            if raster_settings.debug:
                dump = args + ([dcc] if dc is not None else []) + ([features] if features is not None else [])
                torch.save([a.detach().cpu() if a is not None else None for a in dump], "snapshot_fw.dump")
                print("\nAn error occured in forward. Writing snapshot_fw.dump for debugging.")
            raise
        ctx.set_materialize_grads(False)   # an unused inverse-depth output reaches backward as None, not zeros
        ctx.raster_settings = raster_settings
        ctx.pack = pack
        ctx.shapes = dict(means2D=None if means2D is None else tuple(means2D.shape), opacities=tuple(opacities.shape),
                          sh=None if sh is None else tuple(sh.shape), dc=None if dc is None else tuple(dc.shape))
        H, W = int(raster_settings.image_height), int(raster_settings.image_width)
        fc = fmap = None
        if features is not None:
            fc = features.detach().float().contiguous()
            fmap = _features_impl(pack["state"], H, W, fc, color.device)
        if contrib is not None:
            _contrib_impl(pack["state"], H, W, int(args[0].shape[0]), contrib, color.device)
        ctx.save_for_backward(*[a if a is not None else torch.empty(0) for a in args], color, invdepth,
                              dcc if dcc is not None else torch.empty(0), *((fc, fmap) if fc is not None else ()))
        ctx.mark_non_differentiable(radii)
        ctx.camera = [(tuple(t.shape), t.dtype) for t in camera]
        ctx.return_alpha = bool(return_alpha)
        ctx.has_features = features is not None
        out = (color, radii, invdepth)
        if return_alpha:
            out += (_alpha_impl(pack["state"], H, W, color.device),)
        if features is not None:
            out += (fmap,)
        return out

    @staticmethod
    def backward(ctx, grad_out_color, _grad_radii, grad_out_depth, *grad_extra):
        # grad_extra: the gradients of the optional outputs, (alpha)? (features)?
        grad_out_alpha = grad_extra[0] if ctx.return_alpha else None
        grad_out_feat = grad_extra[-1] if ctx.has_features else None
        rs = ctx.raster_settings
        saved = [t if t.numel() > 0 else None for t in ctx.saved_tensors[:7]]
        means3D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp = saved
        out_color, out_invdepth = ctx.saved_tensors[7], ctx.saved_tensors[8]
        dc = ctx.saved_tensors[9] if ctx.saved_tensors[9].numel() > 0 else None
        if means3D is None:
            means3D = ctx.saved_tensors[0]
        dev = means3D.device
        P = int(means3D.shape[0])
        new = lambda *shape: torch.empty(shape, dtype=torch.float32, device=dev)
        grads = dict(means3D=new(P, 3), means2D=new(P, 3), opacities=new(P))
        if sh is not None:
            grads["shs"] = new(*sh.shape)
        if ctx.shapes["dc"] is not None:
            grads["dc"] = new(*ctx.shapes["dc"])
            if sh is None and ctx.shapes["sh"] is not None:     # rest without coefficients (SH degree 0 model)
                grads["shs"] = torch.zeros(ctx.shapes["sh"], dtype=torch.float32, device=dev)
        if colors_precomp is not None:
            grads["colors_precomp"] = new(P, 3)
        if cov3Ds_precomp is not None:
            grads["cov3D_precomp"] = new(P, 6)
        else:
            grads["scales"] = new(P, 3)
            grads["rotations"] = new(P, 4)
        cam_grads = {k: torch.empty(_CAMERA_NUMEL[k], dtype=torch.float32, device=dev)
                     for j, k in enumerate(CAMERA_KEYS) if ctx.camera and ctx.needs_input_grad[13 + j]}
        if grad_out_color is None and grad_out_depth is None and grad_out_alpha is None and grad_out_feat is None:
            return (None,) * (13 + len(ctx.camera))
        gc = _f32c(grad_out_color)
        if gc is None:
            gc = torch.zeros((3, int(rs.image_height), int(rs.image_width)), dtype=torch.float32, device=dev)
        gd = _f32c(grad_out_depth)
        ga = _f32c(grad_out_alpha)
        if dc is None and "dc" in grads:                         # P == 0
            grads["dc"].zero_()
        feats = None
        if grad_out_feat is not None:
            fc, fmap = ctx.saved_tensors[10], ctx.saved_tensors[11]
            feats = dict(features=fc, out=fmap, grad=_f32c(grad_out_feat),
                         dL_dfeatures=torch.empty(fc.shape, dtype=torch.float32, device=dev) if ctx.needs_input_grad[11] else None)
        try:
            _backward_impl(ctx.pack, rs, means3D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp,
                           out_color, out_invdepth, gc, gd, grads, accumulate=False, dc=dc, cam_grads=cam_grads, grad_alpha=ga,
                           feats=feats)
        except Exception:
            if rs.debug:
                split = [ctx.saved_tensors[9].cpu()] if ctx.shapes["dc"] is not None else []
                camera = [getattr(rs, k).detach().cpu() for k in CAMERA_KEYS] if ctx.camera else []
                alpha = [ga.cpu()] if ga is not None else []
                feat = [feats["features"].cpu(), feats["grad"].cpu()] if feats is not None else []
                torch.save([t.detach().cpu() for t in ctx.saved_tensors[:9]] + split + [gc.cpu()] + camera + alpha + feat,
                           "snapshot_bw.dump")
                print("\nAn error occured in backward. Writing snapshot_bw.dump for debugging.\n")
            raise
        g_op = grads["opacities"].reshape(ctx.shapes["opacities"])
        g_cam = tuple(cam_grads[k].view(shape).to(dtype) if k in cam_grads else None
                      for k, (shape, dtype) in zip(CAMERA_KEYS, ctx.camera))
        return (grads["means3D"], grads["means2D"] if ctx.shapes["means2D"] is not None else None, grads.get("shs"),
                grads.get("colors_precomp"), g_op, grads.get("scales"), grads.get("rotations"),
                grads.get("cov3D_precomp"), None, grads.get("dc"), None,
                feats["dL_dfeatures"] if feats is not None else None, None) + g_cam


class GaussianRasterizer(nn.Module):
    def __init__(self, raster_settings: GaussianRasterizationSettings):
        super().__init__()
        self.raster_settings = raster_settings

    def markVisible(self, positions: torch.Tensor) -> torch.Tensor:
        """Frustum test only; bool [P]."""
        with torch.no_grad():
            rs = self.raster_settings
            pos = _f32c(positions)
            P = int(positions.shape[0])
            present = torch.zeros((P,), dtype=torch.uint8, device=positions.device)
            if P > 0:
                view, proj = _f32c(rs.viewmatrix), _f32c(rs.projmatrix)
                with _device_ctx(positions.device):
                    rc = _C.gsb_mark_visible(P, pos.data_ptr(), view.data_ptr(), proj.data_ptr(), present.data_ptr(),
                                             _current_stream(positions.device))
                _check(rc)
            return present.bool()

    def forward(self, means3D, means2D, opacities, shs=None, colors_precomp=None, scales=None, rotations=None,
                cov3D_precomp=None, dc=None, return_alpha=False, features=None, contrib=None):
        """``dc``: the split SH input of the accel branch (gaussian_renderer/__init__.py:90-100) -- ``dc`` [P,1,3] is the DC
        coefficient and ``shs`` [P,M-1,3] the others (may have zero coefficients); gradients come back in the same split.
        ``return_alpha=True``: also returns the rendered alpha [1,H,W] (rasterize_gaussians).  ``features`` [P,C]: also returns
        the feature map [C,H,W], last (rasterize_gaussians).  ``contrib`` (ContributionStats): the forward's contribution
        statistics are added into it (rasterize_gaussians)."""
        rs = self.raster_settings
        if (shs is None and colors_precomp is None) or (shs is not None and colors_precomp is not None):
            raise Exception("Please provide excatly one of either SHs or precomputed colors!")
        if ((scales is None or rotations is None) and cov3D_precomp is None) or \
                ((scales is not None or rotations is not None) and cov3D_precomp is not None):
            raise Exception("Please provide exactly one of either scale/rotation pair or precomputed 3D covariance!")
        if dc is not None and colors_precomp is not None:
            raise Exception("dc is the SH DC coefficient: it goes with shs, not with precomputed colors!")
        return rasterize_gaussians(means3D, means2D, shs, colors_precomp, opacities, scales, rotations, cov3D_precomp,
                                   rs, dc, return_alpha, features, contrib)


# SparseGaussianAdam: bound here only on request (module docstring); sparse_adam.py is importable either way
if os.environ.get("GSB_SPARSE_ADAM") == "1":
    from .sparse_adam import SparseGaussianAdam  # noqa: E402,F401
    __all__.append("SparseGaussianAdam")
