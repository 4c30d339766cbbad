"""Render glue for the H100 rasterizer: ``render()`` with the reference's signature and return dict
(/root/reference/gaussian_renderer/__init__.py:18-128) plus the view-batch path BASELINE.json's
north_star adds ("gaussian_renderer/__init__.py gains a view-batch path"):

* ``render_views`` -- several cameras against the same (replicated) gaussians in one call;
* ``GradientBucket`` -- one flat buffer holding every per-gaussian gradient, so that the data-parallel
  step is a SINGLE all-reduce over NVLink (views shard across ranks, gaussians are replicated;
  SURVEY.md section 8e).  The reference has no distributed path at all (SURVEY.md section 2.3).

The reference's own file stays usable unchanged: it only needs ``diff_gaussian_rasterization`` on the
path (INTEGRATION.md).  This module exists for the view-batch path and for callers that have no
``scene.GaussianModel`` (it duck-types ``pc``).
"""
from __future__ import annotations

import math
from typing import Iterable, List, Optional, Sequence

import torch

import diff_gaussian_rasterization as _dgr
from diff_gaussian_rasterization import GaussianRasterizationSettings, GaussianRasterizer

__all__ = ["render", "render_views", "render_views_backward", "GradientBucket", "AsyncCapacity", "shard_views",
           "pin_to_gpu_numa_node"]


def _eval_sh(deg, sh, dirs):
    # torch-side SH only for pipe.convert_SHs_python; formula /root/reference/utils/sh_utils.py:57-112
    C0, C1 = 0.28209479177387814, 0.4886025119029199
    C2 = [1.0925484305920792, -1.0925484305920792, 0.31539156525252005, -1.0925484305920792, 0.5462742152960396]
    C3 = [-0.5900435899266435, 2.890611442640554, -0.4570457994644658, 0.3731763325901154, -0.4570457994644658,
          1.445305721320277, -0.5900435899266435]
    result = C0 * sh[..., 0]
    if deg > 0:
        x, y, z = dirs[..., 0:1], dirs[..., 1:2], dirs[..., 2:3]
        result = result - C1 * y * sh[..., 1] + C1 * z * sh[..., 2] - C1 * x * sh[..., 3]
        if deg > 1:
            xx, yy, zz, xy, yz, xz = x * x, y * y, z * z, x * y, y * z, x * z
            result = (result + C2[0] * xy * sh[..., 4] + C2[1] * yz * sh[..., 5] + C2[2] * (2.0 * zz - xx - yy) * sh[..., 6]
                      + C2[3] * xz * sh[..., 7] + C2[4] * (xx - yy) * sh[..., 8])
            if deg > 2:
                result = (result + C3[0] * y * (3 * xx - yy) * sh[..., 9] + C3[1] * xy * z * sh[..., 10]
                          + C3[2] * y * (4 * zz - xx - yy) * sh[..., 11] + C3[3] * z * (2 * zz - 3 * xx - 3 * yy) * sh[..., 12]
                          + C3[4] * x * (4 * zz - xx - yy) * sh[..., 13] + C3[5] * z * (xx - yy) * sh[..., 14]
                          + C3[6] * x * (xx - 3 * yy) * sh[..., 15])
    return result


def render(viewpoint_camera, pc, pipe, bg_color: torch.Tensor, scaling_modifier=1.0, separate_sh=False,
           override_color=None, use_trained_exp=False, return_alpha=False, features=None, contrib=None):
    """Same contract as the reference's render(): returns
    {"render", "viewspace_points", "visibility_filter", "radii", "depth"}.  ``return_alpha=True`` adds "alpha": the rendered
    accumulated opacity [1,H,W] (1 - final transmittance, differentiable; the exposure of ``use_trained_exp`` does not apply).
    ``features`` [P,C] (per-gaussian, view-independent, 1 <= C <= 128) adds "features": the feature map [C,H,W] composited
    with the same blend weights over a zero background, differentiable w.r.t. ``features`` and the gaussians (no exposure,
    no clamp).  ``contrib`` (diff_gaussian_rasterization.ContributionStats of the P gaussians): the view's per-gaussian
    contribution statistics (blended pixel count, sum and max of the blend weights) are added into it; the result is unchanged."""
    xyz = pc.get_xyz
    screenspace_points = torch.zeros_like(xyz, dtype=xyz.dtype, requires_grad=True, device=xyz.device) + 0
    try:
        screenspace_points.retain_grad()
    except Exception:
        pass
    raster_settings = GaussianRasterizationSettings(
        image_height=int(viewpoint_camera.image_height), image_width=int(viewpoint_camera.image_width),
        tanfovx=math.tan(viewpoint_camera.FoVx * 0.5), tanfovy=math.tan(viewpoint_camera.FoVy * 0.5),
        bg=bg_color, scale_modifier=scaling_modifier, viewmatrix=viewpoint_camera.world_view_transform,
        projmatrix=viewpoint_camera.full_proj_transform, sh_degree=pc.active_sh_degree,
        campos=viewpoint_camera.camera_center, prefiltered=False, debug=bool(getattr(pipe, "debug", False)),
        antialiasing=bool(getattr(pipe, "antialiasing", False)))
    rasterizer = GaussianRasterizer(raster_settings=raster_settings)

    scales = rotations = cov3D_precomp = None
    if getattr(pipe, "compute_cov3D_python", False):
        cov3D_precomp = pc.get_covariance(scaling_modifier)
    else:
        scales, rotations = pc.get_scaling, pc.get_rotation

    shs = colors_precomp = dc = None
    if override_color is None:
        if getattr(pipe, "convert_SHs_python", False):
            feats = pc.get_features
            shs_view = feats.transpose(1, 2).view(-1, 3, (pc.max_sh_degree + 1) ** 2)
            dir_pp = xyz - viewpoint_camera.camera_center.repeat(feats.shape[0], 1)
            dir_pp = dir_pp / dir_pp.norm(dim=1, keepdim=True)
            colors_precomp = torch.clamp_min(_eval_sh(pc.active_sh_degree, shs_view, dir_pp) + 0.5, 0.0)
        elif separate_sh:
            # the split layout of the accel branch: the rasterizer stages both tensors itself (no [P,M,3] concatenation)
            dc, shs = pc.get_features_dc, pc.get_features_rest
        else:
            shs = pc.get_features
    else:
        colors_precomp = override_color

    out = rasterizer(means3D=xyz, means2D=screenspace_points, shs=shs, colors_precomp=colors_precomp, opacities=pc.get_opacity,
                     scales=scales, rotations=rotations, cov3D_precomp=cov3D_precomp, dc=dc, return_alpha=return_alpha,
                     features=features, contrib=contrib)
    rendered_image, radii, depth_image = out[:3]

    if use_trained_exp:
        exposure = pc.get_exposure_from_name(viewpoint_camera.image_name)
        rendered_image = torch.matmul(rendered_image.permute(1, 2, 0), exposure[:3, :3]).permute(2, 0, 1) \
            + exposure[:3, 3, None, None]
    rendered_image = rendered_image.clamp(0, 1)
    result = {"render": rendered_image, "viewspace_points": screenspace_points,
              "visibility_filter": (radii > 0).nonzero(), "radii": radii, "depth": depth_image}
    if return_alpha:
        result["alpha"] = out[3]
    if features is not None:
        result["features"] = out[-1]
    return result


def render_views(viewpoint_cameras: Sequence, pc, pipe, bg_color: torch.Tensor, **kw) -> List[dict]:
    """View-batch path: the same gaussians rendered from several cameras.  Each entry is a render() dict and
    stays connected to autograd, so ``sum(losses).backward()`` accumulates every view's per-gaussian gradient
    into the parameters' ``.grad`` (which GradientBucket maps onto one flat buffer)."""
    return [render(cam, pc, pipe, bg_color, **kw) for cam in viewpoint_cameras]


def _settings_for(cam, pc, pipe, bg_color, scaling_modifier):
    return GaussianRasterizationSettings(
        image_height=int(cam.image_height), image_width=int(cam.image_width),
        tanfovx=math.tan(cam.FoVx * 0.5), tanfovy=math.tan(cam.FoVy * 0.5), bg=bg_color,
        scale_modifier=scaling_modifier, viewmatrix=cam.world_view_transform, projmatrix=cam.full_proj_transform,
        sh_degree=pc.active_sh_degree, campos=cam.camera_center, prefiltered=False,
        debug=bool(getattr(pipe, "debug", False)), antialiasing=bool(getattr(pipe, "antialiasing", False)))


class AsyncCapacity:
    """Instance-capacity bookkeeping of the SYNC-FREE view-batch step (gsb_forward_batch_async).

    The synchronous path reads the V instance counts back every batch to size the binning buffers: one host wait per
    step, which caps how far the host can run ahead of the device at less than one step -- so any host hiccup (a
    scheduling stall of tens of ms) lands on the device timeline of EVERY rank through the
    all-reduce.  Here the capacity is fixed up front, the counts stay on the device together with their running maximum,
    and the host only looks at that maximum when it chooses to (``check()``: end of an epoch / every N steps).  A step
    whose count exceeded the capacity rendered from truncated lists; ``check()`` then returns False, grows the capacity,
    and the caller re-runs from its last good state (in steady state the counts drift by a few percent per densification
    interval against 25 % of slack, so this is rare; right after densify_and_prune call ``reset()`` and run one
    synchronous step)."""

    def __init__(self, device, capacity: int = 0):
        self.counts = torch.zeros(_dgr.COUNT_SLOTS, dtype=torch.int64, device=device)
        self.capacity = int(capacity)

    def learn(self, num_rendered: Sequence[int]) -> None:
        """Size the capacity from the counts a synchronous step observed."""
        self.capacity = max(self.capacity, _dgr.capacity_for(max(int(n) for n in num_rendered)))

    def observed_max(self) -> int:
        """Largest per-view count since the last reset (synchronises with the device)."""
        return int(self.counts[_dgr.COUNT_SLOTS - 1].item())

    def check(self) -> bool:
        seen = self.observed_max()
        if seen > self.capacity:
            self.capacity = _dgr.capacity_for(seen)
            self.counts.zero_()
            return False
        return True

    def reset(self) -> None:
        self.capacity = 0
        self.counts.zero_()


def pin_to_gpu_numa_node(device_index: int) -> Optional[list]:
    """Restrict this process to the CPU cores that are local to its GPU (one process per GPU: without it the launch
    thread migrates across sockets and shares cores with the other ranks' threads).  Uses NVML's ideal-affinity mask;
    returns the core list, or None when NVML / sched_setaffinity are unavailable.  Never raises."""
    import os
    try:
        import pynvml
        pynvml.nvmlInit()
        vis = os.environ.get("CUDA_VISIBLE_DEVICES")
        idx = device_index
        if vis and all(x.strip().isdigit() for x in vis.split(",")):
            idx = int(vis.split(",")[device_index])
        h = pynvml.nvmlDeviceGetHandleByIndex(idx)
        words = (os.cpu_count() + 63) // 64
        mask = pynvml.nvmlDeviceGetCpuAffinity(h, words)
        cores = [64 * w + b for w in range(words) for b in range(64) if (int(mask[w]) >> b) & 1]
        allowed = sorted(set(cores) & set(os.sched_getaffinity(0)))
        if not allowed:
            return None
        os.sched_setaffinity(0, allowed)
        return allowed
    except Exception:
        return None


def render_views_backward(viewpoint_cameras: Sequence, pc, pipe, bg_color: torch.Tensor, loss_fn, *,
                          scaling_modifier: float = 1.0, densify_stats: Optional[dict] = None,
                          keep_images: bool = False, loss_returns_grad: bool = False, batched: bool = True,
                          overwrite: bool = False, capacity: Optional[AsyncCapacity] = None, grad_chunks: int = 1,
                          on_grad_chunk=None, peers=None, with_alpha: bool = False, features=None, contrib=None) -> dict:
    """Fused view-batch training step: forward + loss + backward for every camera, with the per-gaussian
    gradients of ALL views summed in place.

    The activations (exp / sigmoid / normalize / cat in scene.GaussianModel, gaussian_model.py:102-130) do not
    depend on the view, so they run ONCE per batch; each view then goes straight through the C ABI
    (gsb_forward / gsb_backward with accumulate=1) and adds its gradient w.r.t. the activated tensors into one
    buffer; one ``torch.autograd.backward`` at the end chains that sum into the leaf parameters.  When the
    rasterizer's inputs already ARE leaves whose ``.grad`` is set (GradientBucket), the kernels accumulate
    directly into ``.grad`` and no extra pass over the 59 floats/gaussian is made.

    ``loss_fn(image[3,H,W] (clamped to [0,1] like render() does), invdepth[1,H,W], view_index) -> scalar``, or,
    with ``loss_returns_grad=True``, ``loss_fn(raw_image, invdepth, view_index) -> (loss, dL/d raw_image[, dL/d invdepth])``
    for a loss that brings its own gradient (e.g. ``diff_gaussian_rasterization.l1_loss_and_grad``); no autograd then.  If such
    a loss_fn has a ``grad_out`` parameter it is handed the slot of the batch's gradient buffer to write into (no copy).
    Returns {"losses": [V] tensor, "radii_max": [P] int32, "num_rendered": per-view instance counts, "images": list (if keep_images)}.

    ``overwrite=True``: the gradient buffers are WRITTEN by the first chunk of views instead of added to, so the
    caller does not have to zero them first (saves one memset and one read pass over the 59 floats/gaussian).

    ``batched=True`` (default, up to 16 views of equal size per chunk) goes through gsb_forward_batch /
    gsb_backward_batch: the gaussians' parameters are read once for all views in the per-gaussian kernels, the
    depth sorts / scans / tile sorts of the views run as single batched launches, the summed gradient is written
    once, and there is ONE host read-back per chunk.  ``batched=False`` runs view by view (one read-back each).

    A camera whose ``world_view_transform`` / ``full_proj_transform`` / ``camera_center`` (or ``bg_color``) requires grad
    receives its gradient like a non-leaf gaussian input: each view's camera gradient comes out of the backward kernels
    (gsb_backward_batch_camera / gsb_backward_camera) and is chained into the camera tensors' graphs at the end.  This is
    not available with ``grad_chunks`` > 1, ``on_grad_chunk`` or ``peers`` (ValueError).

    ``with_alpha=True``: ``loss_fn`` also receives the rendered alpha [1,H,W] (1 - final transmittance) as the keyword ``alpha``
    and may use it: the autograd mode differentiates through it; with ``loss_returns_grad=True`` it may return
    ``(loss, dL/d image, dL/d invdepth | None, dL/d alpha | None)``.  The alpha gradient goes into the same backward call in every
    mode (batched or not, sync or async, chunked, peers); a view batch in which no view returns one takes the plain backward.
    ``keep_images=True`` also returns "alphas".

    ``features`` [P,C] (per-gaussian, view-independent; a leaf or not): ``loss_fn`` also receives the view's feature map [C,H,W]
    (render(features=...)) as the keyword ``features``; with ``loss_returns_grad=True`` it may return a fifth element,
    ``dL/d feature map | None`` (the fourth, alpha's, may be None).  dL/dfeatures, summed over the views, goes into ``features``
    like a gaussian input's gradient, and the map's gradient into the same backward call.  Not with ``grad_chunks`` > 1,
    ``on_grad_chunk`` or ``peers`` (ValueError).  ``keep_images=True`` also returns "features" (the maps).

    ``contrib`` (diff_gaussian_rasterization.ContributionStats of the P gaussians): every view's per-gaussian contribution
    statistics are added into it, one launch per forward call (view-batch chunk or single view).  It only reads the forward
    states, so it works in every mode (batched or not, sync or async, chunked, peers) and changes no output or gradient.
    """
    takes_grad_out = False
    if loss_returns_grad:
        try:
            import inspect
            takes_grad_out = "grad_out" in inspect.signature(loss_fn).parameters
        except (TypeError, ValueError):
            takes_grad_out = False
    xyz, opacity = pc.get_xyz, pc.get_opacity
    scales, rotations, shs = pc.get_scaling, pc.get_rotation, pc.get_features
    inputs = dict(means3D=xyz, shs=shs, opacities=opacity, scales=scales, rotations=rotations)
    P = int(xyz.shape[0])
    dev = xyz.device
    if contrib is not None:
        _dgr.check_contrib(contrib, P, dev)

    def grad_target(t):
        if t.is_leaf and t.requires_grad and t.grad is not None and t.grad.is_contiguous():
            return t.grad, True
        return torch.zeros_like(t, dtype=torch.float32, memory_format=torch.contiguous_format), False

    targets = {k: grad_target(v) for k, v in inputs.items()}
    grads = {k: tv[0] for k, tv in targets.items()}
    fc = f_target = None
    if features is not None:
        _dgr.check_features(features, P, dev)
        if grad_chunks > 1 or on_grad_chunk is not None or peers is not None:
            raise ValueError("render_views_backward: features cannot be combined with grad_chunks > 1, on_grad_chunk or peers")
        fc = features.detach().float().contiguous()
        if features.requires_grad:
            f_target = grad_target(features)
            if f_target[1] and f_target[0].dtype != torch.float32:     # the kernels add float32 only
                f_target = (torch.zeros(features.shape, dtype=torch.float32, device=dev), False)
    fmaps = []

    def feature_term(fmap, g_feat):
        """the backward's feature term (None: no view of the call returned a feature-map gradient)"""
        if g_feat is None:
            return None
        return dict(features=fc, out=fmap, grad=g_feat, dL_dfeatures=f_target[0] if f_target is not None else None)

    def view_loss(img_in, dep_in, vi, extra, grad_out=None):
        """(loss, dL/d image, dL/d invdepth, dL/d alpha, dL/d feature map) of one view; extra: loss_fn's keyword inputs"""
        if loss_returns_grad:
            res = loss_fn(img_in, dep_in, vi, grad_out=grad_out, **extra) if grad_out is not None else \
                loss_fn(img_in, dep_in, vi, **extra)
            res = tuple(res) + (None,) * (5 - len(res))
            return res[0], res[1], res[2], res[3] if with_alpha else None, res[4] if fc is not None else None
        img = img_in.detach().requires_grad_(True)
        dep = dep_in.detach().requires_grad_(True)
        extra = {a: t.detach().requires_grad_(True) for a, t in extra.items()}
        with torch.enable_grad():
            loss = loss_fn(img.clamp(0, 1), dep, vi, **extra)
        g = torch.autograd.grad(loss, (img, dep, *extra.values()), allow_unused=True)
        ge = dict(zip(extra.keys(), g[2:]))
        return loss, g[0], g[1], ge.get("alpha"), ge.get("features")
    if densify_stats is not None:
        m2d = torch.empty((P, 3), dtype=torch.float32, device=dev)
    c = {k: _dgr._f32c(v.detach()) for k, v in inputs.items()}
    c["opacities"] = c["opacities"].reshape(-1) if c["opacities"] is not None else None
    losses, images, alphas, num_rendered = [], [], [], []
    radii_max = torch.zeros((P,), dtype=torch.int32, device=dev)
    cam_chain = {}      # id(camera tensor) -> [tensor, summed gradient]  (bg_color is shared by every view)

    def camera_targets(rss):
        """{key: zeroed [V, n] float32} for the camera tensors of `rss` that require grad (None when there are none)."""
        keys = [k for k in _dgr.CAMERA_KEYS if any(getattr(rs, k).requires_grad for rs in rss)]
        if not keys:
            return None
        if grad_chunks > 1 or on_grad_chunk is not None or peers is not None:
            raise ValueError("render_views_backward: cameras that require grad cannot be combined with grad_chunks > 1, "
                             "on_grad_chunk or peers (the camera gradient is a sum over all gaussians of one view)")
        return {k: torch.zeros((len(rss), _dgr._CAMERA_NUMEL[k]), dtype=torch.float32, device=dev) for k in keys}

    def chain_camera(rss, cam_grads):
        for k, g in (cam_grads or {}).items():
            for vi, rs in enumerate(rss):
                t = getattr(rs, k)
                if t.requires_grad:
                    entry = cam_chain.setdefault(id(t), [t, torch.zeros_like(t)])
                    entry[1] += g[vi].view(t.shape).to(t.dtype)

    cams_all = list(viewpoint_cameras) if batched else None
    if batched and cams_all and all(int(cm.image_height) == int(cams_all[0].image_height) and
                                    int(cm.image_width) == int(cams_all[0].image_width) for cm in cams_all):
        for c0 in range(0, len(cams_all), _dgr.MAX_BATCH_VIEWS):
            chunk = cams_all[c0:c0 + _dgr.MAX_BATCH_VIEWS]
            rss = [_settings_for(cm, pc, pipe, bg_color, scaling_modifier) for cm in chunk]
            use_async = capacity is not None and capacity.capacity > 0
            color, radii, invdepth, pack = _dgr._forward_batch_impl(c["means3D"], c["shs"], c["opacities"], c["scales"],
                                                                    c["rotations"], rss,
                                                                    async_counts=capacity.counts if use_async else None,
                                                                    capacity=capacity.capacity if use_async else 0)
            if capacity is not None and not use_async:
                capacity.learn(pack["num_rendered"])
            num_rendered.extend(pack["num_rendered"])
            alpha = _dgr._alpha_impl(pack["states"], int(color.shape[-2]), int(color.shape[-1]), dev) if with_alpha else None
            fmap = _dgr._features_impl(pack["states"], int(color.shape[-2]), int(color.shape[-1]), fc, dev) if fc is not None else None
            if contrib is not None:
                _dgr._contrib_impl(pack["states"], int(color.shape[-2]), int(color.shape[-1]), P, contrib, dev)
            g_color = torch.empty_like(color)
            g_depth = g_alpha = g_feat = None
            for k in range(len(chunk)):
                vi = c0 + k
                akw = dict(alpha=alpha[k]) if with_alpha else {}
                if fc is not None:
                    akw["features"] = fmap[k]
                loss, g_img, g_dep, g_al, g_fe = view_loss(color[k], invdepth[k], vi, akw,
                                                           grad_out=g_color[k] if takes_grad_out else None)
                if g_img is None:
                    g_color[k].zero_()
                elif g_img.data_ptr() != g_color[k].data_ptr():
                    g_color[k].copy_(g_img)
                if g_dep is not None:
                    if g_depth is None:
                        g_depth = torch.zeros_like(invdepth)
                    g_depth[k].copy_(g_dep)
                if g_al is not None:
                    if g_alpha is None:
                        g_alpha = torch.zeros_like(alpha)
                    g_alpha[k].copy_(g_al.reshape(alpha[k].shape))
                if g_fe is not None:
                    if g_feat is None:
                        g_feat = torch.zeros_like(fmap)
                    g_feat[k].copy_(g_fe.reshape(fmap[k].shape))
                losses.append(loss.detach().reshape(()))
                if keep_images:
                    images.append(color[k].detach())
                    if with_alpha:
                        alphas.append(alpha[k])
                    if fc is not None:
                        fmaps.append(fmap[k])
            vg = dict(grads)
            if densify_stats is not None:
                vg["means2D"] = torch.empty((len(chunk), P, 3), dtype=torch.float32, device=dev)
            last_chunk = c0 + _dgr.MAX_BATCH_VIEWS >= len(cams_all)     # gradients are final only after the last view chunk
            cam_grads = camera_targets(rss)
            _dgr._backward_batch_impl(pack, rss, c["means3D"], c["shs"], c["opacities"], c["scales"], c["rotations"], color,
                                      invdepth, g_color, g_depth, vg, accumulate=not (overwrite and c0 == 0),
                                      n_chunks=grad_chunks if last_chunk else 1, on_chunk=on_grad_chunk if last_chunk else None,
                                      peers=peers, cam_grads=cam_grads, grad_alpha=g_alpha, feats=feature_term(fmap, g_feat))
            chain_camera(rss, cam_grads)
            torch.maximum(radii_max, radii.max(dim=0).values, out=radii_max)
            if densify_stats is not None:
                vis = radii > 0                                               # [V,P]
                densify_stats["xyz_gradient_accum"] += (vg["means2D"][:, :, :2].norm(dim=-1) * vis).sum(dim=0)[:, None]
                densify_stats["denom"] += vis.sum(dim=0)[:, None].to(densify_stats["denom"].dtype)
        viewpoint_cameras = []
    for vi, cam in enumerate(viewpoint_cameras):
        rs = _settings_for(cam, pc, pipe, bg_color, scaling_modifier)
        color, radii, invdepth, pack = _dgr._forward_impl(c["means3D"], c["shs"], None, c["opacities"], c["scales"],
                                                          c["rotations"], None, rs)
        num_rendered.append(pack["num_rendered"])
        alpha = _dgr._alpha_impl(pack["state"], int(color.shape[-2]), int(color.shape[-1]), dev) if with_alpha else None
        fmap = _dgr._features_impl(pack["state"], int(color.shape[-2]), int(color.shape[-1]), fc, dev) if fc is not None else None
        if contrib is not None:
            _dgr._contrib_impl(pack["state"], int(color.shape[-2]), int(color.shape[-1]), P, contrib, dev)
        akw = dict(alpha=alpha) if with_alpha else {}
        if fc is not None:
            akw["features"] = fmap
        loss, g_img, g_dep, g_al, g_fe = view_loss(color, invdepth, vi, akw)
        if g_img is None and not loss_returns_grad:
            g_img = torch.zeros_like(color)
        vg = dict(grads)
        if densify_stats is not None:
            vg["means2D"] = m2d
        cam_grads = camera_targets([rs])
        _dgr._backward_impl(pack, rs, c["means3D"], c["shs"], None, c["opacities"], c["scales"], c["rotations"], None,
                            color.detach(), invdepth.detach(), _dgr._f32c(g_img), _dgr._f32c(g_dep), vg,
                            accumulate=not (overwrite and vi == 0), accumulate_means2D=False,
                            cam_grads={k: g[0] for k, g in cam_grads.items()} if cam_grads else None,
                            grad_alpha=_dgr._f32c(g_al.reshape(alpha.shape)) if g_al is not None else None,
                            feats=feature_term(fmap, _dgr._f32c(g_fe.reshape(fmap.shape)) if g_fe is not None else None))
        chain_camera([rs], cam_grads)
        torch.maximum(radii_max, radii, out=radii_max)
        if densify_stats is not None:
            # add_densification_stats (gaussian_model.py:471-473) + max_radii2D update (train.py:166), sync-free
            vis = radii > 0
            densify_stats["xyz_gradient_accum"] += (m2d[:, :2].norm(dim=-1, keepdim=True) * vis[:, None])
            densify_stats["denom"] += vis[:, None].to(densify_stats["denom"].dtype)
        losses.append(loss.detach().reshape(()).clone() if loss_returns_grad else loss.detach())
        if keep_images:
            images.append(color.detach())
            if with_alpha:
                alphas.append(alpha.detach())
            if fc is not None:
                fmaps.append(fmap)
    # chain the summed gradient into non-leaf inputs' graphs (one pass, view independent)
    chain_t, chain_g = [], []
    for k, v in inputs.items():
        g, direct = targets[k]
        if not direct and v.requires_grad:
            chain_t.append(v)
            chain_g.append(g.view_as(v))
    for t, g in cam_chain.values():
        chain_t.append(t)
        chain_g.append(g)
    if f_target is not None and not f_target[1]:
        chain_t.append(features)
        chain_g.append(f_target[0].view_as(features).to(features.dtype))
    if chain_t:
        torch.autograd.backward(chain_t, chain_g)
    if hasattr(pc, "gradients_ready"):      # gaussian_store.GaussianModel: its gradient buffer now belongs to the current parameters
        pc.gradients_ready()
    out = {"losses": torch.stack(losses) if losses else torch.zeros(0, device=dev), "radii_max": radii_max,
           "num_rendered": num_rendered}      # per view; -1 on the sync-free path (known to the device only)
    if keep_images:
        out["images"] = images
        if with_alpha:
            out["alphas"] = alphas
        if fc is not None:
            out["features"] = fmaps
    return out


def shard_views(views: Sequence, rank: int, world_size: int) -> list:
    """Round-robin view partition over ranks (SURVEY.md section 8e)."""
    return [v for i, v in enumerate(views) if i % world_size == rank]


class GradientBucket:
    """Maps the ``.grad`` of every gaussian parameter onto views of ONE flat float32 buffer, so the
    data-parallel reduction is a single ``all_reduce`` (59 floats per gaussian at SH degree 3:
    xyz 3, f_dc 3, f_rest 45, opacity 1, scaling 3, rotation 4; parameter groups at
    /root/reference/scene/gaussian_model.py:183-190), followed by the per-view densification
    statistics the training loop needs identical on every rank."""

    def __init__(self, params: Iterable[torch.Tensor]):
        self.params = [p for p in params]
        if not self.params:
            raise ValueError("GradientBucket needs at least one parameter")
        dev, total = self.params[0].device, sum(p.numel() for p in self.params)
        self.flat = torch.zeros(total, dtype=torch.float32, device=dev)
        # Layout: the widest parameter (the SH coefficients: 48 of the 59 floats per gaussian) LAST, everything else in front of
        # it as one contiguous region -- the chunk-wise reduction then needs one collective per chunk of SH rows plus ONE for the
        # rest, instead of one per (chunk, parameter): twenty latency-bound launches cost what the overlap saves.
        width = lambda p: p.numel() // max(1, p.shape[0])
        self.big = max(self.params, key=width)
        off = 0
        for p in [q for q in self.params if q is not self.big] + [self.big]:
            if p.dtype != torch.float32 or p.device != dev:
                raise ValueError("GradientBucket: float32 parameters on one device only")
            if p is self.big:
                self.rest = self.flat[:off]
            p.grad = self.flat[off:off + p.numel()].view_as(p)
            off += p.numel()

    def zero_(self):
        self.flat.zero_()

    @staticmethod
    def _distributed(group) -> bool:
        import torch.distributed as dist
        return dist.is_available() and dist.is_initialized() and dist.get_world_size(group) > 1

    def all_reduce_rows(self, p_begin: int, p_end: int, group=None):
        """Asynchronous all-reduce of gaussians [p_begin, p_end) of the WIDEST parameter's gradient (a contiguous row range).
        Ordered after the work enqueued so far on the current stream, running on the process group's own stream, i.e.
        concurrently with whatever the caller enqueues next.  Returns a list of handles for ``wait_all`` (empty for world
        size 1).  The other parameters go out with ``all_reduce_rest`` once every chunk has been enqueued."""
        import torch.distributed as dist
        if not self._distributed(group) or p_end <= p_begin:
            return []
        return [dist.all_reduce(self.big.grad[p_begin:p_end], op=dist.ReduceOp.SUM, group=group, async_op=True)]

    def all_reduce_rest(self, group=None):
        """Asynchronous all-reduce of every parameter but the widest one: one collective over their contiguous region."""
        import torch.distributed as dist
        if not self._distributed(group) or self.rest.numel() == 0:
            return []
        return [dist.all_reduce(self.rest, op=dist.ReduceOp.SUM, group=group, async_op=True)]

    @staticmethod
    def wait_all(handles) -> None:
        """The current stream waits for the reductions (no host block)."""
        for h in handles:
            h.wait()

    def all_reduce(self, group=None, average: bool = False):
        """One collective for all per-gaussian gradients.  No-op for world size 1."""
        import torch.distributed as dist
        if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size(group) == 1:
            return self.flat
        dist.all_reduce(self.flat, op=dist.ReduceOp.SUM, group=group)
        if average:
            self.flat.div_(dist.get_world_size(group))
        return self.flat

    @staticmethod
    def reduce_densification_stats(grad_norm_accum: torch.Tensor, denom: torch.Tensor, max_radii2D: torch.Tensor,
                                   group=None):
        """Per-view statistics feeding densify/prune (gaussian_model.py:471-473, train.py:166) must agree on
        all ranks: sum for the accumulated gradient norm and its count, max for the radii."""
        import torch.distributed as dist
        if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size(group) == 1:
            return
        packed = torch.cat([grad_norm_accum.reshape(-1), denom.reshape(-1).to(grad_norm_accum.dtype)])
        dist.all_reduce(packed, op=dist.ReduceOp.SUM, group=group)
        n = grad_norm_accum.numel()
        grad_norm_accum.copy_(packed[:n].view_as(grad_norm_accum))
        denom.copy_(packed[n:].view_as(denom).to(denom.dtype))
        dist.all_reduce(max_radii2D, op=dist.ReduceOp.MAX, group=group)
