"""Training state of the gaussians on ONE flat device buffer, mirroring the parts of the reference's
``scene.GaussianModel`` that sit either side of the rasterizer (SURVEY.md section 8(f) rows 1 and 3;
/root/reference/scene/gaussian_model.py):

    training_setup :176-211 | update_learning_rate :213-223 | reset_opacity :258-261 | densify_and_prune :452-469
    add_densification_stats :471-473 | oneupSHdegree :146-148 | activations :102-130 | optimizer.step() train.py:178-186
    per-image exposures :133-140, :173-176, :201-217, :264-274 (plain torch parameters with their own Adam, as in the reference)

What differs, and why.  The reference keeps six ``nn.Parameter`` tensors, lets autograd chain the rasterizer's gradients
through exp / sigmoid / normalize / cat, runs ``torch.optim.Adam`` group by group, and rebuilds every tensor and both Adam
moments with boolean-mask gathers and ``cat`` when it densifies.  Here the raw parameters, their gradients and both moments
are four flat float32 buffers with the same group-after-group layout (include/gs_b200.h, "store"):

  * the rasterizer's backward writes dLoss/d(activated value) straight into the gradient buffer (the activated tensors
    returned by ``get_xyz`` ... ``get_rotation`` are leaves whose ``.grad`` aliases it),
  * the data-parallel reduction is ONE ``all_reduce`` of ``self.grad``,
  * ``optimizer_step`` is ONE kernel: activation backward + Adam for all six groups + re-activation (``gsb_adam_step``),
  * ``densify_and_prune`` is a plan (one read-back) plus ONE gather into fresh buffers (``gsb_densify_plan/_apply``).

Results are those of the reference (tests/test_store_gpu.py replays the fixture recorded from the reference class).
The kernels are CUDA only: on a CPU tensor the calls raise -- there is no fallback.
"""
from __future__ import annotations

import math
from typing import Dict, Optional

import torch

import diff_gaussian_rasterization as _dgr

__all__ = ["GaussianModel", "expon_lr", "store_offsets"]


class _StoreBucket:
    """GaussianModel.grad as the data-parallel bucket: one all-reduce for everything, or -- overlapped with the chunked
    gradient kernel -- row ranges of the features group (most of the bytes) followed by one launch for the other groups."""

    def __init__(self, model):
        self.m = model

    def zero_(self):
        self.m.grad.zero_()

    @staticmethod
    def _distributed(group) -> bool:
        import torch.distributed as dist
        return dist.is_available() and dist.is_initialized() and dist.get_world_size(group) > 1

    def all_reduce_rows(self, p_begin: int, p_end: int, group=None):
        """Rows [p_begin, p_end) of the features group (3 M of the 11 + 3 M floats per gaussian), asynchronously."""
        import torch.distributed as dist
        if not self._distributed(group) or p_end <= p_begin:
            return []
        m = self.m
        a, w = store_offsets(m.P, m.sh_coeffs)["features"], 3 * m.sh_coeffs
        return [dist.all_reduce(m.grad[a + w * p_begin:a + w * p_end], op=dist.ReduceOp.SUM, group=group, async_op=True)]

    def all_reduce_rest(self, group=None):
        """The other four groups: xyz, and opacity | scaling | rotation (contiguous), as one coalesced launch."""
        import torch.distributed as dist
        if not self._distributed(group):
            return []
        m = self.m
        o = store_offsets(m.P, m.sh_coeffs)
        segs = [m.grad[:o["features"]], m.grad[o["opacity"]:]]
        manager = getattr(dist, "_coalescing_manager", None)
        if manager is None:
            return [dist.all_reduce(t, op=dist.ReduceOp.SUM, group=group, async_op=True) for t in segs]
        with manager(group=group, async_ops=True) as cm:
            for t in segs:
                dist.all_reduce(t, op=dist.ReduceOp.SUM, group=group)
        return [cm]

    @staticmethod
    def wait_all(handles) -> None:
        for h in handles:
            h.wait()

    def all_reduce(self, group=None):
        import torch.distributed as dist
        if dist.is_available() and dist.is_initialized() and dist.get_world_size(group) > 1:
            dist.all_reduce(self.m.grad, op=dist.ReduceOp.SUM, group=group)
        return self.m.grad

GROUPS = ("xyz", "f_dc", "f_rest", "opacity", "scaling", "rotation")


def expon_lr(step: int, lr_init: float, lr_final: float, lr_delay_steps: int = 0, lr_delay_mult: float = 1.0,
             max_steps: int = 1000000) -> float:
    """The position learning-rate schedule (utils/general_utils.py:29-62): log-linear from lr_init to lr_final."""
    if step < 0 or (lr_init == 0.0 and lr_final == 0.0):
        return 0.0
    delay = 1.0
    if lr_delay_steps > 0:
        delay = lr_delay_mult + (1.0 - lr_delay_mult) * math.sin(0.5 * math.pi * min(max(step / lr_delay_steps, 0.0), 1.0))
    t = min(max(step / max_steps, 0.0), 1.0)
    return delay * math.exp(math.log(lr_init) * (1.0 - t) + math.log(lr_final) * t)


def store_offsets(P: int, sh_coeffs: int) -> Dict[str, int]:
    """First float of every group in the flat store (include/gs_b200.h)."""
    feat = 3 * P
    op = feat + 3 * sh_coeffs * P
    return {"xyz": 0, "features": feat, "opacity": op, "scaling": op + P, "rotation": op + 4 * P, "total": op + 8 * P}


class GaussianModel:
    def __init__(self, sh_degree: int, optimizer_type: str = "default"):
        self.active_sh_degree = 0
        self.max_sh_degree = int(sh_degree)
        self.sh_coeffs = (self.max_sh_degree + 1) ** 2
        self.optimizer_type = optimizer_type
        self.P = 0
        self.store = self.grad = self.exp_avg = self.exp_avg_sq = self.act = None
        self.max_radii2D = self.xyz_gradient_accum = self.denom = None
        self.percent_dense = 0.0
        self.spatial_lr_scale = 0.0
        self.step_count = 0                                   # optimizer_step() calls that updated at least one group
        self.group_steps = {n: 0 for n in GROUPS}             # torch.optim.Adam keeps one step count PER PARAMETER
        self._skip_next = set()                               # groups whose parameter was replaced since the last backward
        self.densify_seed = 0                                 # seed of the split-sample draws (identical on every data-parallel rank)
        self._densify_calls = 0
        self.lr: Dict[str, float] = {}
        self.betas, self.eps = (0.9, 0.999), 1e-15
        self._xyz_sched = None
        # per-image exposure (gaussian_model.py:133-140,173-176): ordinary torch parameters next to the flat store -- a [N,3,4]
        # affine colour transform per training image, applied by render(use_trained_exp=True), with its own Adam
        self._exposure = None
        self.exposure_mapping: Dict[str, int] = {}
        self.pretrained_exposures = None
        self.exposure_optimizer = None
        self._exposure_sched = None

    # ---- construction ----------------------------------------------------------------------------------------------
    def create_from_tensors(self, xyz, features_dc, features_rest, scaling, rotation, opacity, spatial_lr_scale: float = 1.0):
        """Raw (pre-activation) parameters, shapes as in the reference: xyz [P,3], features_dc [P,1,3], features_rest
        [P,M-1,3], scaling [P,3] (log), rotation [P,4], opacity [P,1] (logit)."""
        P, M = int(xyz.shape[0]), self.sh_coeffs
        if tuple(features_dc.shape) != (P, 1, 3) or tuple(features_rest.shape) != (P, M - 1, 3):
            raise ValueError(f"features_dc / features_rest must be [P,1,3] / [P,{M - 1},3]")
        self.spatial_lr_scale = float(spatial_lr_scale)
        dev = xyz.device
        self._allocate(P, dev)
        with torch.no_grad():
            self._xyz.copy_(xyz)
            self._features[:, :1].copy_(features_dc)
            self._features[:, 1:].copy_(features_rest)
            self._scaling.copy_(scaling.reshape(P, 3))
            self._rotation.copy_(rotation.reshape(P, 4))
            self._opacity.copy_(opacity.reshape(P, 1))
        self._reactivate()
        self.max_radii2D = torch.zeros(P, device=dev)
        return self

    def create_exposures(self, cam_infos, device=None):
        """One identity 3x4 exposure per training image (gaussian_model.py:173-176).  ``cam_infos``: objects with an
        ``image_name`` attribute (the reference's CameraInfo) or the names themselves."""
        names = [c if isinstance(c, str) else c.image_name for c in cam_infos]
        dev = device if device is not None else (self.store.device if self.store is not None else "cpu")
        self.exposure_mapping = {name: idx for idx, name in enumerate(names)}
        self.pretrained_exposures = None
        self._exposure = torch.nn.Parameter(torch.eye(3, 4, device=dev)[None].repeat(len(names), 1, 1).requires_grad_(True))
        return self

    @property
    def get_exposure(self):
        return self._exposure

    def get_exposure_from_name(self, image_name):
        """gaussian_model.py:136-140: the trained exposure of an image, or the one loaded from exposure.json."""
        if self.pretrained_exposures is None:
            if self._exposure is None:
                raise RuntimeError("no exposures: call create_exposures(cam_infos) (or create_from_pcd(..., cam_infos=...)) first")
            return self._exposure[self.exposure_mapping[image_name]]
        return self.pretrained_exposures[image_name]

    def load_exposures(self, exposure_file: str, device="cuda") -> bool:
        """exposure.json as Scene.save writes it (scene/__init__.py:87-94; read at gaussian_model.py:264-274):
        {image_name: 3x4 nested list}.  Returns False (and keeps training exposures) when the file does not exist."""
        import json
        import os
        if not os.path.exists(exposure_file):
            self.pretrained_exposures = None
            return False
        with open(exposure_file, "r") as f:
            exposures = json.load(f)
        self.pretrained_exposures = {name: torch.tensor(exposures[name], dtype=torch.float32, device=device).requires_grad_(False)
                                     for name in exposures}
        return True

    def save_exposures(self, exposure_file: str) -> None:
        """The exposure.json of scene/__init__.py:87-94."""
        import json
        table = {name: self.get_exposure_from_name(name).detach().cpu().numpy().tolist() for name in self.exposure_mapping}
        with open(exposure_file, "w") as f:
            json.dump(table, f, indent=2)

    def create_from_pcd(self, points: torch.Tensor, colors: torch.Tensor, spatial_lr_scale: float = 1.0, cam_infos=None):
        """Initialisation from a point cloud (gaussian_model.py:150-176): colours -> SH DC band (RGB2SH, utils/sh_utils.py:114-115),
        higher bands zero, isotropic log-scales from the mean squared distance to the three nearest neighbours (the
        ``distCUDA2`` call, here gsb_knn_mean_dist2), identity rotations, opacity 0.1, and -- with ``cam_infos`` -- one identity
        exposure per training image.  ``points`` [N,3], ``colors`` [N,3] in [0,1]."""
        pts = points.detach().to(torch.float32).reshape(-1, 3).contiguous()
        N, M = int(pts.shape[0]), self.sh_coeffs
        dc = ((colors.detach().to(pts.device, torch.float32).reshape(N, 3) - 0.5) / 0.28209479177387814).reshape(N, 1, 3)
        dist2 = torch.clamp_min(_dgr.knn_mean_dist2(pts), 0.0000001)
        scales = torch.log(torch.sqrt(dist2))[:, None].repeat(1, 3)
        rots = torch.zeros((N, 4), device=pts.device)
        rots[:, 0] = 1
        opac = torch.full((N, 1), math.log(0.1 / 0.9), device=pts.device)          # inverse_sigmoid(0.1)
        if cam_infos is not None:
            self.create_exposures(cam_infos, device=pts.device)
        return self.create_from_tensors(pts, dc, torch.zeros((N, M - 1, 3), device=pts.device), scales, rots, opac, spatial_lr_scale)

    def _allocate(self, P: int, device):
        total = store_offsets(P, self.sh_coeffs)["total"]
        self.P = P
        self.store = torch.zeros(total, dtype=torch.float32, device=device)
        self.grad = torch.zeros(total, dtype=torch.float32, device=device)
        self.exp_avg = torch.zeros(total, dtype=torch.float32, device=device)
        self.exp_avg_sq = torch.zeros(total, dtype=torch.float32, device=device)
        self.act = torch.zeros(8 * P, dtype=torch.float32, device=device)
        self._bind()

    def _bind(self):
        """(Re)creates the typed views over the flat buffers.  The activated tensors are autograd leaves whose ``.grad`` is
        the matching slice of ``self.grad``: gaussian_renderer.render_views_backward then accumulates in place."""
        P, M, o = self.P, self.sh_coeffs, store_offsets(self.P, self.sh_coeffs)
        cut = lambda buf, a, n, *shape: buf[a:a + n].view(*shape)
        s = self.store
        self._xyz = cut(s, o["xyz"], 3 * P, P, 3)
        self._features = cut(s, o["features"], 3 * M * P, P, M, 3)
        self._opacity = cut(s, o["opacity"], P, P, 1)
        self._scaling = cut(s, o["scaling"], 3 * P, P, 3)
        self._rotation = cut(s, o["rotation"], 4 * P, P, 4)
        leaves = {"xyz": cut(s, o["xyz"], 3 * P, P, 3), "features": cut(s, o["features"], 3 * M * P, P, M, 3),
                  "opacity": cut(self.act, 0, P, P, 1), "scaling": cut(self.act, P, 3 * P, P, 3),
                  "rotation": cut(self.act, 4 * P, 4 * P, P, 4)}
        gshape = {"xyz": (o["xyz"], 3 * P, (P, 3)), "features": (o["features"], 3 * M * P, (P, M, 3)),
                  "opacity": (o["opacity"], P, (P, 1)), "scaling": (o["scaling"], 3 * P, (P, 3)),
                  "rotation": (o["rotation"], 4 * P, (P, 4))}
        for name, t in leaves.items():
            t.requires_grad_(True)
            a, n, shape = gshape[name]
            t.grad = self.grad[a:a + n].view(*shape)
        self._leaves = leaves

    def _reactivate(self):
        _dgr.activate(self.store, self.act, self.P, self.sh_coeffs)

    # ---- what render() reads (gaussian_model.py:102-130) -----------------------------------------------------------
    @property
    def get_xyz(self):
        return self._leaves["xyz"]

    @property
    def get_features(self):
        return self._leaves["features"]

    @property
    def get_features_dc(self):
        return self._features[:, :1]

    @property
    def get_features_rest(self):
        return self._features[:, 1:]

    @property
    def _features_dc(self):
        return self._features[:, :1]

    @property
    def _features_rest(self):
        return self._features[:, 1:]

    @property
    def get_opacity(self):
        return self._leaves["opacity"]

    @property
    def get_scaling(self):
        return self._leaves["scaling"]

    @property
    def get_rotation(self):
        return self._leaves["rotation"]

    def get_covariance(self, scaling_modifier: float = 1.0):
        raise NotImplementedError("compute_cov3D_python: the rasterizer builds the covariance from scales and rotations itself")

    def oneupSHdegree(self):
        if self.active_sh_degree < self.max_sh_degree:
            self.active_sh_degree += 1

    # ---- optimizer (training_setup :176-211, update_learning_rate :213-223, train.py:178-186) -------------------------
    def training_setup(self, training_args):
        g = lambda k: float(getattr(training_args, k))
        self.percent_dense = g("percent_dense")
        dev = self.store.device
        self.xyz_gradient_accum = torch.zeros((self.P, 1), device=dev)
        self.denom = torch.zeros((self.P, 1), device=dev)
        self.lr = {"xyz": g("position_lr_init") * self.spatial_lr_scale, "f_dc": g("feature_lr"), "f_rest": g("feature_lr") / 20.0,
                   "opacity": g("opacity_lr"), "scaling": g("scaling_lr"), "rotation": g("rotation_lr")}
        self._xyz_sched = dict(lr_init=g("position_lr_init") * self.spatial_lr_scale,
                               lr_final=g("position_lr_final") * self.spatial_lr_scale,
                               lr_delay_mult=g("position_lr_delay_mult"), max_steps=int(g("position_lr_max_steps")))
        self.step_count = 0
        self.group_steps = {n: 0 for n in GROUPS}
        self._skip_next = set()
        self.exp_avg.zero_()
        self.exp_avg_sq.zero_()
        if self._exposure is not None:       # gaussian_model.py:201,208-211 (train.py:178-179 steps it)
            self.exposure_optimizer = torch.optim.Adam([self._exposure])
            if hasattr(training_args, "exposure_lr_init"):
                self._exposure_sched = dict(lr_init=g("exposure_lr_init"), lr_final=g("exposure_lr_final"),
                                            lr_delay_steps=int(g("exposure_lr_delay_steps")), lr_delay_mult=g("exposure_lr_delay_mult"),
                                            max_steps=int(g("iterations")))

    def update_learning_rate(self, iteration: int) -> float:
        if self.pretrained_exposures is None and self.exposure_optimizer is not None and self._exposure_sched is not None:
            for param_group in self.exposure_optimizer.param_groups:
                param_group["lr"] = expon_lr(iteration, **self._exposure_sched)
        self.lr["xyz"] = expon_lr(iteration, **self._xyz_sched)
        return self.lr["xyz"]

    def step_sizes(self):
        """(step_size, sqrt(1 - beta2^t)) per group for the NEXT step, as torch.optim.Adam computes them in double, each
        group with its own step count."""
        if self.optimizer_type == "sparse_adam":
            # [RECALL, UNVERIFIED_VS_REFERENCE] the accel branch's SparseGaussianAdam applies no bias correction
            return [self.lr[n] for n in GROUPS], [1.0] * len(GROUPS)
        t = {n: self.group_steps[n] + 1 for n in GROUPS}
        return ([self.lr[n] / (1.0 - self.betas[0] ** t[n]) for n in GROUPS],
                [math.sqrt(1.0 - self.betas[1] ** t[n]) for n in GROUPS])

    def optimizer_step(self, visible: Optional[torch.Tensor] = None):
        """``optimizer.step()``: consumes ``self.grad`` (dLoss/d activated), updates the store and both moments in place and
        rewrites the activated tensors.  ``visible`` ([P] bool): rows with False are left untouched (train.py:181-183).

        Groups whose parameter ``densify_and_prune`` / ``reset_opacity`` replaced AFTER the gradients were computed are
        SKIPPED: in the reference the fresh nn.Parameter has ``grad is None`` when train.py:178-186 reaches
        ``optimizer.step()``, so Adam neither updates it, nor decays its moments, nor advances its step count.  The store
        cannot see a backward pass happen, so the contract is explicit: whoever fills ``self.grad`` calls
        ``gradients_ready()`` afterwards (``gaussian_renderer.render_views_backward`` does); replacements made after that
        call are the ones skipped here."""
        skip = sum(1 << k for k, n in enumerate(GROUPS) if n in self._skip_next)
        self._skip_next = set()
        if skip == (1 << len(GROUPS)) - 1:
            return
        ss, b2s = self.step_sizes()
        _dgr.adam_step(self.store, self.grad, self.exp_avg, self.exp_avg_sq, self.act, self.P, self.sh_coeffs, ss, self.betas[0],
                       self.betas[1], self.eps, b2s, visible, skip_groups=skip)
        for k, n in enumerate(GROUPS):
            if not (skip >> k) & 1:
                self.group_steps[n] += 1
        self.step_count += 1

    def gradients_ready(self):
        """``self.grad`` now holds the gradients of the CURRENT parameters (a backward pass has just run): replacements made
        before this point no longer make ``optimizer_step`` skip anything."""
        self._skip_next = set()

    def gradient_bucket(self):
        """The gradient buffer as the data-parallel bucket (same interface as gaussian_renderer.GradientBucket)."""
        return _StoreBucket(self)

    def zero_grad(self):
        self.grad.zero_()

    # ---- densification ---------------------------------------------------------------------------------------------
    def add_densification_stats(self, viewspace_grad: torch.Tensor, update_filter: torch.Tensor):
        """``viewspace_grad``: the [P,>=2] gradient of the screen-space means (``viewspace_point_tensor.grad``)."""
        self.xyz_gradient_accum[update_filter] += torch.norm(viewspace_grad[update_filter, :2], dim=-1, keepdim=True)
        self.denom[update_filter] += 1

    def densify_and_prune(self, max_grad: float, min_opacity: float, extent: float, max_screen_size, radii=None,
                          n_children: int = 2, unit_samples=None) -> Dict[str, int]:
        """Clone small / split large gaussians whose mean view-space gradient is >= max_grad, then prune the transparent and
        (when ``max_screen_size`` is set) the oversized ones -- row order, Adam-moment handling and random draw as in the
        reference (one ``torch.randn`` of [n_children * n_split, 3] from the device generator, where the reference calls
        ``torch.normal(mean=0, std=stds)`` with the same shape).  ``unit_samples``: the standard normals to use instead, a
        tensor [n_children * n_split, 3] or a callable ``rows -> tensor`` (tests replaying a recorded draw)."""
        dev = self.store.device
        if self.P == 0:
            return {"n_clone": 0, "n_split": 0, "n_pruned": 0, "P": 0}
        args, keep, (n_clone, n_split, n_pruned, P_new) = _dgr.densify_plan(
            self.store, self.exp_avg, self.exp_avg_sq, self.xyz_gradient_accum, self.denom, self.P, self.sh_coeffs, n_children,
            max_grad, self.percent_dense * extent, min_opacity, 0.1 * extent if max_screen_size else -1.0)
        if not n_split:
            unit = None
        elif unit_samples is None:
            # Data-parallel replicas must draw IDENTICAL children: a dedicated generator seeded from (densify_seed, number of
            # densifications so far) instead of the process-wide one, whose state depends on everything else a rank has drawn.
            gen = torch.Generator(device=dev)
            gen.manual_seed((int(self.densify_seed) * 1000003 + self._densify_calls) & 0x7FFFFFFFFFFFFFFF)
            unit = torch.randn((n_children * n_split, 3), device=dev, generator=gen)
        else:
            unit = unit_samples(n_children * n_split) if callable(unit_samples) else unit_samples
            unit = unit.to(device=dev, dtype=torch.float32).reshape(n_children * n_split, 3).contiguous()
        old = (self.store, self.exp_avg, self.exp_avg_sq)
        total = store_offsets(P_new, self.sh_coeffs)["total"]
        new = [torch.empty(total, dtype=torch.float32, device=dev) for _ in range(3)]
        _dgr.densify_apply(args, unit, n_split, P_new, *new)
        del keep, old
        self.P = P_new
        self.store, self.exp_avg, self.exp_avg_sq = new
        self.grad = torch.zeros(total, dtype=torch.float32, device=dev)
        self.act = torch.empty(8 * P_new, dtype=torch.float32, device=dev)
        self._bind()
        self._reactivate()
        self.xyz_gradient_accum = torch.zeros((P_new, 1), device=dev)
        self.denom = torch.zeros((P_new, 1), device=dev)
        self.max_radii2D = torch.zeros(P_new, device=dev)
        self._densify_calls += 1
        self._skip_next = set(GROUPS)          # every parameter was replaced: the pending optimizer_step() is a no-op (see there)
        return {"n_clone": n_clone, "n_split": n_split, "n_pruned": n_pruned, "P": P_new}

    def prune_points(self, mask: torch.Tensor) -> int:
        """``prune_points(mask)`` of the reference (gaussian_model.py:349-364): rows with ``mask`` True (bool [P]) are removed,
        the survivors keep their order, their parameters and both Adam moments, and every group keeps its step count.  The
        densification statistics (``xyz_gradient_accum``, ``denom``, ``max_radii2D``) are gathered the same way; exposures are
        untouched.  As in the reference, where every parameter becomes a fresh nn.Parameter with ``grad None``, the pending
        ``optimizer_step()`` skips every group.  A plan (one read-back, of the new count) plus ONE gather of the store and both
        moments (gsb_prune_plan / gsb_prune_apply).  Returns the new number of gaussians.

        A typical mask is a contribution score: e.g. ``stats.weight_max < tau`` for a ``ContributionStats`` accumulated over the
        training views (INTEGRATION.md)."""
        if not isinstance(mask, torch.Tensor) or mask.dtype != torch.bool or tuple(mask.shape) != (self.P,):
            raise ValueError(f"prune_points: mask must be a bool tensor of shape ({self.P},)")
        dev = self.store.device
        if mask.device != dev:
            raise ValueError(f"prune_points: mask lives on {mask.device}, the store on {dev}")
        P, M = self.P, self.sh_coeffs
        scratch, P_new = _dgr.prune_plan(mask, P)
        total = store_offsets(P_new, M)["total"]
        new = [torch.empty(total, dtype=torch.float32, device=dev) for _ in range(3)]
        _dgr.prune_apply(scratch, P, M, self.store, self.exp_avg, self.exp_avg_sq, P_new, *new)
        # the per-gaussian statistics: survivor i goes to row (number of survivors before i), removed rows to a spare row P_new
        keep = ~mask
        dest = torch.where(keep, torch.cumsum(keep, 0) - 1, torch.full((), P_new, dtype=torch.int64, device=dev))

        def gather(t):
            if t is None:
                return None
            out = t.new_empty((P_new + 1,) + tuple(t.shape[1:]))
            out.index_copy_(0, dest, t)
            return out[:P_new]

        self.xyz_gradient_accum, self.denom = gather(self.xyz_gradient_accum), gather(self.denom)
        self.max_radii2D = gather(self.max_radii2D)
        self.P = P_new
        self.store, self.exp_avg, self.exp_avg_sq = new
        self.grad = torch.zeros(total, dtype=torch.float32, device=dev)
        self.act = torch.empty(8 * P_new, dtype=torch.float32, device=dev)
        self._bind()
        self._reactivate()
        self._skip_next = set(GROUPS)          # every parameter was replaced: the pending optimizer_step() is a no-op (see there)
        return P_new

    def reset_opacity(self):
        """raw opacity <- logit(min(sigmoid(raw), 0.01)); the group's Adam moments restart at zero (:258-261, :302-314)."""
        o = store_offsets(self.P, self.sh_coeffs)
        a, n = o["opacity"], self.P
        with torch.no_grad():
            y = torch.minimum(torch.sigmoid(self.store[a:a + n]), torch.full((), 0.01, device=self.store.device))
            self.store[a:a + n] = torch.log(y / (1.0 - y))
            self.exp_avg[a:a + n] = 0.0
            self.exp_avg_sq[a:a + n] = 0.0
        self._skip_next.add("opacity")         # replace_tensor_to_optimizer: a fresh parameter, grad None until the next backward
        self._reactivate()

    # ---- point_cloud.ply (save_ply :239-256, load_ply :263-314) --------------------------------------------------------
    def save_ply(self, path: str):
        from .ply import write_gaussian_ply
        c = lambda t: t.detach().cpu().numpy()
        write_gaussian_ply(path, c(self._xyz), c(self._features_dc), c(self._features_rest), c(self._opacity), c(self._scaling),
                           c(self._rotation))

    def load_ply(self, path: str, device="cuda", spatial_lr_scale: Optional[float] = None, use_train_test_exp: bool = False):
        from .ply import read_gaussian_ply
        if use_train_test_exp:               # gaussian_model.py:264-274: <model>/exposure.json two levels above the ply
            import os
            self.load_exposures(os.path.join(os.path.dirname(path), os.pardir, os.pardir, "exposure.json"), device=device)
        a = {k: torch.from_numpy(v).to(device) for k, v in read_gaussian_ply(path, self.max_sh_degree).items()}
        self.create_from_tensors(a["xyz"], a["features_dc"], a["features_rest"], a["scaling"], a["rotation"], a["opacity"],
                                 self.spatial_lr_scale if spatial_lr_scale is None else spatial_lr_scale)
        self.active_sh_degree = self.max_sh_degree
        return self

    # ---- checkpoint (capture :63-76 / restore :78-99) -----------------------------------------------------------------
    def _group_views(self, buf):
        """A flat buffer of the store's layout as the reference's six tensors."""
        P, M, o = self.P, self.sh_coeffs, store_offsets(self.P, self.sh_coeffs)
        feat = buf[o["features"]:o["opacity"]].view(P, M, 3)
        return {"xyz": buf[:3 * P].view(P, 3), "f_dc": feat[:, :1], "f_rest": feat[:, 1:], "opacity": buf[o["opacity"]:o["scaling"]].view(P, 1),
                "scaling": buf[o["scaling"]:o["rotation"]].view(P, 3), "rotation": buf[o["rotation"]:].view(P, 4)}

    def capture(self):
        """The reference's checkpoint tuple (gaussian_model.py:63-76), optimizer state in ``torch.optim.Adam.state_dict()``
        form (six single-parameter groups in the reference's order, per-parameter ``step`` / ``exp_avg`` / ``exp_avg_sq``), so
        that ``torch.save((gaussians.capture(), iteration), path)`` of train.py:212 writes a file the reference can load."""
        raw, m, v = self._group_views(self.store), self._group_views(self.exp_avg), self._group_views(self.exp_avg_sq)
        c = lambda t: t.detach().clone().contiguous()
        state = {k: {"step": torch.tensor(float(self.group_steps[n])), "exp_avg": c(m[n]), "exp_avg_sq": c(v[n])}
                 for k, n in enumerate(GROUPS) if self.group_steps[n] > 0}
        groups = [{"lr": self.lr.get(n, 0.0), "name": n, "betas": tuple(self.betas), "eps": self.eps, "weight_decay": 0, "amsgrad": False,
                   "maximize": False, "foreach": None, "capturable": False, "differentiable": False, "fused": None, "params": [k]}
                  for k, n in enumerate(GROUPS)]
        return (self.active_sh_degree, c(raw["xyz"]), c(raw["f_dc"]), c(raw["f_rest"]), c(raw["scaling"]), c(raw["rotation"]),
                c(raw["opacity"]), self.max_radii2D.clone(), None if self.xyz_gradient_accum is None else self.xyz_gradient_accum.clone(),
                None if self.denom is None else self.denom.clone(), {"state": state, "param_groups": groups}, self.spatial_lr_scale)

    def restore(self, model_args, training_args=None):
        """``restore(model_args, training_args)`` of the reference (gaussian_model.py:78-99): ``model_args`` is the tuple written by
        the reference's or this class's ``capture()`` -- the per-group Adam state (moments and step counts) goes into the flat
        moments.  (As in the reference, the per-image exposures are not part of the tuple: they travel in exposure.json.)"""
        if not isinstance(model_args, (tuple, list)) or len(model_args) != 12:
            raise ValueError("restore: expected the 12-tuple of GaussianModel.capture()")
        (active, xyz, f_dc, f_rest, scaling, rotation, opacity, max_radii2D, grad_accum, denom, opt_dict, spatial) = model_args
        if int(f_rest.shape[1]) + 1 != self.sh_coeffs:
            raise ValueError("checkpoint was written with another SH degree")
        dev = xyz.device
        t = lambda x: x.detach().to(dev, torch.float32)
        self.create_from_tensors(t(xyz), t(f_dc), t(f_rest), t(scaling), t(rotation), t(opacity), float(spatial))
        self.active_sh_degree = int(active)
        if training_args is not None:
            self.training_setup(training_args)
        self.max_radii2D = max_radii2D.detach().to(dev).clone()
        self.xyz_gradient_accum = None if grad_accum is None else grad_accum.detach().to(dev).clone()
        self.denom = None if denom is None else denom.detach().to(dev).clone()
        m, v = self._group_views(self.exp_avg), self._group_views(self.exp_avg_sq)
        names = [g.get("name") for g in opt_dict.get("param_groups", [])]
        for k, n in enumerate(GROUPS):
            idx = opt_dict["param_groups"][names.index(n)]["params"][0] if n in names else k
            st = opt_dict.get("state", {}).get(idx)
            if st is None:
                m[n].zero_(); v[n].zero_(); self.group_steps[n] = 0
                continue
            m[n].copy_(st["exp_avg"].to(dev).view_as(m[n]))
            v[n].copy_(st["exp_avg_sq"].to(dev).view_as(v[n]))
            self.group_steps[n] = int(float(st["step"]))
        self.step_count = max(self.group_steps.values())
        self._skip_next = set()
        for g in opt_dict.get("param_groups", []):
            if g.get("name") in self.lr:
                self.lr[g["name"]] = float(g["lr"])
        return self
