"""Generates tests/golden/reference_prune.npz by running the reference's OWN scene/gaussian_model.py (prune_points :349-364,
_prune_optimizer :330-347) on the CPU in this container, as GaussianModel(3) with torch.optim.Adam and as
GaussianModel(3, "sparse_adam") with tests/sparse_adam_oracle.py's optimizer (see make_golden_sparse.py), stepped in
train.py's order.

Per mode (prefix "a_" default, "s_" sparse_adam):
  2 steps | backward, prune_points(mask1), optimizer.step() (skipped: every parameter is fresh, grad None) | 1 step |
  prune_points(mask2) | 1 step | and, from that state, the edge masks on deep copies: none removed, all removed, only the first
  row, only the last row.
The reference's prune_points also indexes `tmp_radii`, which only densify_and_prune sets: it is set here before pruning.
Recorded after every stage: the raw parameters, both moments, every group's step count and the densification tensors
(xyz_gradient_accum, denom, max_radii2D).  Stand-ins for `plyfile` / `simple_knn._C` / `diff_gaussian_rasterization` and the
CPU torch.zeros as in make_golden_model.py / make_golden_sparse.py; the reference code itself runs unmodified.

    python tests/golden/make_golden_prune.py
"""
import copy
import importlib.util
import os
import sys
import types
from argparse import ArgumentParser

import numpy as np
import torch

REF = "/root/reference"
ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
from sparse_adam_oracle import SparseGaussianAdamOracle  # noqa: E402

sys.path.insert(0, REF)
_zeros = torch.zeros


def _cpu_zeros(*a, **k):
    k.pop("device", None)
    return _zeros(*a, **k)


torch.zeros = _cpu_zeros
ply = types.ModuleType("plyfile")
ply.PlyData = ply.PlyElement = object
sys.modules["plyfile"] = ply
knn = types.ModuleType("simple_knn")
knn_c = types.ModuleType("simple_knn._C")
knn_c.distCUDA2 = None
sys.modules["simple_knn"], sys.modules["simple_knn._C"] = knn, knn_c
dgr = types.ModuleType("diff_gaussian_rasterization")
dgr.SparseGaussianAdam = SparseGaussianAdamOracle
sys.modules["diff_gaussian_rasterization"] = dgr

spec = importlib.util.spec_from_file_location("ref_gaussian_model", os.path.join(REF, "scene", "gaussian_model.py"))
GM = importlib.util.module_from_spec(spec)
spec.loader.exec_module(GM)
from arguments import OptimizationParams  # noqa: E402

opt = OptimizationParams(ArgumentParser())
out = {}
RAW = ("_xyz", "_features_dc", "_features_rest", "_scaling", "_rotation", "_opacity")
names = ("xyz", "features", "opacity", "scaling", "rotation")
shapes = {"xyz": (3,), "features": (16, 3), "opacity": (1,), "scaling": (3,), "rotation": (4,)}
P0, EXTENT = 40, 4.0


def run(mode, prefix, g):
    pc = GM.GaussianModel(3, mode)
    pc.active_sh_degree = 3
    pc.spatial_lr_scale = EXTENT
    nnP = torch.nn.Parameter
    pc._xyz = nnP(torch.randn(P0, 3, generator=g))
    pc._features_dc = nnP(torch.randn(P0, 1, 3, generator=g) * 0.5)
    pc._features_rest = nnP(torch.randn(P0, 15, 3, generator=g) * 0.1)
    pc._scaling = nnP(torch.randn(P0, 3, generator=g) * 1.0 - 3.6)
    pc._rotation = nnP(torch.randn(P0, 4, generator=g))
    pc._opacity = nnP(torch.rand(P0, 1, generator=g) * 9.0 - 6.5)
    pc.max_radii2D = torch.zeros(P0)
    pc.pretrained_exposures = None
    pc._exposure = nnP(torch.eye(3, 4)[None].repeat(1, 1, 1))
    for k in RAW:
        out[prefix + "init" + k] = getattr(pc, k).detach().numpy().copy()
    pc.training_setup(opt)
    assert (mode == "sparse_adam") == isinstance(pc.optimizer, SparseGaussianAdamOracle)
    W = {n: torch.randn(P0, *shapes[n], generator=g) * 1e-3 for n in names}
    U = {n: torch.randn(P0, *shapes[n], generator=g) * 1e-3 for n in names}
    for n in names:
        out[prefix + "w_" + n], out[prefix + "u_" + n] = W[n].numpy(), U[n].numpy()

    def backward(model, iteration):
        model.update_learning_rate(iteration)
        act = {"xyz": model.get_xyz, "features": model.get_features, "opacity": model.get_opacity, "scaling": model.get_scaling,
               "rotation": model.get_rotation}
        P = model.get_xyz.shape[0]
        loss = sum((W[n][:P] * act[n]).sum() + 0.5 * (U[n][:P] * act[n] ** 2).sum() for n in names)
        loss.backward()

    def step(model, tag):
        if mode == "sparse_adam":       # train.py:181-183: step(visible, N)
            N = model.get_xyz.shape[0]
            vis = torch.rand(N, generator=g) < 0.5
            out[f"{prefix}{tag}_vis"] = vis.numpy().copy()
            model.optimizer.step(vis, N)
        else:
            model.optimizer.step()
        model.optimizer.zero_grad(set_to_none=True)

    def snapshot(model, tag):
        t = prefix + tag
        out[t + "_P"] = np.int64(model.get_xyz.shape[0])
        for k in RAW:
            out[t + k] = getattr(model, k).detach().numpy().copy()
        for grp in model.optimizer.param_groups:
            st = model.optimizer.state.get(grp["params"][0], None)
            out[f"{t}_m_{grp['name']}"] = st["exp_avg"].numpy().copy()
            out[f"{t}_v_{grp['name']}"] = st["exp_avg_sq"].numpy().copy()
            out[f"{t}_step_{grp['name']}"] = np.float64(float(st["step"]) if "step" in st else 0.0)
        out[t + "_accum"] = model.xyz_gradient_accum.numpy().copy()
        out[t + "_denom"] = model.denom.numpy().copy()
        out[t + "_max_radii2D"] = model.max_radii2D.numpy().copy()

    def mask_of(model, tag, p):
        m = torch.rand(model.get_xyz.shape[0], generator=g) < p
        out[f"{prefix}{tag}_mask"] = m.numpy().copy()
        return m

    def set_stats(model, tag):
        P = model.get_xyz.shape[0]
        model.xyz_gradient_accum = torch.rand(P, 1, generator=g) * 1e-3
        model.denom = torch.randint(0, 5, (P, 1), generator=g).float()
        model.max_radii2D = torch.rand(P, generator=g) * 40.0
        model.tmp_radii = torch.zeros(P)           # prune_points indexes it (densify_and_prune sets it, :455)
        out[f"{prefix}{tag}_in_accum"] = model.xyz_gradient_accum.numpy().copy()
        out[f"{prefix}{tag}_in_denom"] = model.denom.numpy().copy()
        out[f"{prefix}{tag}_in_max_radii2D"] = model.max_radii2D.numpy().copy()

    it = 0
    for _ in range(2):
        it += 1
        backward(pc, it)
        step(pc, f"s{it}")
    # train.py order: backward, prune (every parameter fresh, grad None), optimizer.step() -- a no-op
    it += 1
    backward(pc, it)
    set_stats(pc, "p1")
    pc.prune_points(mask_of(pc, "p1", 0.3))
    step(pc, "p1")
    snapshot(pc, "p1")
    it += 1
    backward(pc, it)
    step(pc, "s4")
    snapshot(pc, "s4")
    set_stats(pc, "p2")
    pc.prune_points(mask_of(pc, "p2", 0.4))
    snapshot(pc, "p2")
    it += 1
    backward(pc, it)
    step(pc, "s5")
    snapshot(pc, "s5")
    out[prefix + "iterations"] = np.int64(it)
    P = pc.get_xyz.shape[0]
    set_stats(pc, "e")
    edges = {"none": torch.zeros(P, dtype=torch.bool), "all": torch.ones(P, dtype=torch.bool),
             "first": torch.arange(P) == 0, "last": torch.arange(P) == P - 1}
    for name, m in edges.items():
        c = copy.deepcopy(pc)
        c.prune_points(m)
        out[f"{prefix}e_{name}_mask"] = m.numpy().copy()
        snapshot(c, f"e_{name}")
    print(mode, ": P", P0, "->", out[prefix + "p1_P"], "->", out[prefix + "p2_P"])


run("default", "a_", torch.Generator().manual_seed(1357))
run("sparse_adam", "s_", torch.Generator().manual_seed(2468))
OPT = ("position_lr_init", "position_lr_final", "position_lr_delay_mult", "position_lr_max_steps", "feature_lr", "opacity_lr",
       "scaling_lr", "rotation_lr", "percent_dense", "densify_grad_threshold")
for k in OPT:
    out["opt_" + k] = np.float64(getattr(opt, k))
dst = os.path.join(os.path.dirname(os.path.abspath(__file__)), "reference_prune.npz")
np.savez_compressed(dst, **out)
print("wrote", dst, len(out), "arrays,", os.path.getsize(dst) // 1024, "KiB")
