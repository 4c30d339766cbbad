"""Generates tests/golden/reference_sparse_adam.npz by running the reference's OWN scene/gaussian_model.py as
GaussianModel(3, "sparse_adam") (/root/reference/scene/gaussian_model.py: training_setup :178-199, densify_and_prune
:452-469, reset_opacity :258-261, capture / restore :68-100) on the CPU in this container, stepped in train.py's order
(train.py:142-183): loss.backward(), then densify_and_prune or reset_opacity, then optimizer.step(visible, radii.shape[0]).

The accel rasterizer that provides SparseGaussianAdam is not part of /root/reference.  Its place is taken by
tests/sparse_adam_oracle.py's SparseGaussianAdamOracle, handed to the reference file through a stand-in `diff_gaussian_rasterization`
module (the reference imports it at :26).  So the fixture pins what the reference CLASS does with such an optimizer --
which rows exist in which order after each piece of optimizer-state surgery, the state keys, the checkpoint round trip --
and the update rule as the oracle states it (UNVERIFIED_VS_REFERENCE).  Stand-ins for `plyfile` / `simple_knn._C` and the
CPU torch.zeros as in make_golden_model.py; the reference code itself runs unmodified.  Kept small (24 gaussians, growing
to a few dozen): the state keys, step counts and visibility masks are recorded after every stage, parameters and moments
after the stages FULL lists (the densification that follows three steps, the opacity reset, one step after the checkpoint
round trip).

    python tests/golden/make_golden_sparse.py
"""
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

g = torch.Generator().manual_seed(2468)
P0, EXTENT = 24, 4.0
pc = GM.GaussianModel(3, "sparse_adam")
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
    out["init" + k] = getattr(pc, k).detach().numpy().copy()
pc.training_setup(opt)
assert isinstance(pc.optimizer, SparseGaussianAdamOracle), "the reference class fell back to torch.optim.Adam"

names = ("xyz", "features", "opacity", "scaling", "rotation")
shapes = {"xyz": (3,), "features": (16, 3), "opacity": (1,), "scaling": (3,), "rotation": (4,)}
MAXP = 2 * P0
W = {n: torch.randn(MAXP, *shapes[n], generator=g) * 1e-3 for n in names}
U = {n: torch.randn(MAXP, *shapes[n], generator=g) * 1e-3 for n in names}
for n in names:
    out["w_" + n], out["u_" + n] = W[n].numpy(), U[n].numpy()


def backward(model, iteration):
    model.update_learning_rate(iteration)
    act = {"xyz": model.get_xyz, "features": model.get_features, "opacity": model.get_opacity, "scaling": model.get_scaling,
           "rotation": model.get_rotation}
    P = model.get_xyz.shape[0]
    loss = sum((W[n][:P] * act[n]).sum() + 0.5 * (U[n][:P] * act[n] ** 2).sum() for n in names)
    loss.backward()


def step(model, tag):
    """train.py:181-183 with radii of the view just rendered: visible = radii > 0, N = radii.shape[0]."""
    N = model.get_xyz.shape[0]
    vis = torch.rand(N, generator=g) < 0.5
    out[f"{tag}_vis"] = vis.numpy().copy()
    model.optimizer.step(vis, N)
    model.optimizer.zero_grad(set_to_none=True)


FULL = ("d", "r6", "s8")


def snapshot(model, tag):
    """{tag}_P, per group (GROUPS order) {tag}_keys (sorted state keys, "" without state) and {tag}_steps (NaN without state);
    for the FULL stages also the raw parameters and both moments."""
    out[f"{tag}_P"] = np.int64(model.get_xyz.shape[0])
    for k in RAW if tag in FULL else ():
        out[f"{tag}{k}"] = getattr(model, k).detach().numpy().copy()
    keys, steps = [], []
    for grp in model.optimizer.param_groups:
        st = model.optimizer.state.get(grp["params"][0], None)
        keys.append(",".join(sorted(st)) if st is not None else "")
        steps.append(float(st["step"]) if st is not None else float("nan"))
        if st is not None and tag in FULL:
            out[f"{tag}_m_{grp['name']}"] = st["exp_avg"].numpy().copy()
            out[f"{tag}_v_{grp['name']}"] = st["exp_avg_sq"].numpy().copy()
    assert [grp["name"] for grp in model.optimizer.param_groups] == ["xyz", "f_dc", "f_rest", "opacity", "scaling", "rotation"]
    out[f"{tag}_keys"], out[f"{tag}_steps"] = np.array(keys), np.array(steps)


it = 0
for tag in ("s1", "s2", "s3"):
    it += 1
    backward(pc, it)
    step(pc, tag)
    snapshot(pc, tag)

# backward, densify_and_prune (every parameter replaced: .grad None), step(visible, N of the rendered view): a no-op
it += 1
backward(pc, it)
P = pc.get_xyz.shape[0]
denom = torch.randint(0, 4, (P, 1), generator=g).float()
accum = torch.rand(P, 1, generator=g) * 0.0008 * denom
pc.xyz_gradient_accum, pc.denom = accum.clone(), denom.clone()
pc.max_radii2D = torch.rand(P, generator=g) * 40.0
radii = torch.randint(0, 30, (P,), generator=g).int()
out.update(dens_accum=accum.numpy(), dens_denom=denom.numpy(), dens_max_radii2D=pc.max_radii2D.numpy().copy(),
           dens_radii=radii.numpy(), dens_extent=np.float32(EXTENT), dens_seed=np.int64(77))
torch.manual_seed(77)
pc.densify_and_prune(opt.densify_grad_threshold, 0.005, EXTENT, 20, radii)
N_old = P
vis = torch.rand(N_old, generator=g) < 0.5
out["d_vis"] = vis.numpy().copy()
pc.optimizer.step(vis, N_old)
pc.optimizer.zero_grad(set_to_none=True)
snapshot(pc, "d")
print("densify: P", P, "->", pc.get_xyz.shape[0])
assert pc.get_xyz.shape[0] <= MAXP

it += 1
backward(pc, it)
step(pc, "s5")
snapshot(pc, "s5")

# backward, reset_opacity (only the opacity parameter replaced), step: five groups move
it += 1
backward(pc, it)
pc.reset_opacity()
step(pc, "r6")
snapshot(pc, "r6")

it += 1
backward(pc, it)
step(pc, "s7")
snapshot(pc, "s7")

# checkpoint round trip (train.py:188-190 / :51-53): capture(), restore() into a fresh instance, training goes on
ck = pc.capture()
pc2 = GM.GaussianModel(3, "sparse_adam")
pc2._exposure, pc2.pretrained_exposures = pc._exposure, None      # create_from_pcd / load_ply would set these
pc2.restore(ck, opt)
assert isinstance(pc2.optimizer, SparseGaussianAdamOracle)
snapshot(pc2, "c")
it += 1
backward(pc2, it)
step(pc2, "s8")
snapshot(pc2, "s8")

OPT = ("position_lr_init", "position_lr_final", "position_lr_delay_mult", "position_lr_max_steps", "feature_lr", "opacity_lr",
       "scaling_lr", "rotation_lr", "percent_dense", "densify_grad_threshold")
out["opt_names"], out["opt_values"] = np.array(OPT), np.float64([getattr(opt, k) for k in OPT])

dst = os.path.join(os.path.dirname(os.path.abspath(__file__)), "reference_sparse_adam.npz")
np.savez_compressed(dst, **out)
print("wrote", dst, len(out), "arrays,", os.path.getsize(dst) // 1024, "KiB")
