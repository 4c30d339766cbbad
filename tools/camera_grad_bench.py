"""Cost of the camera gradients (gsb_backward_camera / gsb_backward_batch_camera) on bench.py's raster workload: 1 M
gaussians, 1080p, 8 views per step, SH degree 3, fused L1 loss, view-batch step (render_views_backward).

Two legs are timed alternately in one process (CUDA events around K steps):
  plain   -- the cameras and the background are constants (bench.py's default leg);
  camera  -- every view's world_view_transform / full_proj_transform / camera_center and the background require grad, so the
             backward also returns the camera gradients and chains them into those tensors.
Reported: ms per step and Mpix/s of each leg, the per-view time of the backward preprocess kernel and of the two camera
reduction kernels (gsb_kernel_time), and the single-view drop-in path -- render() + backward() per camera -- with a camera
built in torch from a learnable se(3) pose offset, next to the same path with a constant camera and with camera tensors that
are leaves requiring grad.  One JSON line.

    python tools/camera_grad_bench.py                                   # needs an H100
    python tools/camera_grad_bench.py --gaussians 20000 --width 320 --height 192 --steps 5
"""
import argparse
import gc
import json
import math
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (ROOT, os.path.join(ROOT, "gaussian-splatting_b200")):
    if _p not in sys.path:
        sys.path.insert(0, _p)
import bench  # noqa: E402
import diff_gaussian_rasterization as dgr  # noqa: E402
from gaussian_renderer import GradientBucket, render, render_views_backward  # noqa: E402
from gaussian_renderer.synthetic import make_scene  # noqa: E402

KERNELS = ("preprocess_bwd", "camera_bg_partial", "camera_grad_reduce")


def parse(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--gaussians", type=int, default=1_000_000)
    ap.add_argument("--width", type=int, default=1920)
    ap.add_argument("--height", type=int, default=1080)
    ap.add_argument("--views", type=int, default=8)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=2, help="alternations of the two legs")
    return ap.parse_args(argv)


def projection_factor(R0, T0, fovx, fovy, device):
    """The projection matrix P of full_proj_transform = world_view_transform @ P (transposed convention), float32."""
    from gaussian_renderer.synthetic import camera_matrices
    wvt0, full0, _ = camera_matrices(R0, T0, fovx, fovy)
    return torch.linalg.solve(wvt0.double(), full0.double()).float().to(device)


def pose_matrices(R0, T0, proj, w, t):
    """world_view_transform, full_proj_transform, camera_center as torch functions of an se(3) offset (w, t) of the camera
    (R0, T0): scene/cameras.py's construction in differentiable form."""
    dt, dev = w.dtype, w.device
    z = torch.zeros((), dtype=dt, device=dev)
    K = torch.stack([torch.stack([z, -w[2], w[1]]), torch.stack([w[2], z, -w[0]]), torch.stack([-w[1], w[0], z])])
    dR = torch.matrix_exp(K)
    Rw2c = dR @ torch.as_tensor(R0, dtype=dt, device=dev).T
    tc = dR @ torch.as_tensor(T0, dtype=dt, device=dev) + t
    Rt = torch.cat([torch.cat([Rw2c, tc[:, None]], 1), torch.tensor([[0.0, 0.0, 0.0, 1.0]], dtype=dt, device=dev)], 0)
    wvt = Rt.T
    return wvt, wvt @ proj, -(Rw2c.T @ tc)


def main(argv=None):
    a = parse(argv)
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    V, H, W = a.views, a.height, a.width
    pc = bench.BenchGaussians(make_scene(a.gaussians, seed=0, log_scale_mean=bench.LOG_SCALE_MEAN), 3, dev)
    bucket = GradientBucket(pc.parameters())
    pipe = bench.Pipe()
    fovx = math.radians(60.0)
    poses = [bench.view_pose(i, 3.0) for i in range(V)]
    cams = {leg: [bench.BenchCamera(W, H, fovx, *poses[i], dev) for i in range(V)] for leg in ("plain", "camera")}
    bgs = {"plain": torch.zeros(3, device=dev), "camera": torch.zeros(3, device=dev, requires_grad=True)}
    for cm in cams["camera"]:
        for t in (cm.world_view_transform, cm.full_proj_transform, cm.camera_center):
            t.requires_grad_(True)
    gen = torch.Generator().manual_seed(1234)
    gts = [torch.rand(3, H, W, generator=gen).to(dev) for _ in range(V)]

    def loss_fn(img, _invdepth, i, grad_out=None):
        return dgr.l1_loss_and_grad(img, gts[i], grad_out=grad_out)

    def step(leg):
        render_views_backward(cams[leg], pc, pipe, bgs[leg], loss_fn, loss_returns_grad=True, overwrite=True)

    def timed(leg, steps):
        gc.collect()
        gc.disable()
        try:
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(steps):
                step(leg)
            e1.record()
            torch.cuda.synchronize()
        finally:
            gc.enable()
        return e0.elapsed_time(e1) / steps

    for leg in ("plain", "camera"):
        for _ in range(a.warmup):
            step(leg)
    ms = {"plain": [], "camera": []}
    for _ in range(a.rounds):
        for leg in ("plain", "camera"):
            ms[leg].append(round(timed(leg, a.steps), 4))

    kernels = {}
    for leg in ("plain", "camera"):
        dgr.set_option("time_kernels", 2)
        dgr.kernel_time("", reset=True)
        for _ in range(2):
            step(leg)
        torch.cuda.synchronize()
        kernels[leg] = {n: round(dgr.kernel_time(n)[0] / (2 * V), 4) for n in KERNELS}
        dgr.kernel_time("", reset=True)
        dgr.set_option("time_kernels", 0)

    # single-view drop-in path: render() + backward() per camera with (a) a constant camera, (b) camera tensors that are leaves
    # requiring grad (the rasterizer's share of the cost), (c) a camera built in torch from a learnable pose offset every view
    # (b plus torch's own kernels for the construction and its backward)
    w = torch.zeros(3, device=dev, requires_grad=True)
    tr = torch.zeros(3, device=dev, requires_grad=True)
    projs = [projection_factor(*poses[i], cams["plain"][i].FoVx, cams["plain"][i].FoVy, dev) for i in range(V)]
    sv_cam = bench.BenchCamera(W, H, fovx, *poses[0], dev)
    bg0 = torch.zeros(3, device=dev)

    def one_view(i, mode):
        for p in pc.parameters():
            p.grad = None
        cm = {"constant_camera": cams["plain"], "camera_leaves": cams["camera"]}.get(mode, cams["plain"])[i % V]
        if mode == "learnable_pose":
            sv_cam.world_view_transform, sv_cam.full_proj_transform, sv_cam.camera_center = pose_matrices(
                *poses[i % V], projs[i % V], w, tr)
            cm = sv_cam
        (render(cm, pc, pipe, bg0)["render"] - gts[i % V]).abs().mean().backward()

    sv = {}
    n_sv = max(V, min(a.steps * V, 64))
    for _ in range(a.rounds):
        for mode in ("constant_camera", "camera_leaves", "learnable_pose"):
            for i in range(V):
                one_view(i, mode)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for i in range(n_sv):
                one_view(i, mode)
            e1.record()
            torch.cuda.synchronize()
            sv.setdefault(mode, []).append(round(e0.elapsed_time(e1) / n_sv, 4))
    del bucket

    try:
        gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception:
        gpu = torch.cuda.get_device_name(dev)
    mpix = V * H * W / 1e6
    best = {leg: min(v) for leg, v in ms.items()}
    line = {"metric": "camera gradient overhead, view-batch step", "gpu": gpu,
            "config": {"gaussians": a.gaussians, "width": W, "height": H, "views": V, "sh_degree": 3, "steps": a.steps,
                       "rounds": a.rounds},
            "ms_per_step": ms, "mpix_s": {leg: round(mpix / (m / 1e3), 1) for leg, m in best.items()},
            "overhead_frac": round(best["camera"] / best["plain"] - 1.0, 4),
            "kernel_ms_per_view": kernels,
            "single_view_ms": sv}
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
