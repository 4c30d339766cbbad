"""Cost of the rendered alpha (gsb_alpha + the ALPHA instantiations of the backward blend kernel) on bench.py's raster workload:
1 M gaussians, 1080p, 8 views per step, SH degree 3, fused L1 loss, view-batch step (render_views_backward).

Two legs are timed alternately in one process (CUDA events around K steps):
  plain  -- the L1 image loss (bench.py's default leg);
  alpha  -- the same loss plus an L1 of the rendered alpha against a fixed target mask (with_alpha=True, the loss returning
            its own alpha gradient), so every step also runs gsb_alpha and the backward blend kernel with the alpha channel.
Reported: ms per step and Mpix/s of each leg, the per-view time of render_bwd in both legs and of the alpha kernel
(gsb_kernel_time), the single-view drop-in path -- render(..., return_alpha=True) + backward() per camera, next to render()
without alpha -- and the card's name and power limit, read in the same run.  One JSON line.

    python tools/alpha_bench.py                                          # needs an H100
    python tools/alpha_bench.py --gaussians 20000 --width 320 --height 192 --steps 5
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

KERNELS = ("render_bwd", "render_alpha")
LEGS = ("plain", "alpha")


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


def main(argv=None):
    a = parse(argv)
    if not torch.cuda.is_available():
        raise SystemExit("alpha_bench.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    V, H, W = a.views, a.height, a.width
    pc = bench.BenchGaussians(make_scene(a.gaussians, seed=0, log_scale_mean=bench.LOG_SCALE_MEAN), 3, dev)
    bucket = GradientBucket(pc.parameters())
    pipe = bench.Pipe()
    fovx = math.radians(60.0)
    cams = [bench.BenchCamera(W, H, fovx, *bench.view_pose(i, 3.0), dev) for i in range(V)]
    bg = torch.zeros(3, device=dev)
    gen = torch.Generator().manual_seed(1234)
    gts = [torch.rand(3, H, W, generator=gen).to(dev) for _ in range(V)]
    yy, xx = torch.meshgrid(torch.arange(H, device=dev), torch.arange(W, device=dev), indexing="ij")
    mask = (((xx - W / 2) ** 2 + (yy - H / 2) ** 2) < (H / 3) ** 2).float()[None]
    n_alpha = float(H * W)

    def loss_plain(img, _invdepth, i, grad_out=None):
        return dgr.l1_loss_and_grad(img, gts[i], grad_out=grad_out)

    def loss_alpha(img, _invdepth, i, grad_out=None, alpha=None):
        loss, g = dgr.l1_loss_and_grad(img, gts[i], grad_out=grad_out)
        diff = alpha - mask
        return loss + diff.abs().sum() / n_alpha, g, None, torch.sign(diff) / n_alpha

    def step(leg):
        if leg == "plain":
            render_views_backward(cams, pc, pipe, bg, loss_plain, loss_returns_grad=True, overwrite=True)
        else:
            render_views_backward(cams, pc, pipe, bg, loss_alpha, loss_returns_grad=True, overwrite=True, with_alpha=True)

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

    for leg in LEGS:
        for _ in range(a.warmup):
            step(leg)
    ms = {leg: [] for leg in LEGS}
    for _ in range(a.rounds):
        for leg in LEGS:
            ms[leg].append(round(timed(leg, a.steps), 4))

    kernels = {}
    for leg in LEGS:
        dgr.set_option("time_kernels", 1)            # the blend-stage kernels (names render_*)
        dgr.kernel_time("", reset=True)
        for _ in range(2):
            step(leg)
        torch.cuda.synchronize()
        # render_bwd: one launch per step covers the V views; render_alpha likewise
        kernels[leg] = {n: round(dgr.kernel_time(n)[0] / (2 * V), 4) for n in KERNELS}
        dgr.kernel_time("", reset=True)
        dgr.set_option("time_kernels", 0)

    def one_view(i, with_alpha):
        for p in pc.parameters():
            p.grad = None
        pkg = render(cams[i % V], pc, pipe, bg, return_alpha=with_alpha)
        loss = (pkg["render"] - gts[i % V]).abs().mean()
        if with_alpha:
            loss = loss + (pkg["alpha"] - mask).abs().mean()
        loss.backward()

    sv = {}
    n_sv = max(V, min(a.steps * V, 64))
    for _ in range(a.rounds):
        for mode, wa in (("render", False), ("render_return_alpha", True)):
            for i in range(V):
                one_view(i, wa)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for i in range(n_sv):
                one_view(i, wa)
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
    line = {"metric": "rendered alpha overhead, view-batch step", "gpu": gpu,
            "config": {"gaussians": a.gaussians, "width": W, "height": H, "views": V, "sh_degree": 3, "steps": a.steps,
                       "rounds": a.rounds},
            "ms_per_step": ms, "mpix_s": {leg: round(mpix / (m / 1e3), 1) for leg, m in best.items()},
            "overhead_frac": round(best["alpha"] / best["plain"] - 1.0, 4),
            "kernel_ms_per_view": kernels,
            "single_view_ms": sv}
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
