"""Cost of the rendered feature maps (gsb_render_features + the feature pass of the backward) on bench.py's raster workload:
1 M gaussians, 1080p, 8 views per step, SH degree 3, fused L1 image loss, view-batch step (render_views_backward).

For each channel count C (default 8, 16, 32) one process alternates, with CUDA events around K steps:
  plain    -- the L1 image loss (bench.py's default leg);
  features -- the same loss plus an L1 of the feature map against a fixed random target (features=..., the loss returning
              its own feature-map gradient), so every step also runs render_features and render_features_bwd.
Also reported: the per-view time of render_features and render_features_bwd (gsb_kernel_time), and the single-view drop-in
path -- render(features=...) + backward() per camera against the workaround it replaces, ceil(C/3) render() calls with
colors_precomp = three feature channels and bg 0 -- alternated in the same process.  The card's name and power limit are read
in the same run.  One JSON line per C.

    python tools/feature_bench.py                                         # needs an H100
    python tools/feature_bench.py --gaussians 20000 --width 320 --height 192 --steps 5 --channels 8
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

KERNELS = ("render_features", "render_features_bwd", "render_bwd")
LEGS = ("plain", "features")


def parse(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--gaussians", type=int, default=1_000_000)
    ap.add_argument("--width", type=int, default=1920)
    ap.add_argument("--height", type=int, default=1080)
    ap.add_argument("--views", type=int, default=8)
    ap.add_argument("--channels", type=int, nargs="+", default=[8, 16, 32])
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=2, help="alternations of the legs")
    return ap.parse_args(argv)


def _timed(fn, n):
    gc.collect()
    gc.disable()
    try:
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for i in range(n):
            fn(i)
        e1.record()
        torch.cuda.synchronize()
    finally:
        gc.enable()
    return e0.elapsed_time(e1) / n


def main(argv=None):
    a = parse(argv)
    if not torch.cuda.is_available():
        raise SystemExit("feature_bench.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    V, H, W = a.views, a.height, a.width
    pc = bench.BenchGaussians(make_scene(a.gaussians, seed=0, log_scale_mean=bench.LOG_SCALE_MEAN), 3, dev)
    P = int(pc.get_xyz.shape[0])
    bucket = GradientBucket(pc.parameters())
    pipe = bench.Pipe()
    fovx = math.radians(60.0)
    cams = [bench.BenchCamera(W, H, fovx, *bench.view_pose(i, 3.0), dev) for i in range(V)]
    bg = torch.zeros(3, device=dev)
    gen = torch.Generator().manual_seed(1234)
    gts = [torch.rand(3, H, W, generator=gen).to(dev) for _ in range(V)]
    try:
        gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception:
        gpu = torch.cuda.get_device_name(dev)

    def loss_plain(img, _invdepth, i, grad_out=None):
        return dgr.l1_loss_and_grad(img, gts[i], grad_out=grad_out)

    for C in a.channels:
        feats = torch.randn(P, C, generator=gen).to(dev).requires_grad_(True)
        ftgt = torch.randn(C, H, W, generator=gen).to(dev)
        n_f = float(C * H * W)

        def loss_feat(img, _invdepth, i, grad_out=None, features=None):
            loss, g = dgr.l1_loss_and_grad(img, gts[i], grad_out=grad_out)
            diff = features - ftgt
            return loss + diff.abs().sum() / n_f, g, None, None, torch.sign(diff) / n_f

        def step(leg):
            if leg == "plain":
                render_views_backward(cams, pc, pipe, bg, loss_plain, loss_returns_grad=True, overwrite=True)
            else:
                feats.grad = None
                render_views_backward(cams, pc, pipe, bg, loss_feat, loss_returns_grad=True, overwrite=True, features=feats)

        for leg in LEGS:
            for _ in range(a.warmup):
                step(leg)
        ms = {leg: [] for leg in LEGS}
        for _ in range(a.rounds):
            for leg in LEGS:
                ms[leg].append(round(_timed(lambda _i: step(leg), a.steps), 4))

        dgr.set_option("time_kernels", 1)            # the blend-stage kernels (names render_*)
        dgr.kernel_time("", reset=True)
        for _ in range(2):
            step("features")
        torch.cuda.synchronize()
        # one launch per step covers the V views
        kernels = {n: round(dgr.kernel_time(n)[0] / (2 * V), 4) for n in KERNELS}
        dgr.kernel_time("", reset=True)
        dgr.set_option("time_kernels", 0)

        # single view: render(features=...) + backward() against ceil(C/3) colors_precomp calls (bg 0), same loss
        def new_path(i):
            for p in pc.parameters():
                p.grad = None
            feats.grad = None
            pkg = render(cams[i % V], pc, pipe, bg, features=feats)
            ((pkg["features"] - ftgt).abs().mean()).backward()

        def workaround(i):
            for p in pc.parameters():
                p.grad = None
            feats.grad = None
            loss = 0.0
            for c0 in range(0, C, 3):
                cp = feats[:, c0:c0 + 3]
                if cp.shape[1] < 3:
                    cp = torch.cat([cp, cp.new_zeros(P, 3 - cp.shape[1])], 1)
                img = render(cams[i % V], pc, pipe, bg, override_color=cp)["render"]    # render() clamps to [0, 1]
                loss = loss + (img[:min(3, C - c0)] - ftgt[c0:c0 + 3]).abs().sum()
            (loss / n_f).backward()

        sv = {}
        n_sv = max(V, min(a.steps, 16))
        for fn in (new_path, workaround):
            for i in range(V):
                fn(i)
        for _ in range(a.rounds):
            for name, fn in (("render_features", new_path), ("colors_precomp_calls", workaround)):
                sv.setdefault(name, []).append(round(_timed(fn, n_sv), 4))
        best = {leg: min(v) for leg, v in ms.items()}
        sv_best = {k: min(v) for k, v in sv.items()}
        mpix = V * H * W / 1e6
        line = {"metric": "rendered feature maps, cost", "gpu": gpu, "channels": C,
                "config": {"gaussians": a.gaussians, "width": W, "height": H, "views": V, "sh_degree": 3, "steps": a.steps,
                           "rounds": a.rounds},
                "ms_per_step": ms, "mpix_s": {leg: round(mpix / (m / 1e3), 1) for leg, m in best.items()},
                "step_overhead_frac": round(best["features"] / best["plain"] - 1.0, 4),
                "kernel_ms_per_view": kernels,
                "single_view_ms": sv,
                "single_view_speedup_vs_workaround": round(sv_best["colors_precomp_calls"] / sv_best["render_features"], 3)}
        print(json.dumps(line), flush=True)
        del feats
    del bucket


if __name__ == "__main__":
    main()
