"""Cost of the contribution statistics and of prune_points on bench.py's workload: 1 M gaussians, 1080p, 8 views per step,
SH degree 3, fused L1 image loss, view-batch step (render_views_backward).

Reported, with the card's name and power limit read in the same run (one JSON line):
  kernel_ms_per_view     -- gsb_contribution's kernel time per view (gsb_kernel_time, CUDA events);
  ms_per_step            -- the view-batch step without and with contrib= (legs alternated, CUDA events around K steps);
  prune_points_ms        -- GaussianModel.prune_points at 1 M gaussians with a random half removed (plan, read-back, gather;
                            CUDA events, host included);
  after_prune            -- for information: the step time once the half with the lowest weight_max over the 8 views is gone.

    python tools/contrib_bench.py                                         # needs an H100
    python tools/contrib_bench.py --gaussians 20000 --width 320 --height 192 --steps 5
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
from gaussian_renderer import GradientBucket, render_views_backward  # noqa: E402
from gaussian_renderer.synthetic import make_scene  # noqa: E402
from gaussian_store import GaussianModel  # noqa: E402

LEGS = ("plain", "contrib")


def parse(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--gaussians", type=int, default=1_000_000)
    ap.add_argument("--width", type=int, default=1920)
    ap.add_argument("--height", type=int, default=1080)
    ap.add_argument("--views", type=int, default=8)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3, help="alternations of the legs")
    ap.add_argument("--prune_reps", type=int, default=5)
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
        raise SystemExit("contrib_bench.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    V, H, W = a.views, a.height, a.width
    scene = make_scene(a.gaussians, seed=0, log_scale_mean=bench.LOG_SCALE_MEAN)
    pipe = bench.Pipe()
    cams = [bench.BenchCamera(W, H, math.radians(60.0), *bench.view_pose(i, 3.0), dev) for i in range(V)]
    bg = torch.zeros(3, device=dev)
    gen = torch.Generator().manual_seed(1234)
    gts = [torch.rand(3, H, W, generator=gen).to(dev) for _ in range(V)]
    try:
        gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception:
        gpu = torch.cuda.get_device_name(dev)

    def loss(img, _invdepth, i, grad_out=None):
        return dgr.l1_loss_and_grad(img, gts[i], grad_out=grad_out)

    def step_times(pc):
        """{leg: [ms per step per round]}, the stats of the last contrib step"""
        bucket = GradientBucket(pc.parameters())
        P = int(pc.get_xyz.shape[0])
        st = dgr.ContributionStats(P, dev)

        def step(leg):
            render_views_backward(cams, pc, pipe, bg, loss, loss_returns_grad=True, overwrite=True,
                                  contrib=st.zero_() if leg == "contrib" else None)
        for leg in LEGS:
            for _ in range(a.warmup):
                step(leg)
        ms = {leg: [] for leg in LEGS}
        for _ in range(a.rounds):
            for leg in LEGS:
                ms[leg].append(round(_timed(lambda _i: step(leg), a.steps), 4))
        dgr.set_option("time_kernels", 2)
        dgr.kernel_time("", reset=True)
        for _ in range(2):
            step("contrib")
        torch.cuda.synchronize()
        t_ms, launches = dgr.kernel_time("contribution")
        dgr.kernel_time("", reset=True)
        dgr.set_option("time_kernels", 0)
        step("contrib")
        torch.cuda.synchronize()
        del bucket
        return ms, round(t_ms / (2 * V), 4), int(launches), st

    pc = bench.BenchGaussians(scene, 3, dev)
    ms, kernel_ms, launches, st = step_times(pc)
    best = {leg: min(v) for leg, v in ms.items()}

    # prune_points at full size, a random half removed (a fresh store per repetition)
    op = scene["opacities"].clamp(1e-4, 1 - 1e-4)
    raw = dict(xyz=scene["means3D"].to(dev), dc=scene["shs"][:, :1].to(dev), rest=scene["shs"][:, 1:].to(dev),
               scaling=torch.log(scene["scales"]).to(dev), rotation=scene["rotations"].to(dev), opacity=torch.log(op / (1 - op)).to(dev))
    mask = torch.rand(a.gaussians, device=dev, generator=torch.Generator(device=dev).manual_seed(5)) < 0.5
    prune_ms = []
    for _ in range(a.prune_reps):
        gm = GaussianModel(3).create_from_tensors(raw["xyz"], raw["dc"], raw["rest"], raw["scaling"], raw["rotation"], raw["opacity"])
        gm.xyz_gradient_accum = torch.zeros((gm.P, 1), device=dev)
        gm.denom = torch.zeros((gm.P, 1), device=dev)
        prune_ms.append(round(_timed(lambda _i: gm.prune_points(mask), 1), 4))
        del gm
    del raw

    # for information: the step once the half with the lowest weight_max over the V views is gone
    keep = st.weight_max >= st.weight_max.median()
    kc = keep.cpu()
    sub = {k: v[kc] for k, v in scene.items()}
    n_blended = int((st.count > 0).sum())
    del pc, st
    torch.cuda.empty_cache()
    ms_after, _, _, _ = step_times(bench.BenchGaussians(sub, 3, dev))
    mpix = V * H * W / 1e6
    line = {"metric": "contribution statistics and prune_points, cost", "gpu": gpu,
            "config": {"gaussians": a.gaussians, "width": W, "height": H, "views": V, "sh_degree": 3, "steps": a.steps,
                       "rounds": a.rounds},
            "kernel_ms_per_view": kernel_ms, "contribution_launches_per_2_steps": launches,
            "ms_per_step": ms, "mpix_s": {leg: round(mpix / (m / 1e3), 1) for leg, m in best.items()},
            "step_overhead_frac": round(best["contrib"] / best["plain"] - 1.0, 4),
            "prune_points_ms": prune_ms, "prune_points_ms_median_after_first": sorted(prune_ms[1:])[len(prune_ms[1:]) // 2]
            if len(prune_ms) > 1 else None, "prune_points_removed": int(mask.sum()),
            "gaussians_blended_in_8_views": n_blended,
            "after_prune": {"gaussians": int(keep.sum()), "ms_per_step": ms_after["plain"],
                            "mpix_s": round(mpix / (min(ms_after["plain"]) / 1e3), 1)}}
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
