"""Cost of the deterministic backward (torch.use_deterministic_algorithms(True)) on bench.py's workload: 1 M gaussians, 1080p,
8 views per step, SH degree 3, fused L1 image loss, view-batch step (render_views_backward).

Reported, with the card's name and power limit read in the same run (one JSON line):
  ms_per_step        -- the view-batch step with the flag off ("plain") and on ("det"), legs alternated, CUDA events around K
                        steps; "det_nofill" is the det leg with torch.utils.deterministic.fill_uninitialized_memory off (under
                        the flag torch fills every torch.empty with NaN, the forward's state buffers included);
  kernel_ms_per_view -- gsb_kernel_time per view: render_bwd (plain) beside render_bwd_det, det_count, det_prepare, det_reduce
                        and the id sort (the det step's sort kernels minus the plain step's);
  max_memory_mb      -- torch.cuda.max_memory_allocated over steps of each leg, scratch caches dropped before each;
  dropin_ms_per_view -- render() + loss.backward() of one view (the drop-in path), flag off and on.

    python tools/deterministic_bench.py                                   # needs an H100
    python tools/deterministic_bench.py --gaussians 20000 --width 320 --height 192 --steps 5
"""
import argparse
import gc
import json
import math
import os
import subprocess
import sys

import torch

os.environ.setdefault("CUBLAS_WORKSPACE_CONFIG", ":4096:8")     # torch's requirement for deterministic cuBLAS under the flag
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (ROOT, os.path.join(ROOT, "gaussian-splatting_b200")):
    if _p not in sys.path:
        sys.path.insert(0, _p)
import bench  # noqa: E402
import diff_gaussian_rasterization as dgr  # noqa: E402
from gaussian_renderer import GradientBucket, render, render_views_backward  # noqa: E402
from gaussian_renderer.synthetic import make_scene  # noqa: E402

LEGS = ("plain", "det", "det_nofill")
DET_KERNELS = ("render_bwd_det", "det_count", "det_prepare", "det_reduce")


def parse(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--gaussians", type=int, default=1_000_000)
    ap.add_argument("--width", type=int, default=1920)
    ap.add_argument("--height", type=int, default=1080)
    ap.add_argument("--views", type=int, default=8)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3, help="alternations of the legs")
    return ap.parse_args(argv)


def _leg(leg):
    torch.use_deterministic_algorithms(leg != "plain")
    torch.utils.deterministic.fill_uninitialized_memory = leg != "det_nofill"


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
        raise SystemExit("deterministic_bench.py needs a CUDA device")
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

    pc = bench.BenchGaussians(scene, 3, dev)
    bucket = GradientBucket(pc.parameters())

    def step(_i=0):
        render_views_backward(cams, pc, pipe, bg, loss, loss_returns_grad=True, overwrite=True)

    # peak memory per leg, from dropped scratch caches
    mem = {}
    for leg in ("plain", "det"):
        _leg(leg)
        dgr.release_scratch()
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        torch.cuda.reset_peak_memory_stats(dev)
        for _ in range(3):
            step()
        torch.cuda.synchronize()
        mem[leg] = round(torch.cuda.max_memory_allocated(dev) / 2**20, 1)

    for leg in LEGS:
        _leg(leg)
        for _ in range(a.warmup):
            step()
    ms = {leg: [] for leg in LEGS}
    for _ in range(a.rounds):
        for leg in LEGS:
            _leg(leg)
            ms[leg].append(round(_timed(step, a.steps), 4))

    # kernel times per view
    def kernels(leg, names):
        _leg(leg)
        step()
        torch.cuda.synchronize()
        dgr.set_option("time_kernels", 2)
        dgr.kernel_time("", reset=True)
        for _ in range(2):
            step()
        torch.cuda.synchronize()
        out = {n: dgr.kernel_time(n)[0] / (2 * V) for n in names}
        dgr.kernel_time("", reset=True)
        dgr.set_option("time_kernels", 0)
        return out
    sorts = ("sort_hist", "sort_scatter")
    kp = kernels("plain", ("render_bwd",) + sorts)
    kd = kernels("det", DET_KERNELS + sorts)
    kms = {"render_bwd": kp["render_bwd"]}
    kms.update({n: kd[n] for n in DET_KERNELS})
    kms["id_sort"] = sum(kd[n] - kp[n] for n in sorts)
    kms = {k: round(v, 4) for k, v in kms.items()}

    # the drop-in path: render() + loss.backward() of one view
    del bucket
    pc = bench.BenchGaussians(scene, 3, dev)

    def dropin(i):
        out = render(cams[i % V], pc, pipe, bg)
        (out["render"] - gts[i % V]).abs().mean().backward()
    dropin_ms = {}
    for leg in ("plain", "det"):
        _leg(leg)
        for i in range(a.warmup):
            dropin(i)
        dropin_ms[leg] = round(_timed(dropin, a.steps), 4)
        for p in pc.parameters():
            p.grad = None
    _leg("plain")

    best = {leg: min(v) for leg, v in ms.items()}
    mpix = V * H * W / 1e6
    line = {"metric": "deterministic backward, cost", "gpu": gpu,
            "config": {"gaussians": a.gaussians, "width": W, "height": H, "views": V, "sh_degree": 3, "steps": a.steps,
                       "rounds": a.rounds},
            "ms_per_step": ms, "mpix_s": {leg: round(mpix / (m / 1e3), 1) for leg, m in best.items()},
            "det_over_plain": round(best["det"] / best["plain"], 4),
            "det_nofill_over_plain": round(best["det_nofill"] / best["plain"], 4),
            "kernel_ms_per_view": kms, "max_memory_mb": mem, "dropin_ms_per_view": dropin_ms}
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
