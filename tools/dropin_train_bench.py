"""What train.py does per iteration through the drop-in package, with the default optimizer
and with --optimizer_type sparse_adam, on a model shaped like the reference's scene.GaussianModel (six raw nn.Parameters,
activations through autograd; scene/gaussian_model.py:102-130, 178-199).

One camera per iteration: render() -> L1 -> backward() -> optimizer step -> zero_grad(set_to_none=True)  (train.py:111-186).
  arm "adam":   render(separate_sh=False) + torch.optim.Adam                 (what the drop-in runs without the sparse optimizer)
  arm "sparse": render(separate_sh=True)  + SparseGaussianAdam(radii > 0)    (train.py --optimizer_type sparse_adam)
Both arms live in the same process and are timed in alternating blocks after their warm-up.  SparseGaussianAdam saves work in
proportion to the gaussians a view does NOT see, so the mean visible fraction is reported next to the times; the optimizer
kernel's own time and its algorithmic bytes (the visibility mask + 28 B per float of a visible row) are reported too.
Prints one JSON line.

    python tools/dropin_train_bench.py --steps 30 --warmup 3        (1 M gaussians, 1920x1080, SH 3: BASELINE configs[2])
"""
import argparse
import json
import math
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (ROOT, os.path.join(ROOT, "gaussian-splatting_b200")):
    if _p not in sys.path:
        sys.path.insert(0, _p)


class RefShapedModel:
    """scene.GaussianModel's parameters and activations: raw leaves, activated through autograd."""

    def __init__(self, scene, sh_degree, dev):
        leaf = lambda t: torch.nn.Parameter(t.detach().to(dev).contiguous().clone())
        op = scene["opacities"].clamp(1e-6, 1 - 1e-6).reshape(-1, 1)
        self._xyz = leaf(scene["means3D"])
        self._features_dc, self._features_rest = leaf(scene["shs"][:, :1]), leaf(scene["shs"][:, 1:])
        self._opacity, self._scaling = leaf(torch.log(op / (1 - op))), leaf(torch.log(scene["scales"]))
        self._rotation = leaf(scene["rotations"])
        self.active_sh_degree = sh_degree
        self.max_sh_degree = int(round(math.sqrt(scene["shs"].shape[1]))) - 1

    def param_groups(self, spatial_lr_scale=1.0):
        """training_setup's six groups (arguments/__init__.py:77-89 defaults)."""
        return [{"params": [self._xyz], "lr": 0.00016 * spatial_lr_scale, "name": "xyz"},
                {"params": [self._features_dc], "lr": 0.0025, "name": "f_dc"},
                {"params": [self._features_rest], "lr": 0.0025 / 20.0, "name": "f_rest"},
                {"params": [self._opacity], "lr": 0.025, "name": "opacity"},
                {"params": [self._scaling], "lr": 0.005, "name": "scaling"},
                {"params": [self._rotation], "lr": 0.001, "name": "rotation"}]

    get_xyz = property(lambda s: s._xyz)
    get_features = property(lambda s: torch.cat((s._features_dc, s._features_rest), dim=1))
    get_features_dc = property(lambda s: s._features_dc)
    get_features_rest = property(lambda s: s._features_rest)
    get_opacity = property(lambda s: torch.sigmoid(s._opacity))
    get_scaling = property(lambda s: torch.exp(s._scaling))
    get_rotation = property(lambda s: torch.nn.functional.normalize(s._rotation))


def bench_line(a):
    import bench
    import diff_gaussian_rasterization as dgr
    from diff_gaussian_rasterization.sparse_adam import SparseGaussianAdam
    from gaussian_renderer import render
    from gaussian_renderer.synthetic import make_scene

    if not torch.cuda.is_available():
        raise SystemExit("dropin_train_bench.py: no CUDA device; the rasterizer has no CPU path")
    torch.cuda.set_device(0)
    dev = torch.device("cuda", 0)
    torch.manual_seed(0)
    scene = make_scene(a.gaussians, seed=0, log_scale_mean=bench.LOG_SCALE_MEAN)
    H, W, n_cams = a.height, a.width, max(1, a.views)
    cams = [bench.BenchCamera(W, H, math.radians(60.0), *bench.view_pose(i, 3.0), dev) for i in range(n_cams)]
    gen = torch.Generator().manual_seed(1)
    gts = [torch.rand(3, H, W, generator=gen).to(dev) for _ in range(n_cams)]
    pipe, bg = bench.Pipe(), torch.zeros(3, device=dev)
    arms = {}
    for name in ("adam", "sparse"):
        pc = RefShapedModel(scene, a.sh_degree, dev)
        opt = (SparseGaussianAdam if name == "sparse" else torch.optim.Adam)(pc.param_groups(), lr=0.0, eps=1e-15)
        arms[name] = dict(pc=pc, opt=opt, k=0, vis=torch.zeros((), dtype=torch.float64, device=dev), n_vis=0, ms=[])
    del scene
    P = a.gaussians

    def iteration(arm, sparse):
        cam = cams[arm["k"] % n_cams]
        gt = gts[arm["k"] % n_cams]
        arm["k"] += 1
        pkg = render(cam, arm["pc"], pipe, bg, separate_sh=sparse)
        (pkg["render"] - gt).abs().mean().backward()
        if sparse:
            visible = pkg["radii"] > 0
            arm["opt"].step(visible, pkg["radii"].shape[0])
            arm["vis"] += visible.sum()
            arm["n_vis"] += 1
        else:
            arm["opt"].step()
        arm["opt"].zero_grad(set_to_none=True)

    for name, arm in arms.items():
        for _ in range(max(1, a.warmup)):
            iteration(arm, name == "sparse")
    arms["sparse"]["vis"].zero_()
    arms["sparse"]["n_vis"] = 0
    torch.cuda.synchronize()
    block = max(1, min(5, a.steps // 4))
    n_blocks = max(1, math.ceil(a.steps / block))
    for b in range(n_blocks):
        order = ("adam", "sparse") if b % 2 == 0 else ("sparse", "adam")
        for name in order:
            arm = arms[name]
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(block):
                iteration(arm, name == "sparse")
            e1.record()
            e1.synchronize()
            arm["ms"].append(e0.elapsed_time(e1) / block)
    vis_frac = float(arms["sparse"]["vis"]) / max(1, arms["sparse"]["n_vis"]) / P

    # the optimizer kernel alone: CUDA events around each sparse_adam launch, outside the timed blocks
    dgr.kernel_time("", reset=True)
    dgr.set_option("time_kernels", 2)
    try:
        for _ in range(block):
            iteration(arms["sparse"], True)
        torch.cuda.synchronize()
        opt_ms, opt_n = dgr.kernel_time("sparse_adam", reset=True)
    finally:
        dgr.set_option("time_kernels", 0)
        dgr.kernel_time("", reset=True)
    floats_per_row = 11 + 3 * (a.sh_degree + 1) ** 2
    opt_bytes = P + vis_frac * P * floats_per_row * 28
    opt_ms_per = opt_ms / max(1, opt_n)
    summary = lambda ms: {"min": round(min(ms), 3), "median": round(statistics.median(ms), 3), "max": round(max(ms), 3)}
    med_a, med_s = statistics.median(arms["adam"]["ms"]), statistics.median(arms["sparse"]["ms"])
    line = {"metric": "dropin_train ms/iteration @%d gaussians %dx%d SH %d" % (P, W, H, a.sh_degree), "unit": "ms",
            "workload": "dropin_train", "device": torch.cuda.get_device_name(dev),
            "steps_per_arm": n_blocks * block, "block": block, "warmup": a.warmup,
            "adam_separate_sh_false_ms": summary(arms["adam"]["ms"]),
            "sparse_adam_separate_sh_true_ms": summary(arms["sparse"]["ms"]),
            "speedup_median": round(med_a / med_s, 4), "mean_visible_fraction": round(vis_frac, 4),
            "sparse_adam_kernel_ms": round(opt_ms_per, 4), "sparse_adam_kernel_launches": opt_n,
            "sparse_adam_algorithmic_bytes": int(opt_bytes),
            "sparse_adam_effective_GBps": round(opt_bytes / (opt_ms_per * 1e-3) / 1e9, 1) if opt_ms_per > 0 else None}
    print(json.dumps(line))
    return line


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--steps", type=int, default=30, help="timed iterations per arm")
    ap.add_argument("--warmup", type=int, default=3, help="untimed iterations per arm first")
    ap.add_argument("--gaussians", type=int, default=1_000_000)
    ap.add_argument("--width", type=int, default=1920)
    ap.add_argument("--height", type=int, default=1080)
    ap.add_argument("--sh-degree", type=int, default=3)
    ap.add_argument("--views", type=int, default=8, help="cameras the iterations cycle through")
    bench_line(ap.parse_args())


if __name__ == "__main__":
    main()
