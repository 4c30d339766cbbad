"""Deterministic backward on the H100 at bench.py's size (1 M gaussians, 1080p, SH degree 3, 8 views): under
torch.use_deterministic_algorithms(True) repeated backward calls, tile order on and off and sync and async forwards give the
same bits; the values stay within the batch/chunk comparisons' bar of the default backward; and a training loop on the flat
store (view-batch step, fused L1, fused Adam, one densify_and_prune) repeats itself bit for bit, as does the drop-in
render() + loss.backward() path."""
import math
import os
from types import SimpleNamespace

import pytest
import torch

pytestmark = pytest.mark.gpu
# torch's own requirement for deterministic cuBLAS calls under the flag (the camera-gradient chain multiplies matrices)
os.environ.setdefault("CUBLAS_WORKSPACE_CONFIG", ":4096:8")

V, H, W, N = 8, 1080, 1920, 1_000_000
CLOSE = 1e-5
LEAVES = ("_xyz", "_shs", "_opacity", "_scaling", "_rotation")
CAM_KEYS = ("world_view_transform", "full_proj_transform", "camera_center")


@pytest.fixture()
def torch_flag():
    was, warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    yield
    torch.use_deterministic_algorithms(was, warn_only=warn)


@pytest.fixture(scope="module")
def workload():
    import bench
    from gaussian_renderer.synthetic import make_scene
    dev = torch.device("cuda:0")
    scene = make_scene(N, seed=0, log_scale_mean=bench.LOG_SCALE_MEAN)
    cams = [bench.BenchCamera(W, H, math.radians(60.0), *bench.view_pose(i, 3.0), dev) for i in range(V)]
    gen = torch.Generator().manual_seed(7)
    w = dict(c=torch.randn(3, H, W, generator=gen).to(dev), d=torch.randn(1, H, W, generator=gen).to(dev),
             a=torch.randn(1, H, W, generator=gen).to(dev))
    return scene, cams, torch.tensor([0.1, 0.2, 0.3], device=dev), w


def _step(workload, cam_grads=True, **kw):
    """view-batch step with colour + inverse-depth + alpha losses and (cam_grads) camera gradients: every gradient, means2D sums
    included"""
    import bench
    from gaussian_renderer import render_views_backward
    scene, cams0, bg, w = workload
    dev = bg.device
    cams = []
    for c in cams0:
        c2 = bench.BenchCamera.__new__(bench.BenchCamera)
        c2.__dict__.update(c.__dict__)
        for k in CAM_KEYS:
            setattr(c2, k, getattr(c, k).detach().clone().requires_grad_(cam_grads))
        cams.append(c2)
    pc = bench.BenchGaussians(scene, 3, dev)
    stats = dict(xyz_gradient_accum=torch.zeros(N, 1, device=dev), denom=torch.zeros(N, 1, device=dev))

    def loss(img, dep, i, alpha=None):
        return (img * w["c"]).mean() + (dep * w["d"]).mean() + (alpha * w["a"]).mean()
    render_views_backward(cams, pc, bench.Pipe(), bg, loss, with_alpha=True, densify_stats=stats, **kw)
    out = {k: getattr(pc, k).grad for k in LEAVES}
    out["means2D"] = stats["xyz_gradient_accum"]
    for i, c in enumerate(cams):
        for k in CAM_KEYS if cam_grads else ():
            out[f"{k}{i}"] = getattr(c, k).grad
    return out


def _assert_equal(a, b, what):
    for k in b:
        assert torch.equal(a[k], b[k]), f"{what}: {k} differs by {float((a[k] - b[k]).abs().max()):.3e}"


def test_repeats_tile_order_and_async(workload, torch_flag):
    import diff_gaussian_rasterization as dgr
    from gaussian_renderer import AsyncCapacity
    torch.use_deterministic_algorithms(True)
    ref = _step(workload)
    torch.use_deterministic_algorithms(False)
    plain = _step(workload)
    torch.use_deterministic_algorithms(True)
    _assert_equal(_step(workload), ref, "repeat after a default call")
    for k, g in plain.items():
        scale = float(g.abs().max())
        assert float((ref[k] - g).abs().max()) <= CLOSE * scale + 1e-30, k
    dgr.set_option("tile_order", 0)
    try:
        _assert_equal(_step(workload), ref, "tile_order 0")
    finally:
        dgr.set_option("tile_order", 1)
    cap = AsyncCapacity(workload[2].device, capacity=6 << 20)     # above every view's count (about 4.4 M instances)
    _assert_equal(_step(workload, capacity=cap), ref, "async batch")
    # the chunked backward has no camera gradient (its per-view sum spans the chunks)
    _assert_equal(_step(workload, cam_grads=False, grad_chunks=4, on_grad_chunk=lambda *a: None), _step(workload, cam_grads=False),
                  "grad_chunks=4")


def _train(seed_scene, steps=20):
    """20 store steps under the flag: view-batch step + fused L1 + optimizer_step, densify_and_prune at step 10."""
    import diff_gaussian_rasterization as dgr
    import bench
    from gaussian_renderer import render_views_backward
    from gaussian_renderer.synthetic import make_scene
    from gaussian_store import GaussianModel
    dev = torch.device("cuda:0")
    torch.manual_seed(0)
    sc = {k: v.to(dev) for k, v in make_scene(N, seed=seed_scene, log_scale_mean=bench.LOG_SCALE_MEAN).items()}
    m = GaussianModel(3)
    m.active_sh_degree = 3
    op = sc["opacities"].clamp(1e-4, 1 - 1e-4)
    m.create_from_tensors(sc["means3D"], sc["shs"][:, :1].contiguous(), sc["shs"][:, 1:].contiguous(), torch.log(sc["scales"]),
                          sc["rotations"], torch.log(op / (1 - op)).reshape(-1, 1), 4.0)
    m.training_setup(SimpleNamespace(position_lr_init=0.00016, position_lr_final=0.0000016, position_lr_delay_mult=0.01,
                                     position_lr_max_steps=30000, feature_lr=0.0025, opacity_lr=0.025, scaling_lr=0.005,
                                     rotation_lr=0.001, percent_dense=0.01))
    cams = [bench.BenchCamera(W, H, math.radians(60.0), *bench.view_pose(i, 3.0), dev) for i in range(V)]
    gen = torch.Generator().manual_seed(3)
    gts = [torch.rand(3, H, W, generator=gen).to(dev) for _ in range(V)]
    bg = torch.zeros(3, device=dev)
    loss_fn = lambda img, dep, vi: dgr.l1_loss_and_grad(img, gts[vi])
    for it in range(1, steps + 1):
        m.update_learning_rate(it)
        render_views_backward(cams, m, bench.Pipe(), bg, loss_fn, loss_returns_grad=True, overwrite=True,
                              densify_stats=dict(xyz_gradient_accum=m.xyz_gradient_accum, denom=m.denom))
        m.optimizer_step()
        if it == steps // 2:
            m.densify_and_prune(0.0002, 0.005, 4.0, None)
    torch.cuda.synchronize()
    return m.P, m.store.clone(), m.exp_avg.clone(), m.exp_avg_sq.clone()


def test_store_training_repeats_bit_for_bit(torch_flag):
    torch.use_deterministic_algorithms(True)
    a = _train(11)
    b = _train(11)
    assert a[0] == b[0]
    for x, y, what in zip(a[1:], b[1:], ("parameters", "exp_avg", "exp_avg_sq")):
        assert torch.equal(x, y), what


def test_dropin_render_backward_repeats(workload, torch_flag):
    """The drop-in path on a reference-shaped model (six nn.Parameters): identical .grad twice under the flag."""
    import torch.nn as nn
    from gaussian_renderer import render
    scene, cams, bg, w = workload
    dev = bg.device
    op = scene["opacities"].clamp(1e-4, 1 - 1e-4)

    class Model:
        active_sh_degree = max_sh_degree = 3

        def __init__(self):
            self._xyz = nn.Parameter(scene["means3D"].to(dev).clone())
            self._features_dc = nn.Parameter(scene["shs"][:, :1].to(dev).clone())
            self._features_rest = nn.Parameter(scene["shs"][:, 1:].to(dev).clone())
            self._scaling = nn.Parameter(torch.log(scene["scales"]).to(dev))
            self._rotation = nn.Parameter(scene["rotations"].to(dev).clone())
            self._opacity = nn.Parameter(torch.log(op / (1 - op)).reshape(-1, 1).to(dev))

        get_xyz = property(lambda s: s._xyz)
        get_features = property(lambda s: torch.cat((s._features_dc, s._features_rest), 1))
        get_features_dc = property(lambda s: s._features_dc)
        get_features_rest = property(lambda s: s._features_rest)
        get_opacity = property(lambda s: torch.sigmoid(s._opacity))
        get_scaling = property(lambda s: torch.exp(s._scaling))
        get_rotation = property(lambda s: torch.nn.functional.normalize(s._rotation))

        def get_covariance(self, scaling_modifier=1.0):
            raise NotImplementedError

    import bench
    torch.use_deterministic_algorithms(True)
    runs = []
    for _ in range(2):
        pc = Model()
        out = render(cams[0], pc, bench.Pipe(), bg)
        loss = (out["render"] * w["c"]).mean() + (out["depth"] * w["d"]).mean()
        loss.backward()
        runs.append({k: getattr(pc, k).grad.clone() for k in ("_xyz", "_features_dc", "_features_rest", "_scaling", "_rotation",
                                                                "_opacity")})
    _assert_equal(runs[1], runs[0], "drop-in render() + backward")
