"""Contribution statistics and prune_points on the GPU at bench.py's size: 1 M gaussians, 1920x1080, SH degree 3."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

W, H, V, N = 1920, 1080, 8, 1_000_000


@pytest.fixture(scope="module")
def setup():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    import bench
    from gaussian_renderer.synthetic import make_scene
    dev = torch.device("cuda", 0)
    scene = make_scene(N, seed=0, log_scale_mean=bench.LOG_SCALE_MEAN)
    cams = [bench.BenchCamera(W, H, math.radians(60.0), *bench.view_pose(i, 3.0), dev) for i in range(V)]
    return scene, cams, dev


def _inputs(pc):
    return {k: v.detach().float().contiguous() for k, v in dict(m=pc.get_xyz, s=pc.get_features, o=pc.get_opacity.reshape(-1),
                                                               sc=pc.get_scaling, r=pc.get_rotation).items()}


def _settings(dgr, cam, bg, sh_degree=3):
    return dgr.GaussianRasterizationSettings(H, W, math.tan(cam.FoVx / 2), math.tan(cam.FoVy / 2), bg, 1.0, cam.world_view_transform,
                                             cam.full_proj_transform, sh_degree, cam.camera_center, False, False, False)


def _same(a, b, what, rel=1e-5):
    assert torch.equal(a.count, b.count), what
    assert torch.equal(a.weight_max, b.weight_max), what
    err = float((a.weight_sum.double() - b.weight_sum.double()).abs().max())
    assert err <= rel * float(b.weight_sum.abs().max()), (what, err)


def test_one_hot_features_give_the_statistics(setup):
    """128 sampled visible gaussians as one-hot feature channels -- the 16 largest, 56 blended ones and 56 of any kind (most
    visible gaussians of this scene are hidden): channel c is w_k(p) bit for bit, so count and max are exact and the sum
    matches within 1e-5 relative."""
    import bench
    import diff_gaussian_rasterization as dgr
    scene, cams, dev = setup
    pc = bench.BenchGaussians(scene, 3, dev)
    f = _inputs(pc)
    bg = torch.zeros(3, device=dev)
    rs = _settings(dgr, cams[0], bg)
    _, radii, _, pack = dgr._forward_impl(f["m"], f["s"], None, f["o"], f["sc"], f["r"], None, rs)
    st = dgr.ContributionStats(N, dev)
    dgr._contrib_impl(pack["state"], H, W, N, st, dev)
    vis = torch.nonzero(radii > 0).reshape(-1)
    largest = vis[torch.argsort(radii[vis], descending=True)[:16]]
    gen = torch.Generator(device="cpu").manual_seed(3)
    pool = vis[~torch.isin(vis, largest)]
    blended = pool[st.count[pool] > 0]
    blended = blended[torch.randperm(blended.numel(), generator=gen)[:56].to(dev)]
    pool = pool[~torch.isin(pool, blended)]
    ids = torch.cat([largest, blended, pool[torch.randperm(pool.numel(), generator=gen)[:56].to(dev)]])
    assert ids.numel() == 128
    feats = torch.zeros(N, 128, device=dev)
    feats[ids, torch.arange(128, device=dev)] = 1.0
    F = dgr._features_impl(pack["state"], H, W, feats, dev).reshape(128, -1)
    assert torch.equal(st.count[ids], (F > 0).sum(1))
    assert torch.equal(st.weight_max[ids], F.max(1).values)
    ref = F.double().sum(1)
    err = (st.weight_sum[ids].double() - ref).abs()
    assert bool((err <= 1e-5 * ref.abs() + 1e-12).all()), float((err / ref.clamp_min(1e-30)).max())
    assert int((st.count[ids] > 0).sum()) >= 56


def test_view_batch_and_async_equal_single_views(setup):
    """One launch over an 8-view batch equals the sum of the 8 single-view calls; the async batch gives the same."""
    import bench
    import diff_gaussian_rasterization as dgr
    from gaussian_renderer import AsyncCapacity
    scene, cams, dev = setup
    pc = bench.BenchGaussians(scene, 3, dev)
    f = _inputs(pc)
    bg = torch.zeros(3, device=dev)
    rss = [_settings(dgr, c, bg) for c in cams]
    single = dgr.ContributionStats(N, dev)
    for rs in rss:
        _, _, _, p1 = dgr._forward_impl(f["m"], f["s"], None, f["o"], f["sc"], f["r"], None, rs)
        one = dgr.ContributionStats(N, dev)
        dgr._contrib_impl(p1["state"], H, W, N, one, dev)
        single.count += one.count
        single.weight_sum += one.weight_sum
        torch.maximum(single.weight_max, one.weight_max, out=single.weight_max)
        del p1
    _, _, _, pack = dgr._forward_batch_impl(f["m"], f["s"], f["o"], f["sc"], f["r"], rss)
    batch = dgr.ContributionStats(N, dev)
    dgr._contrib_impl(pack["states"], H, W, N, batch, dev)
    _same(batch, single, "sync batch")
    cap = AsyncCapacity(dev)
    cap.learn(pack["num_rendered"])
    del pack
    _, _, _, pack = dgr._forward_batch_impl(f["m"], f["s"], f["o"], f["sc"], f["r"], rss, async_counts=cap.counts,
                                            capacity=cap.capacity)
    asy = dgr.ContributionStats(N, dev)
    dgr._contrib_impl(pack["states"], H, W, N, asy, dev)
    assert cap.check()
    _same(asy, single, "async batch")
    assert int((single.count > 0).sum()) > N // 10


def _store(scene, dev, optimizer_type="default"):
    from gaussian_store import GaussianModel
    gm = GaussianModel(3, optimizer_type)
    op = scene["opacities"].clamp(1e-4, 1 - 1e-4)
    gm.create_from_tensors(scene["means3D"].to(dev), scene["shs"][:, :1].to(dev), scene["shs"][:, 1:].to(dev),
                           torch.log(scene["scales"]).to(dev), scene["rotations"].to(dev), torch.log(op / (1 - op)).to(dev))
    gm.active_sh_degree = 3
    return gm


def test_pruning_unused_gaussians_keeps_the_picture(setup):
    """Prune every gaussian no view blended; re-render: bit-equal but for pixels whose stopper was pruned (final_T < 0.01,
    colour moved by at most final_T (max|colour| + max|bg|))."""
    import diff_gaussian_rasterization as dgr
    scene, cams, dev = setup
    gm = _store(scene, dev)
    bg = torch.tensor([0.1, 0.2, 0.3], device=dev)
    rss = [_settings(dgr, c, bg) for c in cams]
    st = dgr.ContributionStats(gm.P, dev)
    before = []
    for rs in rss:
        f = _inputs(gm)
        color, _, _, pack = dgr._forward_impl(f["m"], f["s"], None, f["o"], f["sc"], f["r"], None, rs)
        dgr._contrib_impl(pack["state"], H, W, gm.P, st, dev)
        T = 1.0 - dgr._alpha_impl(pack["state"], H, W, dev)
        before.append((color, T))
        del pack
    mask = st.count == 0
    n_pruned = int(mask.sum())
    assert 0 < n_pruned < gm.P
    cmax = max(float(c.abs().max()) for c, _ in before)
    gm.prune_points(mask)
    assert gm.P == N - n_pruned
    changed = 0
    for rs, (c0, T0) in zip(rss, before):
        f = _inputs(gm)
        c1, _, _, _ = dgr._forward_impl(f["m"], f["s"], None, f["o"], f["sc"], f["r"], None, rs)
        diff = (c1 != c0).any(0)
        changed += int(diff.sum())
        if bool(diff.any()):
            T = T0[0][diff]
            assert float(T.max()) < 0.01, float(T.max())
            bound = T * (cmax + float(bg.abs().max()))
            assert bool(((c1 - c0).abs()[:, diff] <= bound[None, :] * (1 + 1e-6)).all())
    print(f"pruned {n_pruned} of {N} unused gaussians; {changed} of {V * H * W} pixels changed (stopper pruned)")


@pytest.mark.parametrize("optimizer_type", ["default", "sparse_adam"])
def test_prune_points_equals_boolean_gather_and_trains(setup, optimizer_type):
    """prune_points on the GPU is bit-equal to torch boolean-mask gathers of every group and both moments; the densification
    tensors are gathered, the gradient is zero, every group keeps its step count and skips the next step; then 15 training
    steps run with finite values and advance every group's count by one per step."""
    import bench
    from gaussian_renderer import render_views_backward
    from gaussian_store import GROUPS
    scene, cams, dev = setup
    gm = _store(scene, dev, optimizer_type)
    args = type("A", (), dict(percent_dense=0.01, position_lr_init=1.6e-4, position_lr_final=1.6e-6, position_lr_delay_mult=0.01,
                              position_lr_max_steps=30000, feature_lr=2.5e-3, opacity_lr=2.5e-2, scaling_lr=5e-3,
                              rotation_lr=1e-3))()
    gm.training_setup(args)
    gen = torch.Generator(device=dev).manual_seed(11)
    gts = [torch.rand(3, H, W, device=dev, generator=gen) for _ in range(2)]
    bg = torch.zeros(3, device=dev)

    def step(it):
        gm.update_learning_rate(it)
        gm.zero_grad()
        stats = dict(xyz_gradient_accum=gm.xyz_gradient_accum, denom=gm.denom)
        out = render_views_backward(cams[:2], gm, bench.Pipe(), bg, lambda img, d, i: (img - gts[i]).abs().mean(),
                                    densify_stats=stats)
        gm.optimizer_step()
        return out["losses"]

    for it in range(1, 4):
        step(it)
    gm.max_radii2D = torch.rand(gm.P, device=dev, generator=gen) * 30
    steps0 = dict(gm.group_steps)
    mask = torch.rand(gm.P, device=dev, generator=gen) < 0.5
    keep = ~mask
    P = gm.P
    views = lambda buf: gm._group_views(buf)
    ref = [{n: t[keep].clone() for n, t in views(b).items()} for b in (gm.store, gm.exp_avg, gm.exp_avg_sq)]
    dens = [t[keep].clone() for t in (gm.xyz_gradient_accum, gm.denom, gm.max_radii2D)]
    assert gm.prune_points(mask) == P - int(mask.sum()) == gm.P
    for b, r in zip((gm.store, gm.exp_avg, gm.exp_avg_sq), ref):
        for n, t in views(b).items():
            assert torch.equal(t, r[n]), n
    for a, b in zip((gm.xyz_gradient_accum, gm.denom, gm.max_radii2D), dens):
        assert torch.equal(a, b)
    assert int(gm.grad.abs().sum()) == 0 and gm.group_steps == steps0 and gm._skip_next == set(GROUPS)
    store0 = gm.store.clone()
    gm.optimizer_step()                                       # skipped: the parameters were just replaced
    assert torch.equal(gm.store, store0) and gm.group_steps == steps0
    for it in range(4, 19):
        losses = step(it)
        assert bool(torch.isfinite(losses).all())
    assert all(gm.group_steps[n] == steps0[n] + 15 for n in GROUPS)
    assert bool(torch.isfinite(gm.store).all()) and bool(torch.isfinite(gm.exp_avg_sq).all())
