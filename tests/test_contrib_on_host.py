"""Per-gaussian contribution statistics (gsb_contribution, ContributionStats and the contrib= arguments) and
GaussianModel.prune_points, run from the kernel SOURCES on the CPU (tests/host_emul).

The float64 reference re-evaluates torch_oracle.rasterize's blend, pixel by pixel, from the oracle's own projection
(TO.project) and constants (TO.K), and reduces its accepted pairs (`keep`) and weights (`w`) per gaussian.  Every call checks
that this re-evaluation reproduces the oracle's colour exactly, so the statistics are those of the oracle's blend.  A pair whose
float64 alpha sits within BOUNDARY relative of 1/255, or whose transmittance after it sits within BOUNDARY relative of the 1e-4
stop, may be decided the other way by float32 arithmetic: only the gaussians of such pairs may differ, and they are listed in
the failure message."""
import math

import numpy as np
import pytest
import torch

import gs_test_util as U
from oracle import torch_oracle as TO

BOUNDARY = 1e-6
REL = 1e-5          # weight_sum / weight_max against float64, relative to the largest value of the scene (the forward's 1e-5 bar)
GAUSS_KEYS = ("means3D", "shs", "colors_precomp", "opacities", "scales", "rotations", "cov3D_precomp")


def oracle_contrib(args, cam):
    """(count [P] int64, weight_sum [P] f64, weight_max [P] f64, gaussians with a boundary pair) of the oracle's blend."""
    d = {k: (None if args.get(k) is None else args[k].detach().double()) for k in GAUSS_KEYS}
    P = d["means3D"].shape[0]
    m2d = torch.zeros(P, 3, dtype=torch.float64)
    count = np.zeros(P, np.int64)
    wsum, wmax = np.zeros(P), np.zeros(P)
    boundary = set()
    color_ref, _, _ = TO.rasterize(d["means3D"], m2d, d["shs"], d["colors_precomp"], d["opacities"], d["scales"], d["rotations"],
                                   d["cov3D_precomp"], cam)
    if P == 0:
        return count, wsum, wmax, boundary
    # torch_oracle.rasterize, lines for lines: projection, depth order, per-pixel blend with the same stop rule
    H, W = int(cam.image_height), int(cam.image_width)
    pr = TO.project(d["means3D"], m2d, d["shs"], d["colors_precomp"], d["opacities"], d["scales"], d["rotations"],
                    d["cov3D_precomp"], cam)
    vis_idx = torch.nonzero(pr.visible).reshape(-1)
    idx = vis_idx[torch.argsort(pr.depth[vis_idx], stable=True)]
    xy, conic, opac, rgb, rect = pr.xy[idx], pr.conic[idx], pr.opacity[idx], pr.rgb[idx], pr.rect[idx]
    ys, xs = torch.meshgrid(torch.arange(H), torch.arange(W), indexing="ij")
    px, py = xs.reshape(-1), ys.reshape(-1)
    Tl = TO.K["TILE"]
    tx_, ty_ = (px // Tl)[:, None], (py // Tl)[:, None]
    in_rect = (tx_ >= rect[None, :, 0]) & (tx_ < rect[None, :, 2]) & (ty_ >= rect[None, :, 1]) & (ty_ < rect[None, :, 3])
    dx = xy[None, :, 0] - px[:, None].double()
    dy = xy[None, :, 1] - py[:, None].double()
    power = -0.5 * (conic[None, :, 0] * dx * dx + conic[None, :, 2] * dy * dy) - conic[None, :, 1] * dx * dy
    a_raw = opac[None, :] * torch.exp(torch.clamp_max(power, 0.0))
    alpha = torch.clamp_max(a_raw, TO.K["ALPHA_MAX"])
    valid = in_rect & (power <= 0) & (alpha >= TO.K["ALPHA_MIN"])
    alpha = torch.where(valid, alpha, torch.zeros_like(alpha))
    T_incl = torch.cumprod(1.0 - alpha, dim=1)
    T_excl = torch.cat([torch.ones_like(T_incl[:, :1]), T_incl[:, :-1]], 1)
    keep = valid & (T_incl >= TO.K["T_STOP"])
    w = torch.where(keep, alpha * T_excl, torch.zeros_like(alpha))
    T_fin = torch.where(keep, 1.0 - alpha, torch.ones_like(alpha)).prod(dim=1)
    color = (w @ rgb + T_fin[:, None] * cam.bg.double()[None, :]).reshape(H, W, 3).permute(2, 0, 1)
    assert torch.equal(color, color_ref), "the re-evaluation is not the oracle's blend"
    near = lambda x, edge: (x - edge).abs() <= BOUNDARY * edge
    # pairs the float32 blend may decide the other way: alpha at 1/255, or the stop at 1e-4 among pixels not yet stopped
    stopped_before = torch.cat([torch.zeros_like(keep[:, :1]), (valid & (T_incl < TO.K["T_STOP"])).cummax(dim=1).values[:, :-1]], 1)
    edge = in_rect & (power <= 0) & (near(torch.clamp_max(a_raw, TO.K["ALPHA_MAX"]), TO.K["ALPHA_MIN"]) |
                                     (valid & near(T_incl, TO.K["T_STOP"])))
    # a boundary pair also changes the transmittance of everything behind it in that pixel
    tainted = (edge & ~stopped_before).cummax(dim=1).values & (valid | edge)
    ids = idx.numpy()
    kn, wn = keep.numpy(), w.numpy()
    count[ids] = kn.sum(0)
    wsum[ids] = wn.sum(0)
    wmax[ids] = wn.max(0) if wn.shape[0] else 0.0
    boundary = set(int(ids[j]) for j in np.nonzero(tainted.numpy().any(0))[0])
    return count, wsum, wmax, boundary


def ours(dgr, args, cam, split=False):
    """ContributionStats of one GaussianRasterizer call (under no_grad) on the host build; also returns the outputs."""
    rs = U.settings_to(cam, "cpu")
    t = {k: (v.detach().float().clone() if v is not None else None) for k, v in args.items()}
    P = t["means3D"].shape[0]
    st = dgr.ContributionStats(P, "cpu")
    sh, dc = t["shs"], None
    if split and sh is not None:
        dc, sh = sh[:, :1].contiguous(), sh[:, 1:].contiguous()
    with torch.no_grad():
        out = dgr.GaussianRasterizer(rs)(means3D=t["means3D"], means2D=torch.zeros(P, 3), opacities=t["opacities"], shs=sh,
                                         colors_precomp=t["colors_precomp"], scales=t["scales"], rotations=t["rotations"],
                                         cov3D_precomp=t["cov3D_precomp"], dc=dc, contrib=st)
    return st, out


def assert_matches_oracle(st, ref, what):
    count, wsum, wmax, boundary = ref
    got_c, got_s, got_m = st.count.numpy(), st.weight_sum.double().numpy(), st.weight_max.double().numpy()
    assert st.count.dtype == torch.int64 and st.weight_sum.dtype == torch.float32 and st.weight_max.dtype == torch.float32
    bad = np.nonzero(got_c != count)[0]
    assert set(bad.tolist()) <= boundary, (f"{what}: counts differ away from the alpha / T boundaries for gaussians "
                                           f"{sorted(set(bad.tolist()) - boundary)}; boundary gaussians {sorted(boundary)}")
    ok = np.ones(count.shape[0], bool)
    ok[list(boundary)] = False
    scale_s, scale_m = max(float(np.abs(wsum).max(initial=0.0)), 1e-30), max(float(np.abs(wmax).max(initial=0.0)), 1e-30)
    es = np.abs(got_s - wsum)[ok].max(initial=0.0)
    em = np.abs(got_m - wmax)[ok].max(initial=0.0)
    assert es <= REL * scale_s, f"{what}: weight_sum err {es:.3e} vs max {scale_s:.3e} (boundary gaussians {sorted(boundary)})"
    assert em <= REL * scale_m, f"{what}: weight_max err {em:.3e} vs max {scale_m:.3e} (boundary gaussians {sorted(boundary)})"
    assert np.all(got_m[got_c == 0] == 0.0) and np.all(got_s[got_c == 0] == 0.0), what


# ---- 1. against the oracle ---------------------------------------------------------------------------------------------------
def _scenarios():
    out = []
    for deg in range(4):
        out.append((f"sh{deg}", dict(P=220, seed=10 + deg), dict(w=48, h=32, sh_degree=deg), "sh"))
    out.append(("precomp_colors_and_cov3D", dict(P=220, seed=20), dict(w=48, h=32), "precomp"))
    out.append(("antialiasing", dict(P=220, seed=21, log_scale_mean=-2.6), dict(w=56, h=40, antialiasing=True), "sh"))
    out.append(("ragged", dict(P=200, seed=22), dict(w=70, h=41, sh_degree=2, scale_modifier=0.7), "sh"))
    out.append(("smaller_than_a_tile", dict(P=120, seed=23, log_scale_mean=-2.0), dict(w=11, h=7, sh_degree=1), "sh"))
    out.append(("near_plane_through_cloud", dict(P=300, seed=24, extent=2.0, log_scale_mean=-2.2),
                dict(w=48, h=32, eye=(0.1, -0.2, -0.3), sh_degree=1), "sh"))
    out.append(("many_tile_gaussians", dict(P=60, seed=25, log_scale_mean=-0.8), dict(w=64, h=48, sh_degree=0), "sh"))
    # > 256 gaussians over one tile: several staging rounds per tile, and opacity low enough to get through them
    out.append(("several_staging_rounds", dict(P=900, seed=26, log_scale_mean=-1.6, opacity=0.02), dict(w=24, h=20, sh_degree=0), "sh"))
    return out


@pytest.mark.parametrize("name,scn,camkw,mode", _scenarios(), ids=[s[0] for s in _scenarios()])
def test_statistics_match_oracle(on_host, name, scn, camkw, mode):
    scn = dict(scn)
    P, seed, opacity = scn.pop("P"), scn.pop("seed"), scn.pop("opacity", None)
    scn.setdefault("log_scale_mean", -2.4)
    scene = TO.make_scene(P, seed=seed, **scn)
    if opacity is not None:
        scene["opacities"] = torch.full((P, 1), opacity)
    camkw = dict(camkw)
    w, h = camkw.pop("w"), camkw.pop("h")
    cam = TO.make_camera(w, h, bg=(0.1, 0.3, 0.6), **camkw)
    args = U.make_args(scene, mode)
    st, _ = ours(on_host, args, cam)
    ref = oracle_contrib(args, cam)
    assert_matches_oracle(st, ref, name)
    assert int(st.count.sum()) > 0, name
    if name == "several_staging_rounds":
        assert int((st.count > 0).sum()) > 256, "the scene must put more than one staging round over a tile"


def test_opacity_zero_and_one(on_host):
    """Opacity 0: nothing is counted.  Opacity 1 (alpha capped at 0.99): many pixels reach the T < 1e-4 stop, and the stopper
    is not counted."""
    scene = TO.make_scene(400, seed=25, log_scale_mean=-1.2)
    cam = TO.make_camera(48, 32, sh_degree=0)
    for o in (0.0, 1.0):
        scene["opacities"] = torch.full((400, 1), o)
        args = U.make_args(scene, "sh")
        st, _ = ours(on_host, args, cam)
        assert_matches_oracle(st, oracle_contrib(args, cam), f"opacity {o}")
        if o == 0.0:
            assert int(st.count.sum()) == 0 and torch.all(st.weight_max == 0) and torch.all(st.weight_sum == 0)
        else:
            assert int(st.count.sum()) > 0


def test_empty_culled_and_no_gaussians(on_host):
    """P == 0 (no launch), and a scene behind the camera (a launch, nothing counted)."""
    dgr = on_host
    cam = TO.make_camera(48, 32, sh_degree=0)
    for P in (0, 60):
        scene = TO.make_scene(P, seed=1, sh_coeffs=1)
        scene["means3D"][:, 2] -= 100.0
        st, out = ours(dgr, U.make_args(scene, "sh"), cam)
        assert (out[1] == 0).all() and st.count.shape == (P,)
        assert int(st.count.sum()) == 0 and torch.all(st.weight_max == 0) and torch.all(st.weight_sum == 0)


# ---- 2. exact cross-check with the feature maps ----------------------------------------------------------------------------
@pytest.mark.parametrize("deg,camkw", [(0, dict(w=48, h=32)), (3, dict(w=70, h=41, antialiasing=True)), (1, dict(w=11, h=7))],
                         ids=["sh0", "sh3_ragged_aa", "sub_tile"])
def test_one_hot_features_give_the_statistics_exactly(on_host, deg, camkw):
    """features = eye(P), P <= 128: channel k is w_k(p) bit for bit, so count[k] == (F[k] > 0).sum() and weight_max[k] ==
    F[k].max() exactly, and weight_sum[k] matches F[k].double().sum()."""
    dgr = on_host
    camkw = dict(camkw)
    w, h = camkw.pop("w"), camkw.pop("h")
    scene = TO.make_scene(128, seed=40 + deg, log_scale_mean=-2.2)
    cam = TO.make_camera(w, h, sh_degree=deg, **camkw)
    args = U.make_args(scene, "sh")
    rs = U.settings_to(cam, "cpu")
    st = dgr.ContributionStats(128, "cpu")
    with torch.no_grad():
        out = dgr.GaussianRasterizer(rs)(means3D=args["means3D"], means2D=torch.zeros(128, 3), opacities=args["opacities"],
                                         shs=args["shs"], scales=args["scales"], rotations=args["rotations"],
                                         features=torch.eye(128), contrib=st)
    F = out[-1].reshape(128, -1)
    assert torch.equal(st.count, (F > 0).sum(1))
    assert torch.equal(st.weight_max, F.max(1).values)
    ref = F.double().sum(1)
    assert float((st.weight_sum.double() - ref).abs().max()) <= 1e-6 * float(ref.abs().max()) + 1e-30
    assert int(st.count.sum()) > 0


# ---- 3. batches, modes, launches, errors --------------------------------------------------------------------------------------
def _grads(pc):
    """the leaves' gradients; clears them (BenchGaussians on the CPU shares its leaves with the scene tensors)"""
    out = {}
    for k in ("_xyz", "_shs", "_opacity", "_scaling", "_rotation"):
        out[k] = getattr(pc, k).grad.clone()
        getattr(pc, k).grad = None
    return out


def _views(n=250, seed=60, V=5, W=48, H=32):
    import bench
    scene = TO.make_scene(n, seed=seed, log_scale_mean=-2.4)
    cams = [bench.BenchCamera(W, H, math.radians(60.0), *bench.view_pose(i, 3.0), "cpu") for i in range(V)]
    return scene, cams, torch.tensor([0.1, 0.2, 0.3])


def _flat(pc):
    return {k: v.detach().float().contiguous() for k, v in dict(m=pc.get_xyz, s=pc.get_features, o=pc.get_opacity.reshape(-1),
                                                               sc=pc.get_scaling, r=pc.get_rotation).items()}


def _settings(dgr, cams, bg):
    return [dgr.GaussianRasterizationSettings(int(cm.image_height), int(cm.image_width), math.tan(cm.FoVx / 2),
                                              math.tan(cm.FoVy / 2), bg, 1.0, cm.world_view_transform, cm.full_proj_transform, 3,
                                              cm.camera_center, False, False, False) for cm in cams]


def _single_view_sum(dgr, f, rss, P):
    st = dgr.ContributionStats(P, "cpu")
    parts = []
    for rs in rss:
        _, _, _, p1 = dgr._forward_impl(f["m"], f["s"], None, f["o"], f["sc"], f["r"], None, rs)
        one = dgr.ContributionStats(P, "cpu")
        dgr._contrib_impl(p1["state"], int(rs.image_height), int(rs.image_width), P, one, "cpu")
        parts.append(one)
        st.count += one.count
        st.weight_sum += one.weight_sum
        torch.maximum(st.weight_max, one.weight_max, out=st.weight_max)
    return st, parts


def assert_same_stats(a, b, what):
    assert torch.equal(a.count, b.count), what
    assert torch.equal(a.weight_max, b.weight_max), what
    scale = float(b.weight_sum.abs().max()) + 1e-30
    assert float((a.weight_sum - b.weight_sum).abs().max()) <= 1e-6 * scale, what


def test_view_batch_equals_single_view_calls(on_host):
    """One launch over 5 view-batch states (sync and async forward) equals the sum of 5 single-view calls: count and max
    exactly, the sum within float-atomics order."""
    import bench
    from gaussian_renderer import AsyncCapacity
    dgr = on_host
    scene, cams, bg = _views(V=5)
    pc = bench.BenchGaussians(scene, 3, "cpu")
    f = _flat(pc)
    rss = _settings(dgr, cams, bg)
    single, _ = _single_view_sum(dgr, f, rss, 250)
    assert int(single.count.sum()) > 0
    _, _, _, pack = dgr._forward_batch_impl(f["m"], f["s"], f["o"], f["sc"], f["r"], rss)
    st = dgr.ContributionStats(250, "cpu")
    dgr.reset_launch_count()
    dgr._contrib_impl(pack["states"], 32, 48, 250, st, "cpu")
    assert dgr.launch_count() == 1
    assert_same_stats(st, single, "sync batch")
    cap = AsyncCapacity("cpu", capacity=max(pack["num_rendered"]) + 64)     # exact-size buffers: empty blocks cost here
    _, _, _, pack = dgr._forward_batch_impl(f["m"], f["s"], f["o"], f["sc"], f["r"], rss, async_counts=cap.counts,
                                            capacity=cap.capacity)
    st = dgr.ContributionStats(250, "cpu")
    dgr._contrib_impl(pack["states"], 32, 48, 250, st, "cpu")
    assert_same_stats(st, single, "async batch")
    # accumulation: a second call adds the counts again and leaves the max where it was
    dgr._contrib_impl(pack["states"], 32, 48, 250, st, "cpu")
    assert torch.equal(st.count, 2 * single.count) and torch.equal(st.weight_max, single.weight_max)
    assert st.zero_() is st and int(st.count.abs().sum()) == 0 and float(st.weight_max.abs().sum()) == 0.0


def test_split_sh_state(on_host):
    """The split-SH forward gives the joint forward's statistics (count and max exactly)."""
    scene = TO.make_scene(220, seed=13, log_scale_mean=-2.4)
    cam = TO.make_camera(48, 32, sh_degree=3, bg=(0.1, 0.3, 0.6))
    args = U.make_args(scene, "sh")
    joint, _ = ours(on_host, args, cam)
    split, _ = ours(on_host, args, cam, split=True)
    assert_same_stats(split, joint, "split SH")


def test_render_views_backward_modes(on_host):
    """render_views_backward(contrib=) batched (sync, async), view by view and chunked gives the single-view sum; gradients
    and losses are those of the call without contrib; one extra launch per forward call."""
    import bench
    from gaussian_renderer import AsyncCapacity, render_views_backward
    dgr = on_host
    scene, cams, bg = _views(V=5)
    rss = _settings(dgr, cams, bg)
    f = _flat(bench.BenchGaussians(scene, 3, "cpu"))
    single, _ = _single_view_sum(dgr, f, rss, 250)
    _, _, _, pack = dgr._forward_batch_impl(f["m"], f["s"], f["o"], f["sc"], f["r"], rss)
    cap = AsyncCapacity("cpu", capacity=max(pack["num_rendered"]) + 64)     # exact-size buffers: empty blocks cost here
    loss = lambda img, d, i: img.mean()
    for kw, extra in ((dict(), 1), (dict(batched=False), 5), (dict(capacity=cap), 1),
                      (dict(grad_chunks=3, on_grad_chunk=lambda *a: None), 1)):
        runs = {}
        for with_c in (False, True):
            pc = bench.BenchGaussians(scene, 3, "cpu")
            st = dgr.ContributionStats(250, "cpu") if with_c else None
            dgr.reset_launch_count()
            out = render_views_backward(cams, pc, bench.Pipe(), bg, loss, contrib=st, **kw)
            runs[with_c] = (dgr.launch_count(), out["losses"].clone(), _grads(pc), st)
        assert runs[True][0] == runs[False][0] + extra, kw
        assert torch.equal(runs[True][1], runs[False][1]), kw
        for k, g in runs[False][2].items():
            assert float((runs[True][2][k] - g).abs().max()) <= 1e-5 * float(g.abs().max()) + 1e-30, (kw, k)
        assert_same_stats(runs[True][3], single, str(kw))


def test_render_and_rasterizer_defaults(on_host):
    """render(contrib=) adds one launch and changes nothing; without contrib the launches are those of before; it works under
    torch.no_grad() and with gradients flowing."""
    import bench
    from gaussian_renderer import render
    dgr = on_host
    scene, cams, bg = _views(V=1)
    res, n = {}, {}
    for with_c in (False, True):
        pc = bench.BenchGaussians(scene, 3, "cpu")
        st = dgr.ContributionStats(250, "cpu") if with_c else None
        dgr.reset_launch_count()
        pkg = render(cams[0], pc, bench.Pipe(), bg, contrib=st)
        n[with_c] = dgr.launch_count()
        pkg["render"].sum().backward()
        res[with_c] = (pkg["render"].detach(), _grads(pc), st)
    assert n[True] == n[False] + 1
    assert torch.equal(res[True][0], res[False][0])
    for k, g in res[False][1].items():
        assert float((res[True][1][k] - g).abs().max()) <= 1e-5 * float(g.abs().max()) + 1e-30, k
    single, _ = _single_view_sum(dgr, _flat(bench.BenchGaussians(scene, 3, "cpu")), _settings(dgr, cams, bg), 250)
    assert_same_stats(res[True][2], single, "render")


def test_argument_errors(on_host):
    """gsb_contribution: bad V, NULL outputs, misaligned outputs, a state of another size or P; Python: wrong P, device, dtype."""
    import bench
    from gaussian_renderer import render, render_views_backward
    dgr = on_host
    scene, cams, bg = _views(V=1)
    pc = bench.BenchGaussians(scene, 3, "cpu")
    f = _flat(pc)
    rs = _settings(dgr, cams, bg)[0]
    _, _, _, pack = dgr._forward_impl(f["m"], f["s"], None, f["o"], f["sc"], f["r"], None, rs)
    st = dgr.ContributionStats(250, "cpu")
    states = (dgr._State * 17)()
    states[0] = pack["state"]
    c, s, m = st.count.data_ptr(), st.weight_sum.data_ptr(), st.weight_max.data_ptr()
    for V, H, W, P, ptrs, msg in ((0, 32, 48, 250, (c, s, m), "V=0"), (17, 32, 48, 250, (c, s, m), "V=17"),
                                  (1, 32, 48, 250, (None, s, m), "NULL"), (1, 32, 48, 250, (c, s, None), "NULL"),
                                  (1, 32, 48, 250, (c + 4, s, m), "aligned"), (1, 32, 48, 250, (c, s + 2, m), "aligned"),
                                  (1, 64, 64, 250, (c, s, m), "is not a forward"), (1, 32, 48, 249, (c, s, m), "holds 250")):
        rc = dgr._C.gsb_contribution(V, states, H, W, P, *ptrs, None)
        assert rc != 0 and msg in dgr._C.gsb_last_error().decode(), (msg, dgr._C.gsb_last_error())
    assert dgr._C.gsb_contribution(1, None, 32, 48, 250, c, s, m, None) != 0
    assert int(st.count.abs().sum()) == 0
    bad = [dgr.ContributionStats(249, "cpu"), dgr.ContributionStats(250, "meta"), "not stats"]
    wrong_dtype = dgr.ContributionStats(250, "cpu")
    wrong_dtype.count = wrong_dtype.count.int()
    bad.append(wrong_dtype)
    wrong_dtype = dgr.ContributionStats(250, "cpu")
    wrong_dtype.weight_max = wrong_dtype.weight_max.double()
    bad.append(wrong_dtype)
    for b in bad:
        with pytest.raises(ValueError):
            render(cams[0], pc, bench.Pipe(), bg, contrib=b)
        with pytest.raises(ValueError):
            render_views_backward(cams, pc, bench.Pipe(), bg, lambda img, d, i: img.mean(), contrib=b)


# ---- 5. pruning the unused gaussians leaves the picture alone ----------------------------------------------------------------
def _store(scene, sh_degree=3):
    from gaussian_store import GaussianModel
    P = scene["means3D"].shape[0]
    gm = GaussianModel(sh_degree)
    op = scene["opacities"].clamp(1e-4, 1 - 1e-4)
    gm.create_from_tensors(scene["means3D"], scene["shs"][:, :1], scene["shs"][:, 1:], torch.log(scene["scales"]),
                           scene["rotations"], torch.log(op / (1 - op)))
    assert gm.P == P
    return gm


def check_prune_unused_leaves_picture(dgr, gm, cams, bg, what):
    """Prune every gaussian with count == 0 over `cams`, re-render: bit-equal except pixels where a pruned gaussian was the
    stopper, which had final_T < 0.01 and move by at most final_T (max|colour| + max|bg|)."""
    import bench
    from gaussian_renderer import render
    st = dgr.ContributionStats(gm.P, gm.store.device)
    before = []
    with torch.no_grad():
        for cm in cams:
            pkg = render(cm, gm, bench.Pipe(), bg, contrib=st)
            before.append(pkg["render"].clone())
        # the unclamped colour and final_T of the unpruned forward, per view
        raw = []
        for cm in cams:
            rs = _settings(dgr, [cm], bg)[0]
            f = _flat(gm)
            color, _, _, pack = dgr._forward_impl(f["m"], f["s"], None, f["o"], f["sc"], f["r"], None, rs)
            alpha = dgr._alpha_impl(pack["state"], int(cm.image_height), int(cm.image_width), color.device)
            raw.append((color, 1.0 - alpha))
    mask = st.count == 0
    n_pruned = int(mask.sum())
    assert 0 < n_pruned < gm.P, f"{what}: the scene must have unused gaussians ({n_pruned} of {gm.P})"
    cmax = float(torch.cat([c.reshape(-1) for c, _ in raw]).abs().max())
    gm.prune_points(mask)
    changed = 0
    with torch.no_grad():
        for cm, img0, (c0, T0) in zip(cams, before, raw):
            rs = _settings(dgr, [cm], bg)[0]
            f = _flat(gm)
            c1, _, _, _ = dgr._forward_impl(f["m"], f["s"], None, f["o"], f["sc"], f["r"], None, rs)
            diff = (c1 != c0).any(0)
            changed += int(diff.sum())
            if diff.any():
                T = T0[0][diff]
                assert float(T.max()) < 0.01, f"{what}: a changed pixel had final_T {float(T.max())}"
                bound = T * (cmax + float(bg.abs().max()))
                assert bool(((c1 - c0).abs()[:, diff] <= bound[None, :] * (1 + 1e-6)).all()), what
            img1 = render(cm, gm, bench.Pipe(), bg)["render"]
            assert torch.equal(img1[:, ~diff], img0[:, ~diff]), what
    return n_pruned, changed


def test_pruning_unused_gaussians_keeps_the_picture(on_host):
    import bench
    dgr = on_host
    # dense and mostly opaque (pixels reach the T < 1e-4 stop, so gaussians behind are never blended) plus 60 gaussians too
    # transparent to pass alpha >= 1/255
    scene = TO.make_scene(600, seed=81, log_scale_mean=-2.0)
    scene["opacities"] = torch.rand(600, 1, generator=torch.Generator().manual_seed(5)) * 0.49 + 0.5
    scene["opacities"][::10] = 0.003
    cams = [bench.BenchCamera(48, 32, math.radians(60.0), *bench.view_pose(i, 3.0), "cpu") for i in range(3)]
    gm = _store(scene)
    gm.active_sh_degree = 3
    n_pruned, _ = check_prune_unused_leaves_picture(dgr, gm, cams, torch.tensor([0.1, 0.2, 0.3]), "host")
    assert gm.P == 600 - n_pruned
