"""Rendered alpha (gsb_alpha, gsb_backward_alpha, gsb_backward_batch_alpha and the Python layer above them) run from the kernel
SOURCES on the CPU (tests/host_emul), against float64 autograd through oracle/torch_oracle.py.

The oracle's differentiable alpha is its colour with unit colours and a black background: sum_k alpha_k T_k * 1 = 1 - final_T
with the same blend rules, so every gradient of an alpha loss is the gradient of that colour channel.  The forward is also
checked against the oracle's own (detached) final transmittance.  Bars: forward FWD_BAR absolute, gradients 1e-4 x the tensor's
max magnitude.  Between host-build calls the bar is 1e-5 x max: the backward blend's float atomics (host threads here) land in a
different order from one call to the next."""
import math

import numpy as np
import pytest
import torch

import gs_test_util as U
from oracle import torch_oracle as TO

FWD_BAR = U.FWD_ABS_TOL  # the project's forward bar against the oracle (float32 products and covariances vs float64)
GRAD_BAR = 1e-4
SAME_BAR = 1e-5
GAUSS_KEYS = ("means3D", "means2D", "shs", "colors_precomp", "opacities", "scales", "rotations", "cov3D_precomp")


def _weights(cam, seed=5):
    gen = torch.Generator().manual_seed(seed)
    H, W = cam.image_height, cam.image_width
    return torch.randn(3, H, W, generator=gen), torch.randn(1, H, W, generator=gen), torch.randn(1, H, W, generator=gen)


def oracle_alpha(d, s):
    """Differentiable float64 alpha [1,H,W] of the float64 inputs `d` (a GAUSS_KEYS dict) under settings `s`."""
    P = d["means3D"].shape[0]
    ones = torch.ones(P, 3, dtype=torch.float64)
    col, _, _ = TO.rasterize(d["means3D"], d["means2D"], None, ones, d["opacities"], d["scales"], d["rotations"],
                             d["cov3D_precomp"], s._replace(bg=torch.zeros(3, dtype=torch.float64)))
    return col[:1]


def oracle(args, cam, wc=None, wd=None, wa=None, cam_keys=()):
    """float64 oracle: (alpha, 1 - final_T, grads of sum(color wc) + sum(invdepth wd) + sum(alpha wa) for the gaussian inputs
    and the camera tensors in cam_keys)."""
    P = args["means3D"].shape[0]
    d = {k: (None if args.get(k) is None else args[k].detach().double().clone().requires_grad_(True)) for k in GAUSS_KEYS}
    d["means2D"] = torch.zeros(P, 3, dtype=torch.float64, requires_grad=True)
    cams = {k: getattr(cam, k).detach().double().clone().requires_grad_(True) for k in cam_keys}
    s = cam._replace(**cams)
    color, _, invd, aux = TO.rasterize(d["means3D"], d["means2D"], d["shs"], d["colors_precomp"], d["opacities"], d["scales"],
                                       d["rotations"], d["cov3D_precomp"], s, return_aux=True)
    alpha = oracle_alpha(d, s)
    loss = torch.zeros((), dtype=torch.float64)
    if wc is not None:
        loss = loss + (color * wc.double()).sum() + (invd * wd.double()).sum()
    if wa is not None:
        loss = loss + (alpha * wa.double()).sum()
    grads = {}
    if loss.requires_grad:
        loss.backward()
        for k, t in list(d.items()) + list(cams.items()):
            if t is not None:
                grads[k] = (t.grad if t.grad is not None else torch.zeros_like(t)).numpy()
    return alpha.detach().numpy(), 1.0 - aux["final_T"].numpy()[None], grads, color.detach().numpy()


def ours(dgr, args, cam, wc=None, wd=None, wa=None, split=False, cam_keys=()):
    """Public path: GaussianRasterizer(..., return_alpha=True) + autograd on the host build."""
    rs = U.settings_to(cam, "cpu")
    cams = {k: getattr(rs, k).detach().clone().requires_grad_(True) for k in cam_keys}
    rs = rs._replace(**cams)
    t = {k: (v.detach().float().clone().requires_grad_(True) if v is not None else None) for k, v in args.items()}
    P = t["means3D"].shape[0]
    m2d = torch.zeros(P, 3, requires_grad=True)
    sh, dc = t["shs"], None
    if split and sh is not None:
        full = t["shs"]
        dc = full[:, :1].detach().clone().requires_grad_(True)
        sh = full[:, 1:].detach().clone().requires_grad_(True)
    color, radii, invd, alpha = dgr.GaussianRasterizer(rs)(
        means3D=t["means3D"], means2D=m2d, opacities=t["opacities"], shs=sh, colors_precomp=t["colors_precomp"],
        scales=t["scales"], rotations=t["rotations"], cov3D_precomp=t["cov3D_precomp"], dc=dc, return_alpha=True)
    loss = torch.zeros(())
    if wc is not None:
        loss = loss + (color * wc).sum() + (invd * wd).sum()
    if wa is not None:
        loss = loss + (alpha * wa).sum()
    grads = {}
    if loss.requires_grad:
        loss.backward()
        for k, v in t.items():
            if v is not None and k != "shs":
                grads[k] = v.grad.numpy() if v.grad is not None else np.zeros(v.shape, np.float32)
        if t["shs"] is not None:
            g = torch.cat([dc.grad, sh.grad], 1) if split else t["shs"].grad
            grads["shs"] = g.numpy() if g is not None else np.zeros(t["shs"].shape, np.float32)
        grads["means2D"] = m2d.grad.numpy()
        for k, v in cams.items():
            grads[k] = v.grad.numpy() if v.grad is not None else np.zeros(v.shape, np.float32)
    return alpha.detach().numpy(), grads, radii, color.detach().numpy()


def assert_grads_close(got, ref, what, bar=GRAD_BAR):
    for k, r in ref.items():
        g = np.asarray(got[k], dtype=np.float64).reshape(r.shape)
        scale = np.abs(r).max()
        err = np.abs(g - r).max()
        assert err <= bar * scale + 1e-12, f"{what}: d{k} err {err:.3e} vs max {scale:.3e}"


# ---- forward -------------------------------------------------------------------------------------------------------------
def _fwd_scenarios():
    out = []
    for deg in range(4):
        out.append((f"sh{deg}", dict(P=220, seed=10 + deg), dict(w=48, h=32, sh_degree=deg), "sh"))
    out.append(("precomp", dict(P=220, seed=20), dict(w=48, h=32), "precomp"))
    out.append(("antialiasing", dict(P=220, seed=21, log_scale_mean=-2.6), dict(w=56, h=40, antialiasing=True), "sh"))
    out.append(("scale_modifier_ragged", dict(P=200, seed=22), dict(w=70, h=41, sh_degree=2, scale_modifier=0.7), "sh"))
    out.append(("smaller_than_a_tile", dict(P=120, seed=23, log_scale_mean=-2.0), dict(w=11, h=7, sh_degree=1), "sh"))
    out.append(("near_plane_through_cloud", dict(P=300, seed=24, extent=2.0, log_scale_mean=-2.2),
                dict(w=48, h=32, eye=(0.1, -0.2, -0.3), sh_degree=1), "sh"))
    return out


@pytest.mark.parametrize("name,scn,camkw,mode", _fwd_scenarios(), ids=[s[0] for s in _fwd_scenarios()])
def test_forward_equals_one_minus_final_T(on_host, name, scn, camkw, mode):
    scn = dict(scn)
    P, seed = scn.pop("P"), scn.pop("seed")
    scn.setdefault("log_scale_mean", -2.4)
    scene = TO.make_scene(P, seed=seed, **scn)
    w, h = camkw.pop("w"), camkw.pop("h")
    cam = TO.make_camera(w, h, bg=(0.1, 0.3, 0.6), **camkw)
    args = U.make_args(scene, mode)
    got, _, _, color = ours(on_host, args, cam)
    a_ref, one_minus_T, _, color_ref = oracle(args, cam)
    assert got.shape == (1, h, w) and got.dtype == np.float32
    assert np.abs(got - one_minus_T).max() <= FWD_BAR, name
    assert np.abs(a_ref - one_minus_T).max() <= 1e-12           # the oracle's two definitions agree
    assert got.max() > 0.5, name                                 # the scene covers pixels
    # color = C_fg + (1 - alpha) bg as computed: the render against a black background differs by exactly that term
    bg = cam.bg.double().numpy()[:, None, None]
    fg = ours(on_host, args, cam._replace(bg=torch.zeros(3)))[3]
    assert np.abs(color - (fg + (1.0 - got) * bg)).max() <= 1e-6, name


def test_forward_opacity_zero_and_one(on_host):
    """Opacity 0: nothing blends, alpha = 0.  Opacity 1 (capped at 0.99 per gaussian): many pixels reach the T < 1e-4 stop,
    so alpha saturates at 1 - 1e-4, not 1."""
    scene = TO.make_scene(400, seed=25, log_scale_mean=-1.2)
    cam = TO.make_camera(48, 32, sh_degree=0)
    for o in (0.0, 1.0):
        scene["opacities"] = torch.full((400, 1), o)
        args = U.make_args(scene, "sh")
        got, _, _, _ = ours(on_host, args, cam)
        _, one_minus_T, _, _ = oracle(args, cam)
        assert np.abs(got - one_minus_T).max() <= FWD_BAR, o
        if o == 0.0:
            assert np.all(got == 0.0)
        else:
            # many pixels end at the stop, which never lets T fall below 1e-4
            assert (got > 1 - 1e-3).mean() > 0.1 and float(got.max()) <= 1 - 1e-4 + 1e-7, float(got.max())


def test_empty_and_fully_culled_scenes(on_host):
    """No visible gaussian: alpha == 0 and every gaussian and camera gradient of an alpha loss is exactly 0."""
    dgr = on_host
    cam = TO.make_camera(48, 32, sh_degree=0)
    _, _, wa = _weights(cam)
    for P in (0, 60):
        scene = TO.make_scene(P, seed=1, sh_coeffs=1)
        scene["means3D"][:, 2] -= 100.0
        got, grads, radii, _ = ours(dgr, U.make_args(scene, "sh"), cam, wa=wa, cam_keys=("viewmatrix", "bg")) if P else \
            ours(dgr, U.make_args(scene, "sh"), cam)
        assert (radii == 0).all() and np.all(got == 0.0), P
        for k, g in grads.items():
            assert np.all(g == 0), (P, k)


# ---- gradients -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("deg,mode,camkw", [(0, "sh", {}), (1, "sh", {}), (2, "sh", dict(scale_modifier=0.7)), (3, "sh", {}),
                                            (3, "precomp", {}), (3, "sh", dict(antialiasing=True)),
                                            (1, "sh", dict(eye=(0.1, -0.2, -0.3)))],
                         ids=["sh0", "sh1", "sh2_scale_modifier", "sh3", "precomp", "antialiasing", "near_plane"])
def test_gradients_match_oracle(on_host, deg, mode, camkw):
    """sum(color wc) + sum(invdepth wd) + sum(alpha wa) (render_bwd_kernel<true, true>) and sum(alpha wa) alone
    (<false, true>, with a zero colour gradient) against float64 autograd."""
    near = "eye" in camkw
    scene = TO.make_scene(300 if near else 220, seed=30 + deg, extent=2.0 if near else 1.0,
                          log_scale_mean=-2.2 if near else -2.4)
    cam = TO.make_camera(70, 41, sh_degree=deg, bg=(0.2, 0.4, 0.6), **camkw)
    args = U.make_args(scene, mode)
    wc, wd, wa = _weights(cam)
    _, g, _, _ = ours(on_host, args, cam, wc, wd, wa)
    _, _, r, _ = oracle(args, cam, wc, wd, wa)
    assert_grads_close(g, r, f"full loss deg {deg} {mode} {camkw}")
    _, g, _, _ = ours(on_host, args, cam, wa=wa)
    _, _, r, _ = oracle(args, cam, wa=wa)
    assert_grads_close(g, r, f"alpha loss deg {deg} {mode} {camkw}")
    if mode == "sh":
        assert np.all(g["shs"] == 0)                         # alpha has no colour: no SH gradient at all
    else:
        assert np.all(g["colors_precomp"] == 0)


def test_split_sh_and_camera_gradients(on_host):
    """Split SH input, and cameras that require grad: the pose gradient of an alpha loss matches the oracle, campos gets none
    from it, and dL/dbg does not change when an alpha term is added to a colour loss."""
    dgr = on_host
    keys = ("viewmatrix", "projmatrix", "campos", "bg")
    for deg, M in ((0, 1), (3, 16)):
        scene = TO.make_scene(200, seed=40 + deg, sh_coeffs=M, log_scale_mean=-2.4)
        cam = TO.make_camera(48, 32, sh_degree=deg, bg=(0.1, 0.3, 0.6))
        args = U.make_args(scene, "sh")
        wc, wd, wa = _weights(cam)
        _, g, _, _ = ours(dgr, args, cam, wc, wd, wa, split=True, cam_keys=keys)
        _, _, r, _ = oracle(args, cam, wc, wd, wa, cam_keys=keys)
        r = {k: v for k, v in r.items() if not (k == "campos" and deg == 0)}
        assert_grads_close(g, r, f"split deg {deg}")
        _, g_a, _, _ = ours(dgr, args, cam, wa=wa, split=True, cam_keys=keys)
        _, _, r_a, _ = oracle(args, cam, wa=wa, cam_keys=keys)
        assert_grads_close({k: g_a[k] for k in ("viewmatrix", "projmatrix")}, {k: r_a[k] for k in ("viewmatrix", "projmatrix")},
                           f"pose from alpha, deg {deg}")
        assert np.all(g_a["campos"] == 0) and np.all(g_a["bg"] == 0)
        _, g_c, _, _ = ours(dgr, args, cam, wc, wd, split=True, cam_keys=keys)
        assert np.abs(g["bg"] - g_c["bg"]).max() <= 1e-6 * np.abs(g_c["bg"]).max()


def _state(dgr, args, cam):
    rs = U.settings_to(cam, "cpu")
    f = {k: (v.detach().float().contiguous() if v is not None else None) for k, v in args.items()}
    f["opacities"] = f["opacities"].reshape(-1).contiguous()
    color, radii, invd, pack = dgr._forward_impl(f["means3D"], f["shs"], None, f["opacities"], f["scales"], f["rotations"], None, rs)
    return rs, f, color, invd, pack


def _plain_grads(P, M):
    return dict(means3D=torch.zeros(P, 3), means2D=torch.zeros(P, 3), opacities=torch.zeros(P), shs=torch.zeros(P, M, 3),
                scales=torch.zeros(P, 3), rotations=torch.zeros(P, 4))


def test_null_alpha_gradient_is_the_existing_call_and_zeros_are_close(on_host):
    """gsb_backward_alpha with dL_dalpha NULL launches what gsb_backward does (same results, same launch count); a zero
    dL_dalpha takes the alpha kernel and lands within the atomics-order bar."""
    dgr = on_host
    scene = TO.make_scene(200, seed=50, log_scale_mean=-2.4)
    cam = TO.make_camera(48, 32, sh_degree=3, bg=(0.1, 0.3, 0.6))
    args = U.make_args(scene, "sh")
    wc, wd, _ = _weights(cam)
    rs, f, color, invd, pack = _state(dgr, args, cam)
    P = f["means3D"].shape[0]
    out = {}
    for name in ("plain", "null", "zeros"):
        g = _plain_grads(P, 16)
        keep = []
        cs = dgr._c_settings(rs, pack["sh_coeffs"], keep)
        ci = dgr._c_inputs(P, f["means3D"], f["shs"], None, f["opacities"], f["scales"], f["rotations"], None)
        gg = dgr._Grads()
        for k, v in g.items():
            setattr(gg, {"shs": "dL_dshs"}.get(k, "dL_d" + k), v.data_ptr())
        arena = dgr._Arena(f["means3D"].device)
        dgr.reset_launch_count()
        if name == "plain":
            rc = dgr._C.gsb_backward(dgr.byref(cs), dgr.byref(ci), dgr.byref(pack["state"]), color.data_ptr(), invd.data_ptr(),
                                     wc.data_ptr(), wd.data_ptr(), dgr.byref(gg), 0, arena.cb, None, None)
        else:
            za = torch.zeros(1, 32, 48)
            rc = dgr._C.gsb_backward_alpha(dgr.byref(cs), dgr.byref(ci), None, dgr.byref(pack["state"]), color.data_ptr(),
                                           invd.data_ptr(), wc.data_ptr(), wd.data_ptr(), za.data_ptr() if name == "zeros" else None,
                                           dgr.byref(gg), None, 0, arena.cb, None, None)
        dgr._check(rc, arena)
        out[name] = (g, dgr.launch_count())
    assert out["null"][1] == out["plain"][1] == out["zeros"][1]
    for name in ("null", "zeros"):
        for k, v in out["plain"][0].items():
            assert float((out[name][0][k] - v).abs().max()) <= SAME_BAR * float(v.abs().max()), (name, k)


# ---- view batch ----------------------------------------------------------------------------------------------------------
def _views(n=250, seed=60, V=5, W=48, H=32):
    import bench
    scene = TO.make_scene(n, seed=seed, log_scale_mean=-2.4)
    cams = [bench.BenchCamera(W, H, math.radians(60.0), *bench.view_pose(i, 3.0), "cpu") for i in range(V)]
    gts = [torch.rand(3, H, W, generator=torch.Generator().manual_seed(i)) for i in range(V)]
    masks = [(torch.rand(1, H, W, generator=torch.Generator().manual_seed(100 + i)) > 0.5).float() for i in range(V)]
    return scene, cams, gts, masks, torch.tensor([0.1, 0.2, 0.3])


def _leaf_grads(pc):
    out = {k: getattr(pc, k).grad.clone() for k in ("_xyz", "_shs", "_opacity", "_scaling", "_rotation")}
    for k in out:
        getattr(pc, k).grad = None
    return out


def _assert_same(a, b, what):
    for k, v in b.items():
        assert float((a[k] - v).abs().max()) <= SAME_BAR * float(v.abs().max()) + 1e-12, (what, k)


def test_view_batch_equals_single_view_calls(on_host):
    """render_views_backward(with_alpha=True) with V = 1 and V = 5, batched (sync, async forward, chunked backward) and view
    by view, in both loss modes: the summed gradients equal those of render(return_alpha=True) + autograd per view; the alphas
    it hands to loss_fn and keeps equal render()'s."""
    import bench
    from gaussian_renderer import AsyncCapacity, render, render_views_backward
    for V in (1, 5):
        scene, cams, gts, masks, bg = _views(V=V)
        loss_fn = lambda img, d, i, alpha: (img - gts[i]).abs().mean() + 0.1 * d.mean() + (alpha - masks[i]).abs().mean()

        def loss_grad(img, d, i, alpha):
            n = img.numel()
            return (((img.clamp(0, 1) - gts[i]).abs().mean() + 0.1 * d.mean() + (alpha - masks[i]).abs().mean()),
                    torch.sign(img.clamp(0, 1) - gts[i]) * ((img >= 0) & (img <= 1)) / n, torch.full_like(d, 0.1 / d.numel()),
                    torch.sign(alpha - masks[i]) / alpha.numel())
        pc = bench.BenchGaussians(scene, 3, "cpu")
        alphas = []
        for i, cm in enumerate(cams):
            pkg = render(cm, pc, bench.Pipe(), bg, return_alpha=True)
            loss_fn(pkg["render"], pkg["depth"], i, pkg["alpha"]).backward()
            alphas.append(pkg["alpha"].detach())
        single = _leaf_grads(pc)
        cap = AsyncCapacity("cpu")
        cap.learn([200000])
        for kw in (dict(), dict(batched=False), dict(capacity=cap), dict(grad_chunks=3, on_grad_chunk=lambda *a: None),
                   dict(loss_returns_grad=True), dict(loss_returns_grad=True, batched=False)):
            pc = bench.BenchGaussians(scene, 3, "cpu")
            fn = loss_grad if kw.get("loss_returns_grad") else loss_fn
            out = render_views_backward(cams, pc, bench.Pipe(), bg, fn, with_alpha=True, keep_images=True, **kw)
            _assert_same(_leaf_grads(pc), single, f"V={V} {sorted(kw)}")
            assert len(out["alphas"]) == V
            for a, b in zip(out["alphas"], alphas):
                assert a.shape == (1, 32, 48) and float((a - b).abs().max()) <= 1e-6


def test_view_batch_alpha_kernel_matches_single_states(on_host):
    """gsb_alpha over a view batch's states (one launch) equals the single-view forward's alpha view by view, and an unused
    alpha gradient in the batch takes the plain backward."""
    import bench
    from gaussian_renderer import render_views_backward
    dgr = on_host
    scene, cams, gts, masks, bg = _views(V=5)
    pc = bench.BenchGaussians(scene, 3, "cpu")
    rss = [dgr.GaussianRasterizationSettings(32, 48, math.tan(cm.FoVx / 2), math.tan(cm.FoVy / 2), bg, 1.0, cm.world_view_transform,
                                             cm.full_proj_transform, 3, cm.camera_center, False, False, False) for cm in cams]
    f = {k: v.detach().float().contiguous() for k, v in dict(m=pc.get_xyz, s=pc.get_features, o=pc.get_opacity.reshape(-1),
                                                               sc=pc.get_scaling, r=pc.get_rotation).items()}
    _, _, _, pack = dgr._forward_batch_impl(f["m"], f["s"], f["o"], f["sc"], f["r"], rss)
    dgr.reset_launch_count()
    batch = dgr._alpha_impl(pack["states"], 32, 48, f["m"].device)
    assert dgr.launch_count() == 1 and batch.shape == (5, 1, 32, 48)
    for v, rs in enumerate(rss):
        _, _, _, p1 = dgr._forward_impl(f["m"], f["s"], None, f["o"], f["sc"], f["r"], None, rs)
        assert torch.equal(batch[v], dgr._alpha_impl(p1["state"], 32, 48, f["m"].device))
    # a loss that ignores alpha: same launches as without with_alpha, apart from the one alpha launch of the forward
    counts = []
    for wa in (False, True):
        pc = bench.BenchGaussians(scene, 3, "cpu")
        fn = (lambda img, d, i, alpha: img.mean()) if wa else (lambda img, d, i: img.mean())
        dgr.reset_launch_count()
        render_views_backward(cams, pc, bench.Pipe(), bg, fn, with_alpha=wa)
        counts.append(dgr.launch_count())
    assert counts[1] == counts[0] + 1


def test_peer_path_carries_the_alpha_gradient(on_host):
    """gsb_backward_batch_alpha with a peer table: two "ranks" played one after the other, each adding the gradients of its
    views (colour + alpha loss) into the owner's rows; the owned rows side by side equal the ordinary batched result."""
    import bench
    from gaussian_renderer import GradientBucket, render_views_backward
    scene, cams, gts, masks, bg = _views(n=300, V=2)
    P, rows, world = 300, 256, 2
    width = {"means3D": 3, "opacities": 1, "scales": 3, "rotations": 4, "shs": 48}
    offset, off = {}, 0
    for k, w in width.items():
        offset[k] = off
        off += rows * world * w
    bufs = [torch.zeros(off), torch.zeros(off)]
    loss = lambda mine: (lambda img, d, i, alpha: (img - gts[mine[i]]).abs().mean() + (alpha - masks[mine[i]]).abs().mean())
    for r in range(world):
        mine = [v for v in range(2) if v % world == r]
        pc = bench.BenchGaussians(scene, 3, "cpu")
        named = {"means3D": pc._xyz, "shs": pc._shs, "opacities": pc._opacity, "scales": pc._scaling, "rotations": pc._rotation}
        for k, p in named.items():
            p.grad = bufs[r][offset[k]:offset[k] + rows * world * width[k]].view(rows * world, width[k])[:P].view_as(p)
        render_views_backward([cams[v] for v in mine], pc, bench.Pipe(), bg, loss(mine), with_alpha=True,
                              peers=(world, r, rows, [b.data_ptr() for b in bufs]))
    pc = bench.BenchGaussians(scene, 3, "cpu")
    GradientBucket(pc.parameters())
    render_views_backward(cams, pc, bench.Pipe(), bg, loss(list(range(2))), with_alpha=True)
    ref = {"means3D": pc._xyz.grad, "shs": pc._shs.grad, "opacities": pc._opacity.grad, "scales": pc._scaling.grad,
           "rotations": pc._rotation.grad}
    for k, w in width.items():
        full = [b[offset[k]:offset[k] + rows * world * w].view(rows * world, w) for b in bufs]
        got = torch.cat((full[0][:rows], full[1][rows:P]))
        want = ref[k].reshape(P, w)
        assert float((got - want).abs().max()) <= SAME_BAR * float(want.abs().max()) + 1e-12, k


# ---- Python layer --------------------------------------------------------------------------------------------------------
def test_python_layer_defaults_and_no_grad(on_host):
    """Without return_alpha: the 3-tuple and the launch count of today.  With it: one more launch and a 4-tuple; an unused
    alpha output leaves the backward the plain one; torch.no_grad() works; render() adds "alpha" only on request and the
    exposure of use_trained_exp does not touch it."""
    import bench
    from gaussian_renderer import render
    dgr = on_host
    scene = TO.make_scene(200, seed=70, log_scale_mean=-2.4)
    cam = TO.make_camera(48, 32, sh_degree=3, bg=(0.1, 0.3, 0.6))
    args = U.make_args(scene, "sh")
    rs = U.settings_to(cam, "cpu")
    kw = dict(means3D=args["means3D"], means2D=torch.zeros(200, 3), opacities=args["opacities"], shs=args["shs"],
              scales=args["scales"], rotations=args["rotations"])
    counts, outs = [], []
    for ra in (None, False, True):
        dgr.reset_launch_count()
        out = dgr.GaussianRasterizer(rs)(**kw) if ra is None else dgr.GaussianRasterizer(rs)(**kw, return_alpha=ra)
        counts.append(dgr.launch_count())
        outs.append(out)
    assert len(outs[0]) == len(outs[1]) == 3 and len(outs[2]) == 4
    assert counts[0] == counts[1] == counts[2] - 1
    assert torch.equal(outs[0][0], outs[2][0]) and torch.equal(outs[0][2], outs[2][2])
    with torch.no_grad():
        color, radii, invd, alpha = dgr.GaussianRasterizer(rs)(**kw, return_alpha=True)
    assert torch.equal(alpha, outs[2][3])
    # unused alpha: the plain backward (same launches as a 3-tuple call's backward)
    launches = []
    for ra in (False, True):
        t = {k: v.detach().clone().requires_grad_(True) for k, v in kw.items()}
        out = dgr.GaussianRasterizer(rs)(**t, return_alpha=ra)
        dgr.reset_launch_count()
        out[0].sum().backward()
        launches.append(dgr.launch_count())
    assert launches[0] == launches[1]

    class Exposed(bench.BenchGaussians):
        def get_exposure_from_name(self, name):
            return torch.eye(3, 4) * 0.5

    pc = Exposed(scene, 3, "cpu")
    bcam = bench.BenchCamera(48, 32, math.radians(60.0), *bench.view_pose(0, 3.0), "cpu")
    bcam.image_name = "x"
    plain = render(bcam, pc, bench.Pipe(), torch.tensor([0.1, 0.2, 0.3]))
    assert "alpha" not in plain
    a = render(bcam, pc, bench.Pipe(), torch.tensor([0.1, 0.2, 0.3]), return_alpha=True)
    e = render(bcam, pc, bench.Pipe(), torch.tensor([0.1, 0.2, 0.3]), return_alpha=True, use_trained_exp=True)
    assert a["alpha"].shape == (1, 32, 48) and torch.equal(a["alpha"], e["alpha"])
    assert not torch.equal(a["render"], e["render"])


def test_render_fit_drives_alpha_to_a_mask(on_host):
    """A few Adam steps on opacity through render(return_alpha=True) against a mask lower the alpha loss."""
    import bench
    from gaussian_renderer import render
    scene = TO.make_scene(200, seed=71, log_scale_mean=-2.4)
    pc = bench.BenchGaussians(scene, 3, "cpu")
    cam = bench.BenchCamera(48, 32, math.radians(60.0), *bench.view_pose(0, 3.0), "cpu")
    mask = torch.zeros(1, 32, 48)
    mask[:, 8:24, 12:36] = 1.0
    opt = torch.optim.Adam([pc._opacity, pc._xyz], lr=0.05)
    losses = []
    for _ in range(12):
        opt.zero_grad()
        loss = (render(cam, pc, bench.Pipe(), torch.zeros(3), return_alpha=True)["alpha"] - mask).abs().mean()
        loss.backward()
        opt.step()
        losses.append(float(loss.detach()))
    assert losses[-1] < 0.8 * losses[0], losses


def test_argument_errors(on_host):
    """gsb_alpha: bad V, NULL output, a state of another image size; misaligned dL_dalpha at both backward entry points;
    badly shaped alpha gradients returned by a loss_fn."""
    import bench
    from gaussian_renderer import render_views_backward
    dgr = on_host
    scene = TO.make_scene(120, seed=72, log_scale_mean=-2.4)
    cam = TO.make_camera(48, 32, sh_degree=3)
    args = U.make_args(scene, "sh")
    rs, f, color, invd, pack = _state(dgr, args, cam)
    out = torch.zeros(64 * 64)
    st = (dgr._State * 17)()
    for V, H, W, ptr, msg in ((0, 32, 48, out.data_ptr(), "V=0"), (17, 32, 48, out.data_ptr(), "V=17"),
                              (1, 32, 48, None, "NULL"), (1, 64, 64, out.data_ptr(), "no forward image")):
        st[0] = pack["state"]
        assert dgr._C.gsb_alpha(V, st, H, W, ptr, None) != 0
        assert msg in dgr._C.gsb_last_error().decode()
    with pytest.raises(RuntimeError, match="no forward image"):
        dgr._alpha_impl(pack["state"], 64, 64, f["means3D"].device)
    keep = []
    cs = dgr._c_settings(rs, pack["sh_coeffs"], keep)
    P = f["means3D"].shape[0]
    ci = dgr._c_inputs(P, f["means3D"], f["shs"], None, f["opacities"], f["scales"], f["rotations"], None)
    gg = dgr._Grads()
    buf = torch.zeros(32 * 48 + 1)
    arena = dgr._Arena(f["means3D"].device)
    rc = dgr._C.gsb_backward_alpha(dgr.byref(cs), dgr.byref(ci), None, dgr.byref(pack["state"]), color.data_ptr(), invd.data_ptr(),
                                   torch.zeros_like(color).data_ptr(), None, buf.data_ptr() + 2, dgr.byref(gg), None, 0, arena.cb,
                                   None, None)
    assert rc != 0 and "4-byte aligned" in dgr._C.gsb_last_error().decode()
    sts = (dgr._State * 1)(pack["state"])
    rc = dgr._C.gsb_backward_batch_alpha(1, dgr.byref(cs), dgr.byref(ci), sts, color.data_ptr(), invd.data_ptr(),
                                         torch.zeros_like(color).data_ptr(), None, buf.data_ptr() + 2, dgr.byref(gg), None, None,
                                         0, 1, dgr._CHUNK_FN(), None, arena.cb, None, None)
    assert rc != 0 and "4-byte aligned" in dgr._C.gsb_last_error().decode()
    rc = dgr._C.gsb_backward_batch_alpha(1, dgr.byref(cs), dgr.byref(ci), sts, color.data_ptr(), invd.data_ptr(),
                                         torch.zeros_like(color).data_ptr(), None, None, dgr.byref(gg), None, None,
                                         0, 65, dgr._CHUNK_FN(), None, arena.cb, None, None)
    assert rc != 0 and "n_chunks" in dgr._C.gsb_last_error().decode()
    scene5, cams, gts, masks, bg = _views(n=120, V=2)
    bad = lambda img, d, i, alpha: (img.mean(), torch.zeros_like(img), None, torch.zeros(5))
    with pytest.raises(RuntimeError):
        render_views_backward(cams, bench.BenchGaussians(scene5, 3, "cpu"), bench.Pipe(), bg, bad, with_alpha=True,
                              loss_returns_grad=True)
