"""Camera gradients (gsb_backward_camera / gsb_backward_batch_camera: dL/d viewmatrix, projmatrix, campos and bg) run from the
kernel SOURCES on the CPU (tests/host_emul), against float64 autograd through oracle/torch_oracle.py, whose rasterize() takes
the four camera tensors as differentiable inputs.  Bar: 1e-4 x the tensor's max magnitude.  Also: the other gradients of the
camera call equal those of gsb_backward, the view batch equals its single-view calls, a learnable pose chained through render()
gets the oracle's pose gradient, and the argument checks."""
import math

import numpy as np
import pytest
import torch

import gs_test_util as U
from oracle import torch_oracle as TO

CAM_BAR = 1e-4
KEYS = ("viewmatrix", "projmatrix", "campos", "bg")


def _weights(cam, seed=5):
    gen = torch.Generator().manual_seed(seed)
    H, W = cam.image_height, cam.image_width
    return torch.randn(3, H, W, generator=gen), torch.randn(1, H, W, generator=gen)


def oracle_camera_grads(args, cam, wc, wd):
    """float64 autograd of sum(color * wc) + sum(invdepth * wd) w.r.t. the camera tensors (and the gaussians' inputs)."""
    d = lambda t: None if t is None else t.detach().double()
    cams = {k: getattr(cam, k).detach().double().clone().requires_grad_(True) for k in KEYS}
    s = cam._replace(**cams)
    color, _, invd = TO.rasterize(d(args["means3D"]), None, d(args["shs"]), d(args["colors_precomp"]), d(args["opacities"]),
                                  d(args["scales"]), d(args["rotations"]), d(args["cov3D_precomp"]), s)
    loss = (color * wc.double()).sum() + (invd * wd.double()).sum()
    loss.backward()
    # SH degree 0 / colors_precomp: the view direction is not used, campos gets no gradient at all
    return {k: (cams[k].grad if cams[k].grad is not None else torch.zeros_like(cams[k])).reshape(-1).numpy() for k in KEYS}


def ours_camera_grads(dgr, args, cam, wc, wd, split=False, accumulate=False, prefill=None):
    """Forward + gsb_backward_camera on the host build; returns (camera grads, per-gaussian grads)."""
    rs = U.settings_to(cam, "cpu")
    f = {k: (v.detach().float().contiguous() if v is not None else None) for k, v in args.items()}
    P = f["means3D"].shape[0]
    opac = f["opacities"].reshape(-1).contiguous()
    sh, dc = f["shs"], None
    if split and sh is not None:
        dc, sh = sh[:, :1].contiguous(), (sh[:, 1:].contiguous() if sh.shape[1] > 1 else None)
    color, radii, invd, pack = dgr._forward_impl(f["means3D"], sh, f["colors_precomp"], opac, f["scales"], f["rotations"],
                                                 f["cov3D_precomp"], rs, dc=dc)
    grads = dict(means3D=torch.zeros(P, 3), means2D=torch.zeros(P, 3), opacities=torch.zeros(P))
    if f["shs"] is not None:
        if split:
            grads["dc"] = torch.zeros(P, 1, 3)
            if sh is not None:
                grads["shs"] = torch.zeros_like(sh)
        else:
            grads["shs"] = torch.zeros_like(sh)
    if f["colors_precomp"] is not None:
        grads["colors_precomp"] = torch.zeros(P, 3)
    if f["cov3D_precomp"] is not None:
        grads["cov3D_precomp"] = torch.zeros(P, 6)
    else:
        grads["scales"], grads["rotations"] = torch.zeros(P, 3), torch.zeros(P, 4)
    cg = {k: (prefill[k].clone() if prefill is not None else torch.full((16 if k in ("viewmatrix", "projmatrix") else 3,), float("nan")))
          for k in KEYS}
    dgr._backward_impl(pack, rs, f["means3D"], sh, f["colors_precomp"], opac, f["scales"], f["rotations"], f["cov3D_precomp"],
                       color, invd, wc.contiguous(), wd.contiguous(), grads, accumulate, dc=dc, cam_grads=cg)
    return {k: v.numpy().copy() for k, v in cg.items()}, grads, (color, radii, invd, pack)


def assert_camera_close(got, ref, what, bar=CAM_BAR):
    for k in KEYS:
        g, r = np.asarray(got[k], dtype=np.float64), np.asarray(ref[k], dtype=np.float64)
        assert not np.isnan(g).any(), f"{what}: {k} not written"
        scale = np.abs(r).max()
        err = np.abs(g - r).max()
        assert err <= bar * scale + 1e-12, f"{what}: d{k} err {err:.3e} vs max {scale:.3e}\n ours {g}\n ref  {r}"
    # columns the forward never reads
    assert np.all(np.asarray(got["viewmatrix"]).reshape(4, 4)[:, 3] == 0), what
    assert np.all(np.asarray(got["projmatrix"]).reshape(4, 4)[:, 2] == 0), what


def check(dgr, scene, cam, mode="sh", split=False, seed=5):
    args = U.make_args(scene, mode)
    wc, wd = _weights(cam, seed)
    got, _, _ = ours_camera_grads(dgr, args, cam, wc, wd, split=split)
    ref = oracle_camera_grads(args, cam, wc, wd)
    assert_camera_close(got, ref, f"mode {mode} split {split}")
    return got, ref


@pytest.mark.parametrize("deg", [0, 1, 2, 3])
def test_parity_sh_degrees(on_host, deg):
    scene = TO.make_scene(220, seed=70 + deg, log_scale_mean=-2.4)
    got, _ = check(on_host, scene, TO.make_camera(48, 32, sh_degree=deg, bg=(0.1, 0.3, 0.6)))
    assert (np.abs(got["campos"]).max() > 0) == (deg > 0)    # degree 0 does not read the view direction


def test_parity_precomputed_colors_and_covariance(on_host):
    """colors_precomp: campos only enters through the SH view direction, so its gradient is exactly 0."""
    scene = TO.make_scene(220, seed=80, log_scale_mean=-2.4)
    got, ref = check(on_host, scene, TO.make_camera(48, 32, sh_degree=3, bg=(0.2, 0.2, 0.2)), mode="precomp")
    assert np.all(got["campos"] == 0) and np.abs(ref["campos"]).max() == 0


def test_parity_antialiasing(on_host):
    scene = TO.make_scene(220, seed=81, log_scale_mean=-2.6)
    check(on_host, scene, TO.make_camera(56, 40, sh_degree=3, antialiasing=True, bg=(1.0, 1.0, 1.0)))


def test_parity_ragged_image_and_scale_modifier(on_host):
    scene = TO.make_scene(200, seed=82, log_scale_mean=-2.4)
    check(on_host, scene, TO.make_camera(70, 41, sh_degree=2, scale_modifier=0.7, bg=(0.3, 0.1, 0.5)))


def test_parity_camera_inside_the_cloud(on_host):
    """Gaussians behind the near plane and far outside the frustum: the near cull and the 1.3x clamp of x/z, y/z fire."""
    scene = TO.make_scene(300, seed=83, extent=2.0, log_scale_mean=-2.2)
    cam = TO.make_camera(48, 32, eye=(0.1, -0.2, -0.3), sh_degree=1, bg=(0.4, 0.4, 0.4))
    p_view = scene["means3D"] @ cam.viewmatrix[:3, :3] + cam.viewmatrix[3, :3]
    z = p_view[:, 2]
    front = z > 0.2
    clamped = front & ((p_view[:, 0] / z).abs() > 1.3 * cam.tanfovx)
    assert int((~front).sum()) > 50 and int(clamped.sum()) > 10
    check(on_host, scene, cam)


def test_parity_split_sh(on_host):
    for deg, M in ((0, 1), (3, 16)):
        scene = TO.make_scene(200, seed=84 + deg, sh_coeffs=M, log_scale_mean=-2.4)
        check(on_host, scene, TO.make_camera(48, 32, sh_degree=deg, bg=(0.1, 0.3, 0.6)), split=True)


def test_accumulate_adds_to_prefilled_buffers(on_host):
    dgr = on_host
    scene = TO.make_scene(200, seed=86, log_scale_mean=-2.4)
    cam = TO.make_camera(48, 32, sh_degree=3, bg=(0.1, 0.3, 0.6))
    args = U.make_args(scene, "sh")
    wc, wd = _weights(cam)
    gen = torch.Generator().manual_seed(9)
    pre = {k: torch.randn(16 if k in ("viewmatrix", "projmatrix") else 3, generator=gen) for k in KEYS}
    got, _, _ = ours_camera_grads(dgr, args, cam, wc, wd, accumulate=True, prefill=pre)
    ref = oracle_camera_grads(args, cam, wc, wd)
    for k in KEYS:
        r = ref[k] + pre[k].numpy()
        assert np.abs(got[k] - r).max() <= CAM_BAR * np.abs(ref[k]).max() + 1e-6, k


def test_empty_and_all_culled_scenes(on_host):
    """No visible gaussian: exact zeros for viewmatrix / projmatrix / campos; bg still receives sum(final_T * dL/dcolor)
    (final_T = 1 everywhere, so the sum of dL/dcolor)."""
    dgr = on_host
    cam = TO.make_camera(48, 32, sh_degree=0, bg=(0.2, 0.4, 0.6))
    wc, wd = _weights(cam)
    for P in (0, 60):
        scene = TO.make_scene(P, seed=1, sh_coeffs=1)
        scene["means3D"][:, 2] -= 100.0
        got, _, (_, radii, _, _) = ours_camera_grads(dgr, U.make_args(scene, "sh"), cam, wc, wd)
        assert (radii == 0).all()
        for k in ("viewmatrix", "projmatrix", "campos"):
            assert np.all(got[k] == 0), (P, k)
        ref_bg = wc.double().sum(dim=(1, 2)).numpy()
        assert np.abs(got["bg"] - ref_bg).max() <= 1e-5 * np.abs(ref_bg).max(), P


def test_other_gradients_equal_plain_backward(on_host):
    """The per-gaussian gradients of gsb_backward_camera are those of gsb_backward on the same forward state.  Bit equality
    does not hold on the host build: the backward blend's float atomics (host threads) land in a different order from one
    call to the next, so the bar is the one the split-SH tests use, 1e-5 x max (two plain calls differ by ~3e-7 x max)."""
    dgr = on_host
    scene = TO.make_scene(200, seed=87, log_scale_mean=-2.4)
    cam = TO.make_camera(48, 32, sh_degree=3, bg=(0.1, 0.3, 0.6))
    args = U.make_args(scene, "sh")
    wc, wd = _weights(cam)
    _, g_cam, (color, radii, invd, pack) = ours_camera_grads(dgr, args, cam, wc, wd)
    rs = U.settings_to(cam, "cpu")
    f = {k: (v.float().contiguous() if v is not None else None) for k, v in args.items()}
    plain = {k: torch.zeros_like(v) for k, v in g_cam.items()}
    dgr._backward_impl(pack, rs, f["means3D"], f["shs"], None, f["opacities"].reshape(-1).contiguous(), f["scales"],
                       f["rotations"], None, color, invd, wc.contiguous(), wd.contiguous(), plain, False)
    for k, v in plain.items():
        assert float((v - g_cam[k]).abs().max()) <= 1e-5 * float(v.abs().max()), k


def test_repeated_calls_are_bit_identical(on_host):
    """The camera sums have a fixed order (warp butterfly, then a fixed tree): same accumulators, same bits.  The accumulator
    rows come from the backward blend (float atomics), so the state is shared by reusing one forward and one gradient."""
    dgr = on_host
    scene = TO.make_scene(200, seed=88, log_scale_mean=-2.4)
    cam = TO.make_camera(48, 32, sh_degree=1, bg=(0.1, 0.3, 0.6))
    args = U.make_args(scene, "precomp")
    wc, wd = torch.zeros(3, 32, 48), torch.zeros(1, 32, 48)
    wc[:, 10:20, 5:40] = 1.0          # a gradient only bg and the camera's terms see in a fixed order of few contributions
    a, _, _ = ours_camera_grads(dgr, args, cam, wc, wd)
    b, _, _ = ours_camera_grads(dgr, args, cam, wc, wd)
    assert np.array_equal(a["bg"], b["bg"])


def test_autograd_returns_camera_gradients_shaped_like_inputs(on_host):
    """GaussianRasterizer: camera tensors that require grad receive gradients shaped and typed like them; a camera that
    does not require grad leaves the call exactly as before (no extra inputs)."""
    dgr = on_host
    scene = TO.make_scene(200, seed=89, log_scale_mean=-2.4)
    cam = TO.make_camera(48, 32, sh_degree=3, bg=(0.1, 0.3, 0.6))
    args = U.make_args(scene, "sh")
    wc, wd = _weights(cam)
    ref = oracle_camera_grads(args, cam, wc, wd)
    V = cam.viewmatrix.clone().requires_grad_(True)
    bg = cam.bg.double().clone().requires_grad_(True)           # float64 input: float64 gradient
    rs = U.settings_to(cam, "cpu")._replace(viewmatrix=V, bg=bg)
    rast = dgr.GaussianRasterizer(rs)
    color, _, invd = rast(means3D=args["means3D"], means2D=torch.zeros(200, 3), shs=args["shs"], opacities=args["opacities"],
                          scales=args["scales"], rotations=args["rotations"])
    ((color * wc).sum() + (invd * wd).sum()).backward()
    assert V.grad.shape == (4, 4) and bg.grad.dtype == torch.float64
    assert np.abs(V.grad.reshape(-1).numpy() - ref["viewmatrix"]).max() <= CAM_BAR * np.abs(ref["viewmatrix"]).max()
    assert np.abs(bg.grad.numpy() - ref["bg"]).max() <= CAM_BAR * np.abs(ref["bg"]).max()
    assert dgr._camera_inputs(U.settings_to(cam, "cpu")) == ()
    with torch.no_grad():
        assert dgr._camera_inputs(rs) == ()


def _pose_camera(R0, T0, w, t, fovx, fovy, W, H):
    """world_view_transform / full_proj_transform / camera_center as torch functions of an se(3) offset (w, t) applied to
    the camera (R0, T0) -- the construction of scene/cameras.py in differentiable form, on the device of w."""
    dt, dev = w.dtype, w.device
    z = torch.zeros((), dtype=dt, device=dev)
    K = torch.stack([torch.stack([z, -w[2], w[1]]), torch.stack([w[2], z, -w[0]]), torch.stack([-w[1], w[0], z])])
    dR = torch.matrix_exp(K)
    Rw2c = dR @ torch.as_tensor(R0, dtype=dt, device=dev).T            # world -> camera rotation
    tc = dR @ torch.as_tensor(T0, dtype=dt, device=dev) + t
    top = torch.cat([Rw2c, tc[:, None]], 1)
    Rt = torch.cat([top, torch.tensor([[0.0, 0.0, 0.0, 1.0]], dtype=dt, device=dev)], 0)
    wvt = Rt.T
    proj = TO.get_projection_matrix(0.01, 100.0, fovx, fovy).to(device=dev, dtype=dt).T
    full = wvt @ proj
    center = -(Rw2c.T @ tc)
    return wvt, full, center


def test_learnable_pose_through_render_matches_oracle(on_host):
    """A camera built in torch from a learnable pose offset, rendered through gaussian_renderer.render(): the pose gradient
    equals the float64 oracle's through the same construction."""
    import bench
    from gaussian_renderer import render
    from test_sparse_adam_split_sh_on_host import RefShaped
    scene = TO.make_scene(220, seed=90, log_scale_mean=-2.4)
    W, H, fovx = 48, 32, math.radians(60.0)
    fovy = 2.0 * math.atan(math.tan(fovx / 2) * H / W)
    R0, T0 = bench.view_pose(1, 3.0)
    wc = torch.randn(3, H, W, generator=torch.Generator().manual_seed(4))
    out = {}
    for dt in (torch.float32, torch.float64):
        w = torch.tensor([0.01, -0.02, 0.015], dtype=dt, requires_grad=True)
        t = torch.tensor([0.02, 0.01, -0.03], dtype=dt, requires_grad=True)
        wvt, full, center = _pose_camera(R0, T0, w, t, fovx, fovy, W, H)
        if dt == torch.float32:
            cam = bench.BenchCamera(W, H, fovx, R0, T0, "cpu")
            cam.world_view_transform, cam.full_proj_transform, cam.camera_center = wvt, full, center
            pc = RefShaped(scene)
            img = render(cam, pc, bench.Pipe(), torch.tensor([0.1, 0.2, 0.3]))["render"]
        else:
            s = TO.OracleSettings(H, W, math.tan(fovx / 2), math.tan(fovy / 2), torch.tensor([0.1, 0.2, 0.3], dtype=dt), 1.0,
                                  wvt, full, 3, center)
            d = {k: v.double() for k, v in scene.items()}
            img = TO.rasterize(d["means3D"], None, d["shs"], None, d["opacities"], d["scales"],
                               d["rotations"] / d["rotations"].norm(dim=1, keepdim=True), None, s)[0].clamp(0, 1)
        (img * wc.to(dt)).sum().backward()
        out[dt] = torch.cat([w.grad, t.grad]).double().numpy()
    ref = out[torch.float64]
    assert np.abs(out[torch.float32] - ref).max() <= 1e-3 * np.abs(ref).max(), (out[torch.float32], ref)


def test_view_batch_equals_single_view_calls(on_host):
    """gsb_backward_batch_camera with V = 1 and V = 5: each view's camera gradient equals its single-view call's, and the
    chained result of render_views_backward equals per-view render() + autograd."""
    import bench
    from gaussian_renderer import render, render_views_backward
    dgr = on_host
    scene = TO.make_scene(250, seed=91, log_scale_mean=-2.4)
    W, H = 48, 32
    for V in (1, 5):
        cams = [bench.BenchCamera(W, H, math.radians(60.0), *bench.view_pose(i, 3.0), "cpu") for i in range(V)]
        for cm in cams:
            cm.world_view_transform = cm.world_view_transform.clone().requires_grad_(True)
            cm.full_proj_transform = cm.full_proj_transform.clone().requires_grad_(True)
            cm.camera_center = cm.camera_center.clone().requires_grad_(True)
        bg = torch.tensor([0.1, 0.2, 0.3], requires_grad=True)
        gts = [torch.rand(3, H, W, generator=torch.Generator().manual_seed(i)) for i in range(V)]
        loss_fn = lambda img, d, i: (img - gts[i]).abs().mean() + 0.1 * d.mean()

        def grads():
            g = [[cm.world_view_transform.grad, cm.full_proj_transform.grad, cm.camera_center.grad] for cm in cams]
            out = torch.cat([x.reshape(-1) for row in g for x in row] + [bg.grad])
            for cm in cams:
                cm.world_view_transform.grad = cm.full_proj_transform.grad = cm.camera_center.grad = None
            bg.grad = None
            return out.numpy()

        pc = bench.BenchGaussians(scene, 3, "cpu")
        for i, cm in enumerate(cams):
            pkg = render(cm, pc, bench.Pipe(), bg)
            loss_fn(pkg["render"], pkg["depth"], i).backward()
        single = grads()
        pc = bench.BenchGaussians(scene, 3, "cpu")
        render_views_backward(cams, pc, bench.Pipe(), bg, loss_fn)
        batched = grads()
        assert np.abs(batched - single).max() <= 1e-5 * np.abs(single).max(), V
        pc = bench.BenchGaussians(scene, 3, "cpu")
        render_views_backward(cams, pc, bench.Pipe(), bg, loss_fn, batched=False)
        assert np.abs(grads() - single).max() <= 1e-5 * np.abs(single).max(), V


def test_argument_errors(on_host):
    """Chunked and peer calls with cameras that require grad raise; so do badly shaped or typed outputs and a misaligned
    pointer at the C ABI."""
    import bench
    from gaussian_renderer import render_views_backward
    dgr = on_host
    scene = TO.make_scene(120, seed=92, log_scale_mean=-2.4)
    cams = [bench.BenchCamera(48, 32, math.radians(60.0), *bench.view_pose(i, 3.0), "cpu") for i in range(2)]
    cams[1].camera_center = cams[1].camera_center.clone().requires_grad_(True)
    bg = torch.tensor([0.1, 0.2, 0.3])
    loss_fn = lambda img, d, i: img.mean()
    for kw in (dict(grad_chunks=2), dict(on_grad_chunk=lambda *a: None), dict(peers=(1, 0, 128, [0]))):
        with pytest.raises(ValueError, match="cameras that require grad"):
            render_views_backward(cams, bench.BenchGaussians(scene, 3, "cpu"), bench.Pipe(), bg, loss_fn, **kw)
    with pytest.raises(ValueError, match="chunked or peer"):
        _batch_with_chunks(dgr, scene)

    cam = TO.make_camera(48, 32, sh_degree=3)
    args = U.make_args(scene, "sh")
    wc, wd = _weights(cam)
    for bad in ({"viewmatrix": torch.zeros(4, 4, dtype=torch.float64)}, {"campos": torch.zeros(4)},
                {"projmatrix": torch.zeros(4, 4).t()}):
        with pytest.raises(ValueError, match="camera gradient"):
            _backward_with(dgr, args, cam, wc, wd, bad)
    buf = torch.zeros(20)
    misaligned = dgr._CameraGrads()
    misaligned.dL_dbg = buf.data_ptr() + 2
    rc, msg = _backward_with(dgr, args, cam, wc, wd, None, raw=misaligned)
    assert rc != 0 and "4-byte aligned" in msg


def _batch_with_chunks(dgr, scene):
    rs = U.settings_to(TO.make_camera(48, 32, sh_degree=3), "cpu")
    f = {k: v.float().contiguous() for k, v in scene.items()}
    opac = f["opacities"].reshape(-1).contiguous()
    color, radii, invd, pack = dgr._forward_batch_impl(f["means3D"], f["shs"], opac, f["scales"], f["rotations"], [rs, rs])
    g = dict(means3D=torch.zeros_like(f["means3D"]))
    dgr._backward_batch_impl(pack, [rs, rs], f["means3D"], f["shs"], opac, f["scales"], f["rotations"], color, invd,
                             torch.zeros_like(color), None, g, False, n_chunks=2, cam_grads={"bg": torch.zeros(2, 3)})


def _backward_with(dgr, args, cam, wc, wd, cam_grads, raw=None):
    rs = U.settings_to(cam, "cpu")
    f = {k: (v.float().contiguous() if v is not None else None) for k, v in args.items()}
    opac = f["opacities"].reshape(-1).contiguous()
    color, radii, invd, pack = dgr._forward_impl(f["means3D"], f["shs"], None, opac, f["scales"], f["rotations"], None, rs)
    g = dict(means3D=torch.zeros_like(f["means3D"]))
    if raw is None:
        return dgr._backward_impl(pack, rs, f["means3D"], f["shs"], None, opac, f["scales"], f["rotations"], None, color, invd,
                                  wc.contiguous(), wd.contiguous(), g, False, cam_grads=cam_grads)
    keep = []
    cs = dgr._c_settings(rs, pack["sh_coeffs"], keep)
    ci = dgr._c_inputs(f["means3D"].shape[0], f["means3D"], f["shs"], None, opac, f["scales"], f["rotations"], None)
    gg = dgr._Grads()
    arena = dgr._Arena(f["means3D"].device)
    rc = dgr._C.gsb_backward_camera(dgr.byref(cs), dgr.byref(ci), None, dgr.byref(pack["state"]), color.data_ptr(), invd.data_ptr(),
                                    wc.contiguous().data_ptr(), None, dgr.byref(gg), dgr.byref(raw), 0, arena.cb, None, None)
    return rc, dgr._C.gsb_last_error().decode()
