"""Camera gradients on the H100: parity with the float64 oracle, two identities that need no oracle at 1 M gaussians / 1080p
(moving the world and the camera together leaves the image unchanged), finite differences of the CUDA forward against the
CUDA backward, the view batch against single-view calls, and a pose refinement through render()."""
import math

import numpy as np
import pytest
import torch

import gs_test_util as U
from oracle import torch_oracle as TO
from test_camera_grads_on_host import KEYS, _pose_camera, assert_camera_close, oracle_camera_grads

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
LOG_SCALE_MEAN = -4.6       # 1 M gaussians larger than bench.py's (-5.3): many overlap in every pixel of the 1080p view


def _cuda_camera_grads(args, cam, wc, wd, keys=KEYS):
    """render through GaussianRasterizer with leaf camera tensors; returns (camera grads, gaussian grads, radii)."""
    import diff_gaussian_rasterization as dgr
    rs = U.settings_to(cam, DEV)
    cams = {k: getattr(rs, k).clone().requires_grad_(k in keys) for k in KEYS}
    rs = rs._replace(**cams)
    t = {k: (v.detach().to(DEV).clone().requires_grad_(True) if v is not None else None) for k, v in args.items()}
    color, radii, invd = dgr.GaussianRasterizer(rs)(means3D=t["means3D"], means2D=None, shs=t["shs"],
                                                     colors_precomp=t["colors_precomp"], opacities=t["opacities"],
                                                     scales=t["scales"], rotations=t["rotations"], cov3D_precomp=t["cov3D_precomp"])
    loss = (color * wc.to(DEV)).sum()
    if wd is not None:
        loss = loss + (invd * wd.to(DEV)).sum()
    loss.backward()
    return ({k: cams[k].grad.detach().double().cpu() for k in keys}, {k: v.grad for k, v in t.items() if v is not None}, radii, rs)


@pytest.mark.parametrize("deg,mode,aa", [(0, "sh", False), (3, "sh", True), (3, "precomp", False)])
def test_parity_with_float64_oracle(deg, mode, aa):
    scene = TO.make_scene(600, seed=100 + deg, log_scale_mean=-2.6)
    cam = TO.make_camera(96, 64, sh_degree=deg, antialiasing=aa, bg=(0.1, 0.3, 0.6))
    args = U.make_args(scene, mode)
    gen = torch.Generator().manual_seed(2)
    wc, wd = torch.randn(3, 64, 96, generator=gen), torch.randn(1, 64, 96, generator=gen)
    got, _, _, _ = _cuda_camera_grads(args, cam, wc, wd)
    ref = oracle_camera_grads(args, cam, wc, wd)
    assert_camera_close({k: v.reshape(-1).numpy() for k, v in got.items()}, ref, f"deg {deg} {mode} aa {aa}")


def _big_scene(sh_coeffs):
    scene = TO.make_scene(1_000_000, seed=0, sh_coeffs=sh_coeffs, log_scale_mean=LOG_SCALE_MEAN)
    cam = TO.make_camera(1920, 1080, sh_degree=int(round(math.sqrt(sh_coeffs))) - 1, bg=(0.2, 0.3, 0.1))
    yy, xx = torch.meshgrid(torch.arange(1080, dtype=torch.float32), torch.arange(1920, dtype=torch.float32), indexing="ij")
    wc = torch.stack([1.0 + 0.5 * torch.sin(xx / 170 + c) * torch.cos(yy / 130) for c in range(3)])
    wd = (0.5 + 0.25 * torch.cos(xx / 230) * torch.sin(yy / 190))[None]
    return scene, cam, wc, wd


def test_translation_identity_1m_1080p():
    """Moving the world by delta and the camera with it leaves every pixel unchanged, so
    sum_i dL/dmu_i + dL/dcampos - V[:3,:] dL/dV[3,:]^T - PM[:3,:] dL/dPM[3,:]^T = 0.  Bound relative to the sum of the absolute
    values of the terms: float32 summation error over 1 M gaussians."""
    scene, cam, wc, wd = _big_scene(16)
    args = U.make_args(scene, "sh")
    g, gg, radii, rs = _cuda_camera_grads(args, cam, wc, wd)
    assert int((radii > 0).sum()) > 100_000
    dmu = gg["means3D"].double().cpu()
    V, PM = rs.viewmatrix.detach().double().cpu(), rs.projmatrix.detach().double().cpu()
    dV, dPM = g["viewmatrix"], g["projmatrix"]
    terms = [dmu.sum(0), g["campos"], -(V[:3, :] @ dV[3, :]), -(PM[:3, :] @ dPM[3, :])]
    scale = dmu.abs().sum(0) + g["campos"].abs() + V[:3, :].abs() @ dV[3, :].abs() + PM[:3, :].abs() @ dPM[3, :].abs()
    rel = (sum(terms).abs() / scale).max().item()
    print(f"translation identity: residual / sum|terms| = {rel:.3e}; terms {[t.tolist() for t in terms]}")
    assert rel < TRANSLATION_BAR, rel


def _skew(axis):
    K = torch.zeros(3, 3, dtype=torch.float64)
    i, j = [(1, 2), (2, 0), (0, 1)][axis]
    K[i, j], K[j, i] = -1.0, 1.0
    return K


def test_rotation_identity_cov3d_precomp_sh0():
    """Rotating the world by R = exp(eps K) and the camera with it (means, precomputed covariances, campos, V[:3,:] and
    PM[:3,:] all rotated) leaves the image unchanged at SH degree 0.  Exercises the V[:3,:3] and PM[:3,:] terms."""
    scene, cam, wc, wd = _big_scene(1)
    args = U.make_args(scene, "sh")
    args["cov3D_precomp"] = TO.build_covariance(scene["scales"], 1.0, scene["rotations"], normalize=False)
    args["scales"] = args["rotations"] = None
    g, gg, radii, rs = _cuda_camera_grads(args, cam, wc, wd)
    mu = scene["means3D"].double()
    dmu, dS = gg["means3D"].double().cpu(), gg["cov3D_precomp"].double().cpu()
    c6 = args["cov3D_precomp"].double()
    S = torch.stack([c6[:, 0], c6[:, 1], c6[:, 2], c6[:, 1], c6[:, 3], c6[:, 4], c6[:, 2], c6[:, 4], c6[:, 5]], -1).view(-1, 3, 3)
    V, PM = rs.viewmatrix.detach().double().cpu(), rs.projmatrix.detach().double().cpu()
    cp = rs.campos.detach().double().cpu()
    worst = 0.0
    for axis in range(3):
        K = _skew(axis)
        dSig = K @ S - S @ K                                      # K S + S K^T
        dSig6 = torch.stack([dSig[:, 0, 0], dSig[:, 0, 1], dSig[:, 0, 2], dSig[:, 1, 1], dSig[:, 1, 2], dSig[:, 2, 2]], -1)
        t_mu = (dmu * (mu @ K.T)).sum(-1)
        t_S = (dS * dSig6).sum(-1)
        terms = [t_mu.sum(), t_S.sum(), (g["campos"] * (K @ cp)).sum(), (g["viewmatrix"][:3, :] * (K @ V[:3, :])).sum(),
                 (g["projmatrix"][:3, :] * (K @ PM[:3, :])).sum()]
        scale = (t_mu.abs().sum() + t_S.abs().sum() + (g["campos"] * (K @ cp)).abs().sum()
                 + (g["viewmatrix"][:3, :] * (K @ V[:3, :])).abs().sum() + (g["projmatrix"][:3, :] * (K @ PM[:3, :])).abs().sum())
        rel = float(abs(sum(terms)) / scale)
        print(f"rotation identity, axis {axis}: residual / sum|terms| = {rel:.3e}; terms {[float(t) for t in terms]}")
        worst = max(worst, rel)
    assert worst < ROTATION_BAR, worst


# Bounds of the two identities.  Measured on an H100 80GB HBM3 at a 400 W power limit: residual / sum|terms| = 3.4e-9 and 6.8e-9
# (translation, two runs), at most 6.4e-9 (rotation, three axes, two runs) -- float32 summation error.  The bound leaves a factor
# of ~15; a wrong or missing term shows as O(1e-2) or more.
TRANSLATION_BAR = 1e-7
ROTATION_BAR = 1e-7


def test_finite_differences_of_cuda_forward_match_cuda_backward_for_the_camera():
    """Central differences of the CUDA forward (loss accumulated in float64) for every entry of V and PM the forward reads,
    campos and bg, against the CUDA backward.  A camera perturbation moves every gaussian's 1/255 contour, a boundary term the
    analytic gradient ignores (as for the means): the bars are correlation and relative L2 error.  bg enters linearly."""
    import diff_gaussian_rasterization as dgr
    H, W = 96, 144
    scene = TO.make_scene(400, seed=91, log_scale_mean=-2.2)
    scene["opacities"] = scene["opacities"].clamp(0.05, 0.9)
    cam = TO.make_camera(W, H, sh_degree=3, antialiasing=True, bg=(0.2, 0.3, 0.1), scale_modifier=0.9)
    yy, xx = torch.meshgrid(torch.arange(H, dtype=torch.float64), torch.arange(W, dtype=torch.float64), indexing="ij")
    wc = torch.stack([1.0 + 0.5 * torch.sin(xx / 17 + c) * torch.cos(yy / 13) for c in range(3)])
    wd = (0.5 + 0.25 * torch.cos(xx / 23) * torch.sin(yy / 19))[None]
    args = U.make_args(scene, "sh")
    g, _, _, rs = _cuda_camera_grads(args, cam, wc.float(), wd.float())
    ins = {k: (v.to(DEV).float().contiguous() if v is not None else None) for k, v in args.items()}
    wc_d, wd_d = wc.to(DEV), wd.to(DEV)

    def image(k, flat_index, h):
        t = {kk: getattr(rs, kk).detach().contiguous().clone() for kk in KEYS}     # viewmatrix is a transposed view
        t[k].view(-1)[flat_index] += h
        r = dgr.GaussianRasterizer(rs._replace(**t))
        with torch.no_grad():
            color, _, invd = r(means3D=ins["means3D"], means2D=None, shs=ins["shs"], opacities=ins["opacities"], scales=ins["scales"],
                               rotations=ins["rotations"])
        return color.double(), invd.double()

    entries = [("viewmatrix", 4 * r + c, 1e-3) for r in range(4) for c in range(3)]
    entries += [("projmatrix", 4 * r + c, 1e-3) for r in range(4) for c in (0, 1, 3)]
    entries += [("campos", c, 1e-2) for c in range(3)] + [("bg", c, 1e-2) for c in range(3)]
    fd, an, kind = [], [], []
    for k, idx, h in entries:
        cp, dp = image(k, idx, h)
        cm, dm = image(k, idx, -h)
        d = ((cp - cm) * wc_d).sum() + ((dp - dm) * wd_d).sum()
        fd.append(float(d) / (2 * h))
        an.append(float(g[k].reshape(-1)[idx]))
        kind.append(k)
    fd, an, kind = np.array(fd), np.array(an), np.array(kind)
    report = {}
    for name, sel in (("camera", kind != "bg"), ("bg", kind == "bg")):
        rel_l2 = float(np.linalg.norm(fd[sel] - an[sel]) / (np.linalg.norm(an[sel]) + 1e-30))
        report[name] = (rel_l2, float(np.corrcoef(fd[sel], an[sel])[0, 1]))
    print("camera finite differences vs backward (rel L2, correlation):", report)
    print("entries:", [(str(k), round(float(a), 4), round(float(b), 4)) for k, a, b in zip(kind, fd, an)])
    assert report["camera"][0] < 0.12 and report["camera"][1] > 0.99, report
    assert report["bg"][0] < 1e-3, report


def test_view_batch_matches_single_view_calls():
    """gsb_backward_batch_camera with V = 5 (render_views_backward) against per-view render() + autograd."""
    import bench
    from gaussian_renderer import render, render_views_backward
    scene = TO.make_scene(20_000, seed=93, log_scale_mean=-3.4)
    W, H, V = 320, 192, 5
    cams = [bench.BenchCamera(W, H, math.radians(60.0), *bench.view_pose(i, 3.0), DEV) for i in range(V)]
    for cm in cams:
        for t in (cm.world_view_transform, cm.full_proj_transform, cm.camera_center):
            t.requires_grad_(True)
    bg = torch.tensor([0.1, 0.2, 0.3], device=DEV, requires_grad=True)
    gts = [torch.rand(3, H, W, generator=torch.Generator().manual_seed(i)).to(DEV) for i in range(V)]
    loss_fn = lambda img, d, i: (img - gts[i]).abs().mean() + 0.1 * d.mean()

    def take():
        out = torch.cat([t.grad.reshape(-1) for cm in cams for t in (cm.world_view_transform, cm.full_proj_transform,
                                                                       cm.camera_center)] + [bg.grad])
        for cm in cams:
            cm.world_view_transform.grad = cm.full_proj_transform.grad = cm.camera_center.grad = None
        bg.grad = None
        return out.double().cpu().numpy()

    pc = bench.BenchGaussians(scene, 3, DEV)
    for i, cm in enumerate(cams):
        pkg = render(cm, pc, bench.Pipe(), bg)
        loss_fn(pkg["render"], pkg["depth"], i).backward()
    single = take()
    render_views_backward(cams, bench.BenchGaussians(scene, 3, DEV), bench.Pipe(), bg, loss_fn)
    batched = take()
    assert np.abs(batched - single).max() <= 1e-4 * np.abs(single).max()


def test_pose_refinement_through_render():
    """Gaussians fixed, target rendered from the true camera; a learnable se(3) offset optimised with Adam through render()
    reduces the pose error by an order of magnitude.  Measured on an H100 80GB HBM3: 9.6e-2 -> 6.0e-5 in 400 steps."""
    import bench
    from gaussian_renderer import render
    scene = TO.make_scene(50_000, seed=94, log_scale_mean=-3.2)
    W, H, fovx = 256, 192, math.radians(60.0)
    fovy = 2.0 * math.atan(math.tan(fovx / 2) * H / W)
    R0, T0 = bench.view_pose(2, 3.0)
    pc = bench.BenchGaussians(scene, 3, DEV)
    for p in pc.parameters():
        p.requires_grad_(False)
    bg = torch.tensor([0.1, 0.1, 0.1], device=DEV)
    cam = bench.BenchCamera(W, H, fovx, R0, T0, DEV)
    w_true = torch.tensor([0.02, -0.03, 0.015], device=DEV)
    t_true = torch.tensor([0.05, -0.04, 0.06], device=DEV)

    def rendered(w, t):
        cam.world_view_transform, cam.full_proj_transform, cam.camera_center = _pose_camera(R0, T0, w, t, fovx, fovy, W, H)
        return render(cam, pc, bench.Pipe(), bg)["render"]

    with torch.no_grad():
        target = rendered(w_true, t_true)
    w = torch.zeros(3, device=DEV, requires_grad=True)
    t = torch.zeros(3, device=DEV, requires_grad=True)
    err = lambda: float(torch.cat([w - w_true, t - t_true]).norm())
    e0 = err()
    opt = torch.optim.Adam([w, t], lr=1e-2)
    sched = torch.optim.lr_scheduler.CosineAnnealingLR(opt, POSE_STEPS)
    for _ in range(POSE_STEPS):
        opt.zero_grad()
        ((rendered(w, t) - target) ** 2).mean().backward()
        opt.step()
        sched.step()
    e1 = err()
    print(f"pose refinement: error {e0:.4e} -> {e1:.4e} in {POSE_STEPS} steps (ratio {e0 / e1:.1f})")
    assert e1 < e0 / 10, (e0, e1)


POSE_STEPS = 400
