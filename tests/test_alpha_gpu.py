"""Rendered alpha on the H100: parity with the float64 oracle, two identities that need no oracle at 1 M gaussians / 1080p,
central differences of the CUDA alpha forward against the CUDA backward, the view batch against single-view calls (and chunked
against plain), and a short fit of alpha to a mask through render(return_alpha=True)."""
import math

import numpy as np
import pytest
import torch

import gs_test_util as U
from oracle import torch_oracle as TO
from test_alpha_on_host import assert_grads_close, oracle

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
LOG_SCALE_MEAN = -4.6       # as the camera-gradient GPU tests: many gaussians overlap in every pixel of the 1080p view
GEOM = ("means3D", "means2D", "opacities", "scales", "rotations")


def _cuda(args, cam, wc=None, wa=None, bg=None):
    """GaussianRasterizer(..., return_alpha=True) on the GPU; loss sum(color wc) + sum(alpha wa); returns
    (color, alpha, grads, radii) with grads on the device."""
    import diff_gaussian_rasterization as dgr
    rs = U.settings_to(cam, DEV)
    if bg is not None:
        rs = rs._replace(bg=torch.as_tensor(bg, dtype=torch.float32, device=DEV))
    t = {k: (v.detach().to(DEV).clone().requires_grad_(True) if v is not None else None) for k, v in args.items()}
    m2d = torch.zeros(t["means3D"].shape[0], 3, device=DEV, requires_grad=True)
    color, radii, _, alpha = dgr.GaussianRasterizer(rs)(
        means3D=t["means3D"], means2D=m2d, shs=t["shs"], colors_precomp=t["colors_precomp"], opacities=t["opacities"],
        scales=t["scales"], rotations=t["rotations"], cov3D_precomp=t["cov3D_precomp"], return_alpha=True)
    grads = None
    if wc is not None or wa is not None:
        loss = torch.zeros((), device=DEV)
        if wc is not None:
            loss = loss + (color * wc.to(DEV)).sum()
        if wa is not None:
            loss = loss + (alpha * wa.to(DEV)).sum()
        loss.backward()
        grads = {k: v.grad for k, v in t.items() if v is not None}
        grads["means2D"] = m2d.grad
    return color.detach(), alpha.detach(), grads, radii


@pytest.mark.parametrize("deg,mode,aa", [(0, "sh", False), (3, "sh", True), (3, "precomp", False)])
def test_parity_with_float64_oracle(deg, mode, aa):
    scene = TO.make_scene(600, seed=110 + deg, log_scale_mean=-2.6)
    cam = TO.make_camera(96, 64, sh_degree=deg, antialiasing=aa, bg=(0.1, 0.3, 0.6))
    args = U.make_args(scene, mode)
    gen = torch.Generator().manual_seed(2)
    wc, wd, wa = torch.randn(3, 64, 96, generator=gen), torch.randn(1, 64, 96, generator=gen), torch.randn(1, 64, 96, generator=gen)
    import diff_gaussian_rasterization as dgr
    rs = U.settings_to(cam, DEV)
    t = {k: (v.detach().to(DEV).clone().requires_grad_(True) if v is not None else None) for k, v in args.items()}
    m2d = torch.zeros(600, 3, device=DEV, requires_grad=True)
    color, _, invd, alpha = dgr.GaussianRasterizer(rs)(
        means3D=t["means3D"], means2D=m2d, shs=t["shs"], colors_precomp=t["colors_precomp"], opacities=t["opacities"],
        scales=t["scales"], rotations=t["rotations"], cov3D_precomp=t["cov3D_precomp"], return_alpha=True)
    ((color * wc.to(DEV)).sum() + (invd * wd.to(DEV)).sum() + (alpha * wa.to(DEV)).sum()).backward()
    a_ref, one_minus_T, ref, _ = oracle(args, cam, wc, wd, wa)
    assert np.abs(alpha.detach().cpu().numpy() - one_minus_T).max() <= U.FWD_ABS_TOL
    got = {k: v.grad.cpu().numpy() for k, v in t.items() if v is not None}
    got["means2D"] = m2d.grad.cpu().numpy()
    assert_grads_close(got, ref, f"deg {deg} {mode} aa {aa}")


def _big():
    scene = TO.make_scene(1_000_000, seed=0, sh_coeffs=16, log_scale_mean=LOG_SCALE_MEAN)
    cam = TO.make_camera(1920, 1080, sh_degree=3, bg=(0.2, 0.3, 0.1))
    yy, xx = torch.meshgrid(torch.arange(1080, dtype=torch.float32), torch.arange(1920, dtype=torch.float32), indexing="ij")
    G = (1.0 + 0.5 * torch.sin(xx / 170) * torch.cos(yy / 130))[None]
    return scene, cam, G


def test_background_identity_1m_1080p():
    """color(bg1) - color(bg0) = (1 - alpha)(bg1 - bg0): the same final_T carries the background and defines alpha."""
    scene, cam, _ = _big()
    args = U.make_args(scene, "sh")
    c0, a0, _, radii = _cuda(args, cam, bg=(0.0, 0.0, 0.0))
    c1, a1, _, _ = _cuda(args, cam, bg=(0.7, 0.4, 1.0))
    assert int((radii > 0).sum()) > 100_000 and torch.equal(a0, a1)
    assert 0.05 < float(a0.mean()) < 0.999
    d = torch.tensor([0.7, 0.4, 1.0], device=DEV)[:, None, None]
    err = float(((c1 - c0) - (1.0 - a0) * d).abs().max())
    print(f"background identity: max |residual| = {err:.3e}")
    assert err <= BG_BAR, err


# Bounds of the two identities.  Measured on an H100 80GB HBM3 at a 700 W power limit: background residual 7.2e-8; unit colours
# |color_c - alpha| <= 7.7e-7 (forward) and gradient rel err <= 3.1e-6 (rotations; 1e-7..7e-7 for the rest).  A wrong or missing
# term shows as O(1e-2) or more.
BG_BAR = 2e-6
UNIT_FWD_BAR = 1e-5


def test_unit_colour_identity_1m_1080p():
    """colors_precomp = 1 and bg = 0: every colour channel is alpha (to float32 rounding of two different sums), and the
    gradients of sum(alpha G) equal those of sum(color_r G) for every geometric input."""
    scene, cam, G = _big()
    P = scene["means3D"].shape[0]
    args = U.make_args(scene, "sh")
    args.update(shs=None, colors_precomp=torch.ones(P, 3))
    cam = cam._replace(bg=torch.zeros(3))
    wr = torch.cat([G, torch.zeros(2, *G.shape[1:])])
    color, alpha, g_col, _ = _cuda(args, cam, wc=wr)
    _, _, g_al, _ = _cuda(args, cam, wa=G)
    ferr = float((color - alpha).abs().max())
    print(f"unit colour identity: forward max |color_c - alpha| = {ferr:.3e}")
    assert ferr <= UNIT_FWD_BAR
    worst = {}
    for k in GEOM:
        r, v = g_col[k].double(), g_al[k].double()
        worst[k] = float((v - r).abs().max() / r.abs().max())
    print("unit colour identity: gradient rel err", worst)
    assert max(worst.values()) <= 1e-4, worst
    assert float(g_al["colors_precomp"].abs().max()) == 0.0


def test_finite_differences_of_cuda_alpha_forward_match_cuda_backward():
    """Central differences of the CUDA alpha forward (float64 accumulation) against the CUDA backward of sum(alpha wa), with the
    acceptance rule of test_round2_gpu's finite-difference test.  The SH coefficients do not enter alpha: exactly zero."""
    import diff_gaussian_rasterization as dgr
    dev = torch.device("cuda", 0)
    H, W = 96, 144
    scene = TO.make_scene(400, seed=91, log_scale_mean=-2.2)
    scene["opacities"] = scene["opacities"].clamp(0.05, 0.9)
    cam = U.settings_to(TO.make_camera(W, H, sh_degree=3, antialiasing=True, bg=(0.2, 0.3, 0.1), scale_modifier=0.9), dev)
    yy, xx = torch.meshgrid(torch.arange(H, dtype=torch.float64), torch.arange(W, dtype=torch.float64), indexing="ij")
    wa = (1.0 + 0.5 * torch.sin(xx / 17) * torch.cos(yy / 13))[None].to(dev)
    base = {k: scene[k].to(dev).clone() for k in ("means3D", "shs", "opacities", "scales", "rotations")}
    rast = dgr.GaussianRasterizer(raster_settings=cam)

    def alpha_of(p):
        return rast(means3D=p["means3D"], means2D=torch.zeros_like(p["means3D"]), shs=p["shs"], opacities=p["opacities"],
                    scales=p["scales"], rotations=p["rotations"], return_alpha=True)[3]

    leaves = {k: v.clone().requires_grad_(True) for k, v in base.items()}
    out = rast(means3D=leaves["means3D"], means2D=torch.zeros_like(leaves["means3D"], requires_grad=True), shs=leaves["shs"],
               opacities=leaves["opacities"], scales=leaves["scales"], rotations=leaves["rotations"], return_alpha=True)
    (out[3] * wa.float()).sum().backward()
    grads = {k: v.grad.detach() for k, v in leaves.items()}
    assert grads["shs"] is not None and float(grads["shs"].abs().max()) == 0.0
    visible = (out[1] > 0).nonzero().reshape(-1)
    assert visible.numel() > 200
    steps = {"means3D": 2e-3, "scales": None, "rotations": 2e-2, "opacities": 1e-2}
    rng = np.random.default_rng(3)
    report = {}
    with torch.no_grad():
        for kind, h in steps.items():
            fd, an = [], []
            for _ in range(48):
                i = int(visible[rng.integers(visible.numel())])
                idx = (i,) + tuple(int(rng.integers(s)) for s in base[kind].shape[1:])
                hh = h if h is not None else 0.03 * float(base[kind][idx])
                plus = {k: v.clone() for k, v in base.items()}
                minus = {k: v.clone() for k, v in base.items()}
                plus[kind][idx] += hh
                minus[kind][idx] -= hh
                d = ((alpha_of(plus).double() - alpha_of(minus).double()) * wa).sum()
                fd.append(float(d) / (2 * hh))
                an.append(float(grads[kind][idx]))
            fd, an = np.array(fd), np.array(an)
            rms = float(np.sqrt((an ** 2).mean()))
            rel_l2 = float(np.linalg.norm(fd - an) / (np.linalg.norm(an) + 1e-30))
            ok = np.abs(fd - an) <= 0.15 * np.abs(an) + 0.05 * rms
            report[kind] = (rel_l2, float(ok.mean()), float(np.corrcoef(fd, an)[0, 1]))
    print("alpha finite differences vs backward (rel L2, fraction within bound, correlation):", report)
    for kind, (rel_l2, frac_ok, corr) in report.items():
        assert rel_l2 < (0.12 if kind in ("means3D", "scales", "rotations") else 0.03) and frac_ok >= 0.85 and corr > 0.995, (kind, report)


def test_view_batch_agrees_with_single_view_and_chunked_with_plain():
    """render_views_backward(with_alpha=True) at 200 k gaussians, 640x360, 6 views: batched (plain, chunked, async) and view by
    view against render(return_alpha=True) + autograd per view, within 1e-4 x max (float atomics order)."""
    import bench
    from gaussian_renderer import AsyncCapacity, render, render_views_backward
    from gaussian_renderer.synthetic import make_scene
    dev = torch.device("cuda", 0)
    V, W, H = 6, 640, 360
    scene = make_scene(200_000, seed=3, log_scale_mean=-4.0)
    cams = [bench.BenchCamera(W, H, math.radians(60.0), *bench.view_pose(i, 3.0), dev) for i in range(V)]
    gen = torch.Generator().manual_seed(5)
    gts = [torch.rand(3, H, W, generator=gen).to(dev) for _ in range(V)]
    masks = [(torch.rand(1, H, W, generator=gen) > 0.5).float().to(dev) for _ in range(V)]
    bg = torch.tensor([0.1, 0.2, 0.3], device=dev)
    loss_fn = lambda img, d, i, alpha: (img - gts[i]).abs().mean() + (alpha - masks[i]).abs().mean()

    def grads(pc):
        return {k: getattr(pc, k).grad.detach().clone() for k in ("_xyz", "_shs", "_opacity", "_scaling", "_rotation")}

    pc = bench.BenchGaussians(scene, 3, dev)
    ref_alpha = []
    for i, cm in enumerate(cams):
        pkg = render(cm, pc, bench.Pipe(), bg, return_alpha=True)
        loss_fn(pkg["render"], pkg["depth"], i, pkg["alpha"]).backward()
        ref_alpha.append(pkg["alpha"].detach())
    single = grads(pc)
    cap = AsyncCapacity(dev)
    cap.learn([4 << 20])
    report = {}
    for name, kw in (("batched", {}), ("view_by_view", dict(batched=False)), ("chunked", dict(grad_chunks=4)),
                     ("async", dict(capacity=cap))):
        pc = bench.BenchGaussians(scene, 3, dev)
        out = render_views_backward(cams, pc, bench.Pipe(), bg, loss_fn, with_alpha=True, keep_images=True, **kw)
        g = grads(pc)
        report[name] = max(float((g[k] - v).abs().max() / v.abs().max()) for k, v in single.items())
        assert all(torch.equal(a, b) for a, b in zip(out["alphas"], ref_alpha)), name
    if cap.capacity:
        assert cap.check()
    print("view batch vs single view, worst gradient rel err:", report)
    assert max(report.values()) <= 1e-4, report


def test_fit_alpha_to_a_mask_through_render():
    """40 Adam steps on the gaussians' positions and opacities through render(return_alpha=True) against a disc mask: the
    L1 alpha loss falls to less than half its start."""
    import bench
    from gaussian_renderer import render
    from gaussian_renderer.synthetic import make_scene
    dev = torch.device("cuda", 0)
    W, H = 320, 192
    pc = bench.BenchGaussians(make_scene(20_000, seed=4, log_scale_mean=-3.5), 3, dev)
    cam = bench.BenchCamera(W, H, math.radians(60.0), *bench.view_pose(0, 3.0), dev)
    yy, xx = torch.meshgrid(torch.arange(H, device=dev), torch.arange(W, device=dev), indexing="ij")
    mask = (((xx - W / 2) ** 2 + (yy - H / 2) ** 2) < (H / 3) ** 2).float()[None]
    opt = torch.optim.Adam([pc._xyz, pc._opacity], lr=0.01)
    losses = []
    for _ in range(40):
        opt.zero_grad()
        loss = (render(cam, pc, bench.Pipe(), torch.zeros(3, device=dev), return_alpha=True)["alpha"] - mask).abs().mean()
        loss.backward()
        opt.step()
        with torch.no_grad():
            pc._opacity.clamp_(0.0, 1.0)
        losses.append(float(loss.detach()))
    print(f"alpha fit: L1 {losses[0]:.4f} -> {losses[-1]:.4f}")
    assert losses[-1] < 0.5 * losses[0], losses
