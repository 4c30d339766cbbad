"""Deterministic backward (gsb_set_deterministic, torch.use_deterministic_algorithms in the Python layer) run from the kernel
SOURCES on the CPU (tests/host_emul).  The host build runs a block's threads as concurrent host threads, so the default
backward's float atomics really do land in a varying order here, and the comparisons below that must be bit-equal would not
be without the deterministic path."""
import ctypes
import math
import threading
import warnings

import numpy as np
import pytest
import torch

import gs_test_util as U
from oracle import torch_oracle as TO

CLOSE = 1e-6       # deterministic vs default backward, relative to each tensor's largest magnitude (float reassociation)
LEAVES = ("_xyz", "_shs", "_opacity", "_scaling", "_rotation")


@pytest.fixture()
def torch_flag():
    """Restores torch's deterministic-algorithms flag (and warn_only) after the test."""
    was, warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    yield
    torch.use_deterministic_algorithms(was, warn_only=warn)


def _det(on: bool):
    torch.use_deterministic_algorithms(on)


def _views(n=250, seed=60, V=5, W=48, H=32):
    import bench
    scene = TO.make_scene(n, seed=seed, log_scale_mean=-2.4)
    cams = [bench.BenchCamera(W, H, math.radians(60.0), *bench.view_pose(i, 3.0), "cpu") for i in range(V)]
    return scene, cams, torch.tensor([0.1, 0.2, 0.3])


def _step(scene, cams, bg, **kw):
    """render_views_backward with a colour + inverse-depth + alpha loss; returns the leaves' gradients, means2D included."""
    import bench
    from gaussian_renderer import render_views_backward
    pc = bench.BenchGaussians(scene, 3, "cpu")
    P = scene["means3D"].shape[0]
    stats = dict(xyz_gradient_accum=torch.zeros(P, 1), denom=torch.zeros(P, 1))
    gen = torch.Generator().manual_seed(9)
    H, W = int(cams[0].image_height), int(cams[0].image_width)
    wc, wd, wa = torch.randn(3, H, W, generator=gen), torch.randn(1, H, W, generator=gen), torch.randn(1, H, W, generator=gen)

    def loss(img, dep, i, alpha=None):
        return (img * wc).sum() + (dep * wd).sum() + (alpha * wa).sum()
    render_views_backward(cams, pc, bench.Pipe(), bg, loss, with_alpha=True, densify_stats=stats, **kw)
    out = {}
    for k in LEAVES:     # on the CPU BenchGaussians shares its leaves with the scene tensors: take the gradient and clear it
        out[k] = getattr(pc, k).grad.clone()
        getattr(pc, k).grad = None
    out["means2D"] = stats["xyz_gradient_accum"].clone()     # sums of |dL/dmeans2D| over the views
    return out


def _assert_equal(a, b, what):
    for k in b:
        assert torch.equal(a[k], b[k]), f"{what}: {k} differs by {float((a[k] - b[k]).abs().max()):.3e}"


def _assert_close(a, b, what, bar=CLOSE):
    for k in b:
        scale = float(b[k].abs().max())
        err = float((a[k] - b[k]).abs().max())
        assert err <= bar * scale + 1e-30, f"{what}: {k} err {err:.3e} vs max {scale:.3e}"


@pytest.mark.parametrize("V", [1, 5])
def test_view_batch_is_invariant(on_host, torch_flag, V):
    """Under the flag the view-batch backward gives the same bits with tile order on and off, chunked, after an async forward
    with a capacity above the count, and on a repeat; and it stays within float reassociation of the default backward."""
    from gaussian_renderer import AsyncCapacity
    dgr = on_host
    scene, cams, bg = _views(V=V)
    _det(False)
    plain = _step(scene, cams, bg)
    _det(True)
    ref = _step(scene, cams, bg)
    _assert_close(ref, plain, "det vs default")
    _assert_equal(_step(scene, cams, bg), ref, "repeat")
    dgr.set_option("tile_order", 0)
    try:
        _assert_equal(_step(scene, cams, bg), ref, "tile_order 0")
    finally:
        dgr.set_option("tile_order", 1)
    _assert_equal(_step(scene, cams, bg, grad_chunks=2, on_grad_chunk=lambda *a: None), ref, "grad_chunks=2")
    cap = AsyncCapacity("cpu", capacity=4096)
    _assert_equal(_step(scene, cams, bg, capacity=cap), ref, "async batch")
    _assert_equal(_step(scene, cams, bg, batched=False), _step(scene, cams, bg, batched=False), "view by view, repeat")


def _single(dgr, args, cam, split=False, cam_keys=("viewmatrix", "projmatrix", "campos", "bg")):
    """GaussianRasterizer(return_alpha=True) + autograd with colour, inverse-depth and alpha losses and camera gradients."""
    rs = U.settings_to(cam, "cpu")
    cams = {k: getattr(rs, k).detach().clone().requires_grad_(True) for k in cam_keys}
    rs = rs._replace(**cams)
    t = {k: (v.detach().float().clone().requires_grad_(True) if v is not None else None) for k, v in args.items()}
    P = t["means3D"].shape[0]
    m2d = torch.zeros(P, 3, requires_grad=True)
    sh, dc = t["shs"], None
    if split:
        dc = t["shs"][:, :1].detach().clone().requires_grad_(True)
        sh = t["shs"][:, 1:].detach().clone().requires_grad_(True)
    color, _, invd, alpha = dgr.GaussianRasterizer(rs)(
        means3D=t["means3D"], means2D=m2d, opacities=t["opacities"], shs=sh, colors_precomp=t["colors_precomp"],
        scales=t["scales"], rotations=t["rotations"], cov3D_precomp=t["cov3D_precomp"], dc=dc, return_alpha=True)
    gen = torch.Generator().manual_seed(5)
    loss = (color * torch.randn(color.shape, generator=gen)).sum() + (invd * torch.randn(invd.shape, generator=gen)).sum() + \
        (alpha * torch.randn(alpha.shape, generator=gen)).sum()
    loss.backward()
    out = {k: v.grad.clone() for k, v in t.items() if v is not None and k != "shs"}
    out["shs"] = torch.cat([dc.grad, sh.grad], 1) if split else t["shs"].grad.clone()
    out["means2D"] = m2d.grad.clone()
    out.update({k: v.grad.clone() for k, v in cams.items()})
    return out


@pytest.mark.parametrize("split", [False, True])
def test_single_view_is_invariant(on_host, torch_flag, split):
    """The drop-in path (alpha, inverse depth, camera gradients, joint and split SH): repeats and tile order give the same bits."""
    dgr = on_host
    scene = TO.make_scene(300, seed=31, log_scale_mean=-2.4)
    cam = TO.make_camera(48, 32, sh_degree=3, bg=(0.1, 0.3, 0.6))
    args = U.make_args(scene, "sh")
    _det(False)
    plain = _single(dgr, args, cam, split)
    _det(True)
    ref = _single(dgr, args, cam, split)
    _assert_close(ref, plain, "det vs default")
    _assert_equal(_single(dgr, args, cam, split), ref, "repeat")
    dgr.set_option("tile_order", 0)
    try:
        _assert_equal(_single(dgr, args, cam, split), ref, "tile_order 0")
    finally:
        dgr.set_option("tile_order", 1)


@pytest.mark.parametrize("mode", ["sh", "precomp"])
def test_against_oracle(on_host, torch_flag, mode):
    """Under the flag the gradients meet the project's float64-oracle bars."""
    scene = TO.make_scene(220, seed=17, log_scale_mean=-2.6)
    cam = TO.make_camera(48, 32, sh_degree=2, bg=(0.2, 0.1, 0.4))
    args = U.make_args(scene, mode)
    gen = torch.Generator().manual_seed(2)
    wc, wd = torch.randn(3, 32, 48, generator=gen).numpy(), torch.randn(1, 32, 48, generator=gen).numpy()
    _det(True)
    got = U.run_cuda(args, cam, wc, wd, device="cpu")
    ref = U.run_oracle(args, cam, wc, wd)
    U.assert_grads_close(got["grads"], ref["grads"], flips=U.count_flips(got["color"], ref["color"]))


def _one_band_scene(P=400, W=64, H=48, seed=3):
    """Sub-pixel gaussians, each at least 4 pixels inside one 16 x 8 band of one tile: one (list entry, warp) addend each."""
    cam = TO.make_camera(W, H, sh_degree=1, bg=(0.1, 0.2, 0.3))
    scene = TO.make_scene(P, seed=seed, log_scale_mean=-7.0, log_scale_std=0.1)
    d = {k: v.double() for k, v in scene.items()}
    pr = TO.project(d["means3D"], torch.zeros(P, 3, dtype=torch.float64), d["shs"], None, d["opacities"], d["scales"],
                    d["rotations"], None, cam)
    x, y = pr.xy[:, 0], pr.xy[:, 1]
    fx, fy = torch.remainder(x, 16.0), torch.remainder(y, 8.0)
    keep = pr.visible & (fx >= 4) & (fx <= 12) & (fy >= 3.5) & (fy <= 4.5) & (x > 0) & (y > 0) & (x < W) & (y < H)
    idx = torch.nonzero(keep).reshape(-1)
    return {k: v[idx] for k, v in scene.items()}, cam


def test_single_addend_is_bit_exact(on_host, torch_flag):
    """With one addend per gaussian the deterministic partials are the default path's sums: bit-equal gradients."""
    scene, cam = _one_band_scene()
    assert scene["means3D"].shape[0] >= 5
    args = U.make_args(scene, "sh")
    gen = torch.Generator().manual_seed(4)
    wc, wd = torch.randn(3, 48, 64, generator=gen).numpy(), torch.randn(1, 48, 64, generator=gen).numpy()
    _det(False)
    plain = U.run_cuda(args, cam, wc, wd, device="cpu")["grads"]
    _det(True)
    det = U.run_cuda(args, cam, wc, wd, device="cpu")["grads"]
    assert np.abs(plain["opacities"]).max() > 0
    for k, g in plain.items():
        if g is not None:
            assert np.array_equal(det[k], g), k


def test_no_unwritten_partial_is_read(on_host, torch_flag, monkeypatch):
    """Every scratch buffer filled with NaN before use: the deterministic gradients are finite and those of a normal run."""
    dgr = on_host
    scene, cams, bg = _views(V=3)
    _det(True)
    ref = _step(scene, cams, bg)
    dgr.release_scratch()
    real = dgr._Arena._alloc

    def nan_alloc(self, ctx, which, nbytes):
        p = real(self, ctx, which, nbytes)
        if int(which) >= 3 and p:
            self.bufs[int(which)].fill_(0xFF)     # all-ones bytes: float NaN, u32 0xffffffff
        return p
    monkeypatch.setattr(dgr._Arena, "_alloc", nan_alloc)
    got = _step(scene, cams, bg)
    for k, g in got.items():
        assert torch.isfinite(g).all(), k
    _assert_equal(got, ref, "NaN-filled scratch")
    dgr.release_scratch()


def test_switch_is_per_thread(on_host):
    C = on_host._C
    C.gsb_set_deterministic(0)
    assert C.gsb_set_deterministic(1) == 0
    assert C.gsb_set_deterministic(1) == 1
    seen = []
    th = threading.Thread(target=lambda: seen.append(C.gsb_set_deterministic(0)))
    th.start()
    th.join()
    assert seen == [0]                           # another thread starts with the switch off
    assert C.gsb_set_deterministic(0) == 1       # and did not touch this one's


def test_launch_counts(on_host, torch_flag):
    """Flag off: the default launches.  Flag on: 4 + ceil(ceil(log2 P) / 8) more per backward call (count, prepare, sort
    histogram, sort passes, reduce)."""
    dgr = on_host
    scene, cams, bg = _views(V=2)
    n = {}
    for on in (False, True, False):
        _det(on)
        dgr.reset_launch_count()
        _step(scene, cams, bg)
        n.setdefault(on, []).append(dgr.launch_count())
    assert n[False][0] == n[False][1]
    bits = math.ceil(math.log2(250))
    assert n[True][0] == n[False][0] + 4 + math.ceil(bits / 8)


def test_paths_without_a_deterministic_implementation(on_host, torch_flag):
    """features= with a map loss, contrib= and peers= raise RuntimeError under the flag and warn with warn_only=True; a feature
    forward without a map loss is deterministic and allowed."""
    import bench
    from gaussian_renderer import render_views_backward
    dgr = on_host
    scene, cams, bg = _views(V=2)
    P = scene["means3D"].shape[0]
    feats = torch.randn(P, 4)

    def run(**kw):
        pc = bench.BenchGaussians(scene, 3, "cpu")
        fl = kw.pop("feature_loss", False)

        def loss(img, dep, i, features=None):
            return img.mean() + (features.mean() if fl else 0.0)
        return render_views_backward(cams, pc, bench.Pipe(), bg, loss, **kw)
    cases = [dict(features=feats, feature_loss=True), dict(contrib=dgr.ContributionStats(P, "cpu"))]
    for kw in cases:
        torch.use_deterministic_algorithms(True)
        with pytest.raises(RuntimeError, match="use_deterministic_algorithms"):
            run(**dict(kw))
        torch.use_deterministic_algorithms(True, warn_only=True)
        with pytest.warns(UserWarning, match="deterministic"):
            run(**dict(kw))
    torch.use_deterministic_algorithms(True)
    with warnings.catch_warnings():
        warnings.simplefilter("error")
        run(features=feats)                      # the feature map without a loss on it: no feature backward
    # peers: the Python layer refuses before any peer memory is touched
    _, _, _, pack = dgr._forward_batch_impl(*_flat(bench.BenchGaussians(scene, 3, "cpu")), _settings(dgr, cams, bg))
    with pytest.raises(RuntimeError, match="use_deterministic_algorithms"):
        _peer_backward(dgr, scene, pack, cams, bg)


def _flat(pc):
    return [t.detach().float().contiguous() for t in (pc.get_xyz, pc.get_features, pc.get_opacity.reshape(-1), pc.get_scaling,
                                                      pc.get_rotation)]


def _settings(dgr, cams, bg):
    return [dgr.GaussianRasterizationSettings(int(cm.image_height), int(cm.image_width), math.tan(cm.FoVx / 2),
                                              math.tan(cm.FoVy / 2), bg, 1.0, cm.world_view_transform, cm.full_proj_transform, 3,
                                              cm.camera_center, False, False, False) for cm in cams]


def _batch_grads(P, V, M=16):
    return dict(means3D=torch.zeros(P, 3), means2D=torch.zeros(V, P, 3), shs=torch.zeros(P, M, 3), opacities=torch.zeros(P),
                scales=torch.zeros(P, 3), rotations=torch.zeros(P, 4))


def _peer_backward(dgr, scene, pack, cams, bg, feats=None):
    import bench
    f = _flat(bench.BenchGaussians(scene, 3, "cpu"))
    P, V = f[0].shape[0], len(cams)
    H, W = int(cams[0].image_height), int(cams[0].image_width)
    g = _batch_grads(P, V)
    peers = None if feats is not None else (1, 0, P, [g["means3D"].data_ptr()])
    col, dep = torch.zeros(V, 3, H, W), torch.zeros(V, 1, H, W)
    dgr._backward_batch_impl(pack, _settings(dgr, cams, bg), *f, col, dep, torch.ones(V, 3, H, W), torch.ones(V, 1, H, W), g, True,
                             peers=peers, feats=feats)


def test_c_refuses_feature_term_and_peers(on_host, monkeypatch):
    """With the switch on, the C ABI returns GSB_ERR_ARGUMENT for a feature term with a map gradient and for peers."""
    import bench
    dgr = on_host
    monkeypatch.setattr(dgr, "_deterministic", lambda what=None: True)     # hand the switch to the C unconditionally
    scene, cams, bg = _views(V=2)
    P = scene["means3D"].shape[0]
    H, W = int(cams[0].image_height), int(cams[0].image_width)
    _, _, _, pack = dgr._forward_batch_impl(*_flat(bench.BenchGaussians(scene, 3, "cpu")), _settings(dgr, cams, bg))
    with pytest.raises(RuntimeError, match="no deterministic implementation"):
        _peer_backward(dgr, scene, pack, cams, bg)
    feats = dict(features=torch.randn(P, 4), out=torch.zeros(2, 4, H, W), grad=torch.ones(2, 4, H, W), dL_dfeatures=None)
    with pytest.raises(RuntimeError, match="no deterministic implementation"):
        _peer_backward(dgr, scene, pack, cams, bg, feats=feats)
    dgr._C.gsb_set_deterministic(0)
    assert ctypes.c_int32(dgr._C.gsb_set_deterministic(0)).value == 0
