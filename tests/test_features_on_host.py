"""Rendered feature maps (gsb_render_features, gsb_backward_features, gsb_backward_batch_features and the Python layer above
them) run from the kernel SOURCES on the CPU (tests/host_emul), against float64 autograd through oracle/torch_oracle.py.

The oracle's feature map is its colour output run group by group: colors_precomp = features[:, 3j:3j+3] (the last group padded
with zero channels) against a black background, so every gradient of a feature loss is the gradient of those colour calls.
The forward must also EQUAL the host build's own colors_precomp calls.  Bars: forward FWD_BAR absolute against the oracle,
gradients 1e-4 x the tensor's max magnitude.  Between host-build calls the bar is 1e-5 x max: the backward blend's float
atomics (host threads here) land in a different order from one call to the next."""
import math

import numpy as np
import pytest
import torch

import gs_test_util as U
from oracle import torch_oracle as TO

FWD_BAR = U.FWD_ABS_TOL
GRAD_BAR = 1e-4
SAME_BAR = 1e-5
GAUSS_KEYS = ("means3D", "means2D", "shs", "colors_precomp", "opacities", "scales", "rotations", "cov3D_precomp")


def _features(P, C, seed=3):
    return torch.randn(P, C, generator=torch.Generator().manual_seed(seed))


def _weights(cam, C, seed=5):
    gen = torch.Generator().manual_seed(seed)
    H, W = cam.image_height, cam.image_width
    return (torch.randn(3, H, W, generator=gen), torch.randn(1, H, W, generator=gen), torch.randn(1, H, W, generator=gen),
            torch.randn(C, H, W, generator=gen))


def _groups(C):
    return [(j, min(j + 3, C)) for j in range(0, C, 3)]


def _pad3(f):
    return torch.cat([f, f.new_zeros(f.shape[0], 3 - f.shape[1])], 1) if f.shape[1] < 3 else f


def oracle_features(d, feats, s):
    """Differentiable float64 feature map [C,H,W]: the oracle's colour, three channels at a time, with bg 0."""
    s0 = s._replace(bg=torch.zeros(3, dtype=torch.float64))
    maps = []
    for a, b in _groups(feats.shape[1]):
        col, _, _ = TO.rasterize(d["means3D"], d["means2D"], None, _pad3(feats[:, a:b]), d["opacities"], d["scales"],
                                 d["rotations"], d["cov3D_precomp"], s0)
        maps.append(col[:b - a])
    return torch.cat(maps, 0)


def oracle(args, cam, feats, wc=None, wd=None, wa=None, wf=None, cam_keys=()):
    """float64 oracle: (feature map, grads of sum(color wc) + sum(invdepth wd) + sum(alpha wa) + sum(F wf) for the gaussian
    inputs, the features and the camera tensors in cam_keys)."""
    P = args["means3D"].shape[0]
    d = {k: (None if args.get(k) is None else args[k].detach().double().clone().requires_grad_(True)) for k in GAUSS_KEYS}
    d["means2D"] = torch.zeros(P, 3, dtype=torch.float64, requires_grad=True)
    f = feats.detach().double().clone().requires_grad_(True)
    cams = {k: getattr(cam, k).detach().double().clone().requires_grad_(True) for k in cam_keys}
    s = cam._replace(**cams)
    F = oracle_features(d, f, s)
    loss = torch.zeros((), dtype=torch.float64)
    if wc is not None:
        color, _, invd = TO.rasterize(d["means3D"], d["means2D"], d["shs"], d["colors_precomp"], d["opacities"], d["scales"],
                                      d["rotations"], d["cov3D_precomp"], s)
        ones = torch.ones(P, 3, dtype=torch.float64)
        alpha, _, _ = TO.rasterize(d["means3D"], d["means2D"], None, ones, d["opacities"], d["scales"], d["rotations"],
                                   d["cov3D_precomp"], s._replace(bg=torch.zeros(3, dtype=torch.float64)))
        loss = loss + (color * wc.double()).sum() + (invd * wd.double()).sum() + (alpha[:1] * wa.double()).sum()
    if wf is not None:
        loss = loss + (F * wf.double()).sum()
    grads = {}
    if loss.requires_grad:
        loss.backward()
        for k, t in list(d.items()) + list(cams.items()) + [("features", f)]:
            if t is not None:
                grads[k] = (t.grad if t.grad is not None else torch.zeros_like(t)).numpy()
    return F.detach().numpy(), grads


def ours(dgr, args, cam, feats, wc=None, wd=None, wa=None, wf=None, split=False, cam_keys=(), bg=None):
    """Public path: GaussianRasterizer(..., return_alpha=True, features=...) + autograd on the host build."""
    rs = U.settings_to(cam, "cpu")
    if bg is not None:
        rs = rs._replace(bg=bg)
    cams = {k: getattr(rs, k).detach().clone().requires_grad_(True) for k in cam_keys}
    rs = rs._replace(**cams)
    t = {k: (v.detach().float().clone().requires_grad_(True) if v is not None else None) for k, v in args.items()}
    f = feats.detach().clone().requires_grad_(True)
    P = t["means3D"].shape[0]
    m2d = torch.zeros(P, 3, requires_grad=True)
    sh, dc = t["shs"], None
    if split and sh is not None:
        dc = t["shs"][:, :1].detach().clone().requires_grad_(True)
        sh = t["shs"][:, 1:].detach().clone().requires_grad_(True)
    color, radii, invd, alpha, F = dgr.GaussianRasterizer(rs)(
        means3D=t["means3D"], means2D=m2d, opacities=t["opacities"], shs=sh, colors_precomp=t["colors_precomp"],
        scales=t["scales"], rotations=t["rotations"], cov3D_precomp=t["cov3D_precomp"], dc=dc, return_alpha=True, features=f)
    loss = torch.zeros(())
    if wc is not None:
        loss = loss + (color * wc).sum() + (invd * wd).sum() + (alpha * wa).sum()
    if wf is not None:
        loss = loss + (F * wf).sum()
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
        grads["features"] = f.grad.numpy() if f.grad is not None else np.zeros(f.shape, np.float32)
        for k, v in cams.items():
            grads[k] = v.grad.numpy() if v.grad is not None else np.zeros(v.shape, np.float32)
    return F.detach(), grads, radii


def colors_precomp_calls(dgr, args, cam, feats, wf=None):
    """The workaround: one colors_precomp call per three channels with bg 0.  Returns (maps [C,H,W], summed geometric
    gradients of sum(F wf), dL/dfeatures)."""
    rs = U.settings_to(cam, "cpu")._replace(bg=torch.zeros(3))
    C = feats.shape[1]
    t = {k: (v.detach().float().clone().requires_grad_(True) if v is not None else None) for k, v in args.items()
         if k in ("means3D", "opacities", "scales", "rotations", "cov3D_precomp")}
    P = t["means3D"].shape[0]
    m2d = torch.zeros(P, 3, requires_grad=True)
    maps, gfeat = [], torch.zeros(P, C)
    for a, b in _groups(C):
        cp = _pad3(feats[:, a:b]).detach().clone().requires_grad_(True)
        col, _, _ = dgr.GaussianRasterizer(rs)(means3D=t["means3D"], means2D=m2d, opacities=t["opacities"], colors_precomp=cp,
                                               scales=t.get("scales"), rotations=t.get("rotations"),
                                               cov3D_precomp=t.get("cov3D_precomp"))
        maps.append(col[:b - a].detach())
        if wf is not None:
            (col[:b - a] * wf[a:b]).sum().backward()
            gfeat[:, a:b] = cp.grad[:, :b - a]
    geo = {k: v.grad.numpy() for k, v in t.items() if v is not None and v.grad is not None}
    geo["means2D"] = m2d.grad.numpy() if m2d.grad is not None else None
    return torch.cat(maps, 0), geo, gfeat.numpy()


def assert_grads_close(got, ref, what, bar=GRAD_BAR):
    for k, r in ref.items():
        g = np.asarray(got[k], dtype=np.float64).reshape(r.shape)
        scale = np.abs(r).max()
        err = np.abs(g - r).max()
        assert err <= bar * scale + 1e-12, f"{what}: d{k} err {err:.3e} vs max {scale:.3e}"


# ---- forward -------------------------------------------------------------------------------------------------------------
def _fwd_scenarios():
    out = []
    for deg, C in zip(range(4), (1, 3, 5, 8)):
        out.append((f"sh{deg}_C{C}", dict(P=220, seed=10 + deg), dict(w=48, h=32, sh_degree=deg), "sh", C))
    out.append(("precomp_C16", dict(P=220, seed=20), dict(w=48, h=32), "precomp", 16))
    out.append(("antialiasing_C5", dict(P=220, seed=21, log_scale_mean=-2.6), dict(w=56, h=40, antialiasing=True), "sh", 5))
    out.append(("ragged_C8", dict(P=200, seed=22), dict(w=70, h=41, sh_degree=2, scale_modifier=0.7), "sh", 8))
    out.append(("smaller_than_a_tile_C3", dict(P=120, seed=23, log_scale_mean=-2.0), dict(w=11, h=7, sh_degree=1), "sh", 3))
    out.append(("near_plane_through_cloud_C16", dict(P=300, seed=24, extent=2.0, log_scale_mean=-2.2),
                dict(w=48, h=32, eye=(0.1, -0.2, -0.3), sh_degree=1), "sh", 16))
    return out


@pytest.mark.parametrize("name,scn,camkw,mode,C", _fwd_scenarios(), ids=[s[0] for s in _fwd_scenarios()])
def test_forward_matches_oracle_and_equals_colors_precomp_calls(on_host, name, scn, camkw, mode, C):
    scn = dict(scn)
    P, seed = scn.pop("P"), scn.pop("seed")
    scn.setdefault("log_scale_mean", -2.4)
    scene = TO.make_scene(P, seed=seed, **scn)
    camkw = dict(camkw)
    w, h = camkw.pop("w"), camkw.pop("h")
    cam = TO.make_camera(w, h, bg=(0.1, 0.3, 0.6), **camkw)
    args = U.make_args(scene, mode)
    feats = _features(P, C, seed)
    got, _, _ = ours(on_host, args, cam, feats)
    ref, _ = oracle(args, cam, feats)
    assert got.shape == (C, h, w) and got.dtype == torch.float32
    assert np.abs(got.numpy() - ref).max() <= FWD_BAR, name
    assert float(got.abs().max()) > 0.1, name                    # the scene covers pixels
    maps, _, _ = colors_precomp_calls(on_host, args, cam, feats)
    assert torch.equal(got, maps), name                           # the colour path's own arithmetic, bit for bit


def test_forward_128_channels_equals_colors_precomp_calls(on_host):
    """C = 128 (16 groups of 8): every channel equals its colors_precomp call; a few groups also against the oracle."""
    scene = TO.make_scene(150, seed=26, log_scale_mean=-2.4)
    cam = TO.make_camera(40, 24, sh_degree=3)
    args = U.make_args(scene, "sh")
    feats = _features(150, 128, 26)
    got, _, _ = ours(on_host, args, cam, feats)
    maps, _, _ = colors_precomp_calls(on_host, args, cam, feats)
    assert got.shape == (128, 24, 40) and torch.equal(got, maps)
    ref, _ = oracle(args, cam, feats[:, 120:])
    assert np.abs(got[120:].numpy() - ref).max() <= FWD_BAR


def test_forward_opacity_zero_and_one(on_host):
    """Opacity 0: nothing blends, the map is 0.  Opacity 1 (capped at 0.99): many pixels reach the T < 1e-4 stop."""
    scene = TO.make_scene(400, seed=25, log_scale_mean=-1.2)
    cam = TO.make_camera(48, 32, sh_degree=0)
    feats = _features(400, 5, 25)
    for o in (0.0, 1.0):
        scene["opacities"] = torch.full((400, 1), o)
        args = U.make_args(scene, "sh")
        got, _, _ = ours(on_host, args, cam, feats)
        ref, _ = oracle(args, cam, feats)
        assert np.abs(got.numpy() - ref).max() <= FWD_BAR, o
        if o == 0.0:
            assert torch.all(got == 0.0)
        else:
            maps, _, _ = colors_precomp_calls(on_host, args, cam, feats)
            assert torch.equal(got, maps)


def test_empty_and_fully_culled_scenes(on_host):
    """No visible gaussian: the map is 0 and every gradient of a feature loss is exactly 0."""
    dgr = on_host
    cam = TO.make_camera(48, 32, sh_degree=0)
    wf = _weights(cam, 4)[3]
    for P in (0, 60):
        scene = TO.make_scene(P, seed=1, sh_coeffs=1)
        scene["means3D"][:, 2] -= 100.0
        got, grads, radii = ours(dgr, U.make_args(scene, "sh"), cam, _features(P, 4), wf=wf, cam_keys=("viewmatrix",))
        assert got.shape == (4, 32, 48) and (radii == 0).all() and torch.all(got == 0.0), P
        for k, g in grads.items():
            assert np.all(g == 0), (P, k)


# ---- gradients -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("deg,mode,camkw,C", [(0, "sh", {}, 1), (1, "sh", {}, 5), (2, "sh", dict(scale_modifier=0.7), 8),
                                              (3, "sh", {}, 16), (3, "precomp", {}, 3), (3, "sh", dict(antialiasing=True), 8),
                                              (1, "sh", dict(eye=(0.1, -0.2, -0.3)), 4)],
                         ids=["sh0_C1", "sh1_C5", "sh2_scale_modifier_C8", "sh3_C16", "precomp_C3", "antialiasing_C8",
                              "near_plane_C4"])
def test_gradients_match_oracle(on_host, deg, mode, camkw, C):
    """sum(F wf) alone, and colour + invdepth + alpha + feature terms together, against float64 autograd; for the feature-only
    loss the geometric gradients also equal the sum of the per-group colors_precomp calls' and dL/dfeatures their colour
    gradients."""
    near = "eye" in camkw
    scene = TO.make_scene(300 if near else 220, seed=30 + deg, extent=2.0 if near else 1.0,
                          log_scale_mean=-2.2 if near else -2.4)
    cam = TO.make_camera(70, 41, sh_degree=deg, bg=(0.2, 0.4, 0.6), **camkw)
    args = U.make_args(scene, mode)
    feats = _features(scene["means3D"].shape[0], C, deg)
    wc, wd, wa, wf = _weights(cam, C)
    _, g, _ = ours(on_host, args, cam, feats, wf=wf)
    _, r = oracle(args, cam, feats, wf=wf)
    assert_grads_close(g, r, f"feature loss deg {deg} {mode} {camkw}")
    assert np.all(g["shs" if mode == "sh" else "colors_precomp"] == 0)      # no colour gradient from features
    _, geo, gfeat = colors_precomp_calls(on_host, args, cam, feats, wf)
    assert_grads_close({k: g[k] for k in geo}, geo, "vs per-group calls", bar=SAME_BAR)
    assert_grads_close({"features": g["features"]}, {"features": gfeat}, "dL/dfeatures vs per-group calls", bar=SAME_BAR)
    _, g, _ = ours(on_host, args, cam, feats, wc, wd, wa, wf)
    _, r = oracle(args, cam, feats, wc, wd, wa, wf)
    assert_grads_close(g, r, f"combined loss deg {deg} {mode} {camkw}")


def test_split_sh_and_camera_gradients(on_host):
    """Split SH input and cameras that require grad, with a feature term: pose gradients match the oracle; features add
    nothing to dL/dbg or dL/dcampos."""
    dgr = on_host
    keys = ("viewmatrix", "projmatrix", "campos", "bg")
    for deg, M in ((0, 1), (3, 16)):
        scene = TO.make_scene(200, seed=40 + deg, sh_coeffs=M, log_scale_mean=-2.4)
        cam = TO.make_camera(48, 32, sh_degree=deg, bg=(0.1, 0.3, 0.6))
        args = U.make_args(scene, "sh")
        feats = _features(200, 6, deg)
        wc, wd, wa, wf = _weights(cam, 6)
        _, g, _ = ours(dgr, args, cam, feats, wc, wd, wa, wf, split=True, cam_keys=keys)
        _, r = oracle(args, cam, feats, wc, wd, wa, wf, cam_keys=keys)
        r = {k: v for k, v in r.items() if not (k == "campos" and deg == 0)}
        assert_grads_close(g, r, f"split deg {deg}")
        _, g_f, _ = ours(dgr, args, cam, feats, wf=wf, split=True, cam_keys=keys)
        _, r_f = oracle(args, cam, feats, wf=wf, cam_keys=keys)
        assert_grads_close({k: g_f[k] for k in ("viewmatrix", "projmatrix", "features")},
                           {k: r_f[k] for k in ("viewmatrix", "projmatrix", "features")}, f"pose from features, deg {deg}")
        assert np.all(g_f["campos"] == 0) and np.all(g_f["bg"] == 0)


# ---- C ABI ---------------------------------------------------------------------------------------------------------------
def _state(dgr, args, cam):
    rs = U.settings_to(cam, "cpu")
    f = {k: (v.detach().float().contiguous() if v is not None else None) for k, v in args.items()}
    f["opacities"] = f["opacities"].reshape(-1).contiguous()
    color, radii, invd, pack = dgr._forward_impl(f["means3D"], f["shs"], None, f["opacities"], f["scales"], f["rotations"], None, rs)
    return rs, f, color, invd, pack


def _abi_backward(dgr, rs, f, color, invd, pack, wc, wd, feat=None, entry="features"):
    P = f["means3D"].shape[0]
    g = dict(means3D=torch.zeros(P, 3), means2D=torch.zeros(P, 3), opacities=torch.zeros(P), shs=torch.zeros(P, 16, 3),
             scales=torch.zeros(P, 3), rotations=torch.zeros(P, 4))
    keep = []
    cs = dgr._c_settings(rs, pack["sh_coeffs"], keep)
    ci = dgr._c_inputs(P, f["means3D"], f["shs"], None, f["opacities"], f["scales"], f["rotations"], None)
    gg = dgr._Grads()
    for k, v in g.items():
        setattr(gg, {"shs": "dL_dshs"}.get(k, "dL_d" + k), v.data_ptr())
    arena = dgr._Arena(f["means3D"].device)
    dgr.reset_launch_count()
    if entry == "alpha":
        rc = dgr._C.gsb_backward_alpha(dgr.byref(cs), dgr.byref(ci), None, dgr.byref(pack["state"]), color.data_ptr(),
                                       invd.data_ptr(), wc.data_ptr(), wd.data_ptr(), None, dgr.byref(gg), None, 0, arena.cb, None,
                                       None)
    else:
        rc = dgr._C.gsb_backward_features(dgr.byref(cs), dgr.byref(ci), None, dgr.byref(pack["state"]), color.data_ptr(),
                                          invd.data_ptr(), wc.data_ptr(), wd.data_ptr(), None, dgr.byref(gg), None,
                                          dgr.byref(feat) if feat is not None else None, 0, arena.cb, None, None)
    return rc, g, dgr.launch_count(), arena


def test_null_features_is_the_existing_call(on_host):
    """gsb_backward_features with features NULL launches what gsb_backward_alpha does, with the same results; a zero feature
    gradient adds one launch and lands within the atomics-order bar."""
    dgr = on_host
    scene = TO.make_scene(200, seed=50, log_scale_mean=-2.4)
    cam = TO.make_camera(48, 32, sh_degree=3, bg=(0.1, 0.3, 0.6))
    args = U.make_args(scene, "sh")
    wc, wd, _, _ = _weights(cam, 1)
    rs, f, color, invd, pack = _state(dgr, args, cam)
    feats = _features(200, 8)
    fmap = dgr._features_impl(pack["state"], 32, 48, feats, f["means3D"].device)
    out = {}
    term = dict(features=feats, out=fmap, grad=torch.zeros_like(fmap), dL_dfeatures=torch.ones(200, 8))   # GsbFeatures' tensors
    for name in ("alpha", "null", "zeros"):
        ft = dgr._feature_term(term) if name == "zeros" else None
        rc, g, n, arena = _abi_backward(dgr, rs, f, color, invd, pack, wc, wd, ft, "alpha" if name == "alpha" else "features")
        dgr._check(rc, arena)
        out[name] = (g, n)
    assert out["null"][1] == out["alpha"][1] and out["zeros"][1] == out["alpha"][1] + 1
    for name in ("null", "zeros"):
        for k, v in out["alpha"][0].items():
            assert float((out[name][0][k] - v).abs().max()) <= SAME_BAR * float(v.abs().max()), (name, k)


def test_argument_errors(on_host):
    """gsb_render_features: bad V, channels, NULL output, NULL features, a state of another size; GsbFeatures: channels out
    of range, outputs without features, a gradient without the forward map; chunked or peer batches with features; the Python
    checks (ValueError)."""
    import bench
    from gaussian_renderer import render, render_views_backward
    dgr = on_host
    scene = TO.make_scene(120, seed=72, log_scale_mean=-2.4)
    cam = TO.make_camera(48, 32, sh_degree=3)
    args = U.make_args(scene, "sh")
    rs, f, color, invd, pack = _state(dgr, args, cam)
    feats = _features(120, 4)
    out = torch.zeros(129 * 64 * 64)
    st = (dgr._State * 17)()
    st[0] = pack["state"]
    for V, H, W, P, C, fp, op, msg in ((0, 32, 48, 120, 4, feats, out, "V=0"), (17, 32, 48, 120, 4, feats, out, "V=17"),
                                       (1, 32, 48, 120, 0, feats, out, "channels 0"),
                                       (1, 32, 48, 120, 129, feats, out, "channels 129"),
                                       (1, 32, 48, 120, 4, feats, None, "NULL"), (1, 32, 48, 120, 4, None, out, "NULL"),
                                       (1, 64, 64, 120, 4, feats, out, "is not a forward"),
                                       (1, 32, 48, 119, 4, feats, out, "is not a forward")):
        rc = dgr._C.gsb_render_features(V, st, H, W, P, C, fp.data_ptr() if fp is not None else None,
                                        op.data_ptr() if op is not None else None, None)
        assert rc != 0 and msg in dgr._C.gsb_last_error().decode(), msg
    fmap = dgr._features_impl(pack["state"], 32, 48, feats, f["means3D"].device)
    wc, wd, _, _ = _weights(cam, 1)
    bad = [(dict(channels=0), "outside 1..128"), (dict(channels=129), "outside 1..128"),
           (dict(features=None), "without features"), (dict(out_features=None), "without out_features")]
    term = dict(features=feats, out=fmap, grad=torch.zeros_like(fmap), dL_dfeatures=torch.zeros(120, 4))
    for change, msg in bad:
        ft = dgr._feature_term(term)
        for k, v in change.items():
            setattr(ft, k, v)
        rc, _, _, _ = _abi_backward(dgr, rs, f, color, invd, pack, wc, wd, ft)
        assert rc != 0 and msg in dgr._C.gsb_last_error().decode(), msg
    # view batch: chunks and peers are refused with features
    keep = []
    cs = dgr._c_settings(rs, pack["sh_coeffs"], keep)
    ci = dgr._c_inputs(120, f["means3D"], f["shs"], None, f["opacities"], f["scales"], f["rotations"], None)
    gg = dgr._Grads()
    ft = dgr._feature_term(dict(term, dL_dfeatures=None))
    sts = (dgr._State * 1)(pack["state"])
    pt = dgr._PeerTable()
    pt.world, pt.rank, pt.rows_per_rank = 1, 0, 256
    for peers, n_chunks in ((None, 2), (dgr.byref(pt), 1)):
        arena = dgr._Arena(f["means3D"].device)
        rc = dgr._C.gsb_backward_batch_features(1, dgr.byref(cs), dgr.byref(ci), sts, color.data_ptr(), invd.data_ptr(),
                                                wc.data_ptr(), None, None, dgr.byref(gg), None, dgr.byref(ft), peers, 0, n_chunks,
                                                dgr._CHUNK_FN(), None, arena.cb, None, None)
        assert rc != 0 and "chunked or peer" in dgr._C.gsb_last_error().decode()
    # Python layer
    rsp = U.settings_to(cam, "cpu")
    kw = dict(means3D=args["means3D"], means2D=torch.zeros(120, 3), opacities=args["opacities"], shs=args["shs"],
              scales=args["scales"], rotations=args["rotations"])
    for bad_f in (torch.zeros(120), torch.zeros(119, 4), torch.zeros(120, 0), torch.zeros(120, 129), torch.zeros(1, 120, 4)):
        with pytest.raises(ValueError):
            dgr.GaussianRasterizer(rsp)(**kw, features=bad_f)
    scene5 = TO.make_scene(120, seed=3, log_scale_mean=-2.4)
    bcam = bench.BenchCamera(48, 32, math.radians(60.0), *bench.view_pose(0, 3.0), "cpu")
    pc = bench.BenchGaussians(scene5, 3, "cpu")
    with pytest.raises(ValueError):
        render(bcam, pc, bench.Pipe(), torch.zeros(3), features=torch.zeros(7, 4))
    for kw2 in (dict(grad_chunks=2), dict(on_grad_chunk=lambda *a: None), dict(peers=(1, 0, 256, [0]))):
        with pytest.raises(ValueError):
            render_views_backward([bcam], pc, bench.Pipe(), torch.zeros(3), lambda img, d, i, features: img.mean(),
                                  features=torch.zeros(120, 4), **kw2)


# ---- view batch ----------------------------------------------------------------------------------------------------------
def _views(n=250, seed=60, V=5, W=48, H=32):
    import bench
    scene = TO.make_scene(n, seed=seed, log_scale_mean=-2.4)
    cams = [bench.BenchCamera(W, H, math.radians(60.0), *bench.view_pose(i, 3.0), "cpu") for i in range(V)]
    gts = [torch.rand(3, H, W, generator=torch.Generator().manual_seed(i)) for i in range(V)]
    ftgt = [torch.randn(6, H, W, generator=torch.Generator().manual_seed(200 + i)) for i in range(V)]
    return scene, cams, gts, ftgt, torch.tensor([0.1, 0.2, 0.3])


def _leaf_grads(pc, extra=()):
    out = {k: getattr(pc, k).grad.clone() for k in ("_xyz", "_shs", "_opacity", "_scaling", "_rotation")}
    for k in out:
        getattr(pc, k).grad = None
    for i, t in enumerate(extra):
        out[f"features{i}"] = t.grad.clone()
        t.grad = None
    return out


def _assert_same(a, b, what):
    for k, v in b.items():
        assert float((a[k] - v).abs().max()) <= SAME_BAR * float(v.abs().max()) + 1e-12, (what, k)


def test_view_batch_equals_single_view_calls(on_host):
    """render_views_backward(features=...) with V = 1 and V = 5, batched (sync, async forward) and view by view, in both
    loss modes, with a leaf and with a non-leaf feature tensor: the summed gradients equal those of render(features=...) +
    autograd per view; the maps handed to loss_fn and kept equal render()'s."""
    import bench
    from gaussian_renderer import AsyncCapacity, render, render_views_backward
    for V in (1, 5):
        scene, cams, gts, ftgt, bg = _views(V=V)
        raw = torch.randn(250, 6, generator=torch.Generator().manual_seed(9))
        loss_fn = lambda img, d, i, features: (img - gts[i]).abs().mean() + 0.5 * ((features - ftgt[i]) ** 2).mean()

        def loss_grad(img, d, i, features):
            n = img.numel()
            return ((img.clamp(0, 1) - gts[i]).abs().mean() + 0.5 * ((features - ftgt[i]) ** 2).mean(),
                    torch.sign(img.clamp(0, 1) - gts[i]) * ((img >= 0) & (img <= 1)) / n, None, None,
                    (features - ftgt[i]) / features.numel())
        pc = bench.BenchGaussians(scene, 3, "cpu")
        leaf = raw.clone().requires_grad_(True)
        maps = []
        for i, cm in enumerate(cams):
            pkg = render(cm, pc, bench.Pipe(), bg, features=leaf)
            loss_fn(pkg["render"], pkg["depth"], i, pkg["features"]).backward()
            maps.append(pkg["features"].detach())
        single = _leaf_grads(pc, (leaf,))
        cap = AsyncCapacity("cpu")
        cap.learn([200000])
        for kw in (dict(), dict(batched=False), dict(capacity=cap), dict(loss_returns_grad=True),
                   dict(loss_returns_grad=True, batched=False), dict(non_leaf=True)):
            kw = dict(kw)
            non_leaf = kw.pop("non_leaf", False)
            pc = bench.BenchGaussians(scene, 3, "cpu")
            leaf = raw.clone().requires_grad_(True)
            feats = leaf * 1.0 if non_leaf else leaf
            fn = loss_grad if kw.get("loss_returns_grad") else loss_fn
            out = render_views_backward(cams, pc, bench.Pipe(), bg, fn, features=feats, keep_images=True, **kw)
            _assert_same(_leaf_grads(pc, (leaf,)), single, f"V={V} {sorted(kw)} non_leaf={non_leaf}")
            assert len(out["features"]) == V
            for a, b in zip(out["features"], maps):
                assert a.shape == (6, 32, 48) and torch.equal(a, b)


def test_view_batch_kernel_matches_single_states_and_defaults(on_host):
    """gsb_render_features over a view batch's states (one launch) equals the single-view forwards' maps; without features
    every call launches what it did before; an unused map leaves the backward the plain one."""
    import bench
    from gaussian_renderer import render_views_backward
    dgr = on_host
    scene, cams, gts, ftgt, bg = _views(V=5)
    pc = bench.BenchGaussians(scene, 3, "cpu")
    rss = [dgr.GaussianRasterizationSettings(32, 48, math.tan(cm.FoVx / 2), math.tan(cm.FoVy / 2), bg, 1.0, cm.world_view_transform,
                                             cm.full_proj_transform, 3, cm.camera_center, False, False, False) for cm in cams]
    f = {k: v.detach().float().contiguous() for k, v in dict(m=pc.get_xyz, s=pc.get_features, o=pc.get_opacity.reshape(-1),
                                                               sc=pc.get_scaling, r=pc.get_rotation).items()}
    feats = _features(250, 13)
    _, _, _, pack = dgr._forward_batch_impl(f["m"], f["s"], f["o"], f["sc"], f["r"], rss)
    dgr.reset_launch_count()
    batch = dgr._features_impl(pack["states"], 32, 48, feats, f["m"].device)
    assert dgr.launch_count() == 1 and batch.shape == (5, 13, 32, 48)
    for v, rs in enumerate(rss):
        _, _, _, p1 = dgr._forward_impl(f["m"], f["s"], None, f["o"], f["sc"], f["r"], None, rs)
        assert torch.equal(batch[v], dgr._features_impl(p1["state"], 32, 48, feats, f["m"].device))
    counts = []
    for with_f in (False, True):
        pc = bench.BenchGaussians(scene, 3, "cpu")
        kw = dict(features=feats) if with_f else {}
        fn = (lambda img, d, i, features: img.mean()) if with_f else (lambda img, d, i: img.mean())
        dgr.reset_launch_count()
        render_views_backward(cams, pc, bench.Pipe(), bg, fn, **kw)
        counts.append(dgr.launch_count())
    assert counts[1] == counts[0] + 1          # the forward's one feature launch; the unused map adds no backward launch
    # GaussianRasterizer: without features the 3-tuple and the launches of before; with them one more forward launch and
    # one more backward launch when the map's gradient is used
    args = U.make_args(scene, "sh")
    rs = U.settings_to(TO.make_camera(48, 32, sh_degree=3, bg=(0.1, 0.3, 0.6)), "cpu")
    kw = dict(means3D=args["means3D"], means2D=torch.zeros(250, 3), opacities=args["opacities"], shs=args["shs"],
              scales=args["scales"], rotations=args["rotations"])
    fw, bw = [], []
    for mode in ("none", "unused", "used"):
        t = {k: v.detach().clone().requires_grad_(True) for k, v in kw.items()}
        dgr.reset_launch_count()
        out = dgr.GaussianRasterizer(rs)(**t) if mode == "none" else dgr.GaussianRasterizer(rs)(**t, features=feats)
        fw.append(dgr.launch_count())
        assert len(out) == (3 if mode == "none" else 4)
        loss = out[0].sum() + (out[3].sum() if mode == "used" else 0.0)
        dgr.reset_launch_count()
        loss.backward()
        bw.append(dgr.launch_count())
    assert fw[1] == fw[2] == fw[0] + 1 and bw[1] == bw[0] and bw[2] == bw[0] + 1
    with torch.no_grad():
        out = dgr.GaussianRasterizer(rs)(**kw, return_alpha=True, features=feats)
    assert len(out) == 5 and out[4].shape == (13, 32, 48)


def test_render_fit_learns_features(on_host):
    """Geometry frozen, features learned from zero with Adam through render(): the map is linear in the features, so the
    loss falls by orders of magnitude."""
    import bench
    from gaussian_renderer import render
    scene = TO.make_scene(200, seed=71, log_scale_mean=-2.4)
    pc = bench.BenchGaussians(scene, 3, "cpu")
    cam = bench.BenchCamera(48, 32, math.radians(60.0), *bench.view_pose(0, 3.0), "cpu")
    with torch.no_grad():
        target = render(cam, pc, bench.Pipe(), torch.zeros(3), features=_features(200, 4, 71))["features"]
    learned = torch.zeros(200, 4, requires_grad=True)
    opt = torch.optim.Adam([learned], lr=0.1)
    losses = []
    for _ in range(60):
        opt.zero_grad()
        loss = ((render(cam, pc, bench.Pipe(), torch.zeros(3), features=learned)["features"] - target) ** 2).mean()
        loss.backward()
        opt.step()
        losses.append(float(loss.detach()))
    assert pc._xyz.grad is not None
    assert losses[-1] < 1e-2 * losses[0], losses
