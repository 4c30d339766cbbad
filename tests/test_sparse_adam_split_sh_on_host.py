"""Split SH input (gsb_forward_split_sh / gsb_backward_split_sh) and SparseGaussianAdam (gsb_sparse_adam_step) run from the
kernel SOURCES on the CPU (tests/host_emul).  The split path must reproduce the joint path's image, radii and inverse depth
bit for bit, and its gradients with dL_ddc / dL_drest in the places of rows 0 / 1.. of the joint dL_dshs.  The gradients
are compared at GRAD_BAR x max: the backward blend's float atomics, host threads here, land in a different order from one
run to the next (two joint runs differ by ~3e-7 x max).  The optimizer is checked against tests/sparse_adam_oracle.py,
against the flat store's sparse mode and against a fixture recorded from the reference's own scene.GaussianModel (tests/golden/make_golden_sparse.py)."""
import os
import subprocess
import sys
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import gs_test_util as U
from oracle import torch_oracle as TO
from oracle.model_oracle import GROUPS
from sparse_adam_oracle import SparseGaussianAdamOracle, SparseModelOracle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "gaussian-splatting_b200")
GOLD = os.path.join(ROOT, "tests", "golden", "reference_sparse_adam.npz")
RAW_KEY = {"xyz": "_xyz", "f_dc": "_features_dc", "f_rest": "_features_rest", "opacity": "_opacity", "scaling": "_scaling",
           "rotation": "_rotation"}
ACT = ("xyz", "features", "opacity", "scaling", "rotation")
SHAPES = {"xyz": (3,), "f_dc": (1, 3), "f_rest": (15, 3), "opacity": (1,), "scaling": (3,), "rotation": (4,)}
GRAD_BAR = 1e-5
LRS = {"xyz": 1.6e-4, "f_dc": 2.5e-3, "f_rest": 1.25e-4, "opacity": 2.5e-2, "scaling": 5e-3, "rotation": 1e-3}


def raster_split_vs_joint(dgr, P, M, deg, aa, W, H, accumulate, seed=0, dev="cpu", log_scale_mean=-2.4):
    """Forward + backward of the same inputs through the joint and the split entry points; returns both results."""
    scene = {k: v.to(dev) for k, v in TO.make_scene(P, seed=seed, sh_coeffs=M, log_scale_mean=log_scale_mean).items()}
    cam = TO.make_camera(W, H, sh_degree=deg, antialiasing=aa, bg=(0.1, 0.3, 0.6))
    rs = U.settings_to(cam, dev)
    gen = torch.Generator().manual_seed(seed + 1)
    gc, gd = torch.randn(3, H, W, generator=gen).to(dev), torch.randn(1, H, W, generator=gen).to(dev)
    sh = scene["shs"].contiguous()
    means, opac, sc, rot = scene["means3D"], scene["opacities"].reshape(-1).contiguous(), scene["scales"], scene["rotations"]
    base = {k: torch.randn(*s, generator=gen).to(dev) for k, s in
            (("means3D", (P, 3)), ("means2D", (P, 3)), ("opacities", (P,)), ("scales", (P, 3)), ("rotations", (P, 4)), ("shs", (P, M, 3)))}
    out = {}
    for split in (False, True):
        dc = sh[:, :1].contiguous() if split else None
        rest = (sh[:, 1:].contiguous() if M > 1 else None) if split else sh
        color, radii, invd, pack = dgr._forward_impl(means, rest, None, opac, sc, rot, None, rs, dc=dc)
        grads = {k: (v.clone() if accumulate else torch.full_like(v, float("nan"))) for k, v in base.items() if k != "shs"}
        if split:
            grads["dc"] = base["shs"][:, :1].contiguous() if accumulate else torch.full((P, 1, 3), float("nan"), device=dev)
            if M > 1:
                grads["shs"] = base["shs"][:, 1:].contiguous() if accumulate else torch.full((P, M - 1, 3), float("nan"), device=dev)
        else:
            grads["shs"] = base["shs"].clone() if accumulate else torch.full((P, M, 3), float("nan"), device=dev)
        dgr._backward_impl(pack, rs, means, rest, None, opac, sc, rot, None, color, invd, gc, gd, grads, accumulate, dc=dc)
        if split:
            grads["shs"] = torch.cat((grads["dc"], grads["shs"]), 1) if M > 1 else grads["dc"]
            del grads["dc"]
        out[split] = dict(color=color, radii=radii, invdepth=invd, grads=grads)
    return out[False], out[True]


@pytest.mark.parametrize("deg,M", [(0, 1), (0, 16), (1, 4), (2, 9), (3, 16)])
@pytest.mark.parametrize("aa", [False, True])
def test_split_sh_is_bit_equal_to_joint(on_host, deg, M, aa):
    """Every combination of pre_tma (joint path: TMA rows vs staged rows; the split path always stages) and accumulate, on a
    ragged image (40 x 27: partial tiles)."""
    dgr = on_host
    for tma in (0, 1):
        dgr.set_option("pre_tma", tma)
        try:
            for acc in (False, True):
                j, s = raster_split_vs_joint(dgr, 120, M, deg, aa, 40, 27, acc, seed=deg * 7 + M)
                what = f"deg {deg} M {M} aa {aa} pre_tma {tma} accumulate {acc}"
                assert int((j["radii"] > 0).sum()) > 10, what
                for k in ("color", "radii", "invdepth"):
                    assert torch.equal(j[k], s[k]), f"{k}: {what}"
                for k, v in j["grads"].items():
                    w = s["grads"][k]
                    assert not torch.isnan(v).any() and not torch.isnan(w).any(), f"grad {k} not written: {what}"
                    assert float((v - w).abs().max()) <= GRAD_BAR * float(v.abs().max()), f"grad {k}: {what}"
        finally:
            dgr.set_option("pre_tma", 1)


def test_rasterizer_api_split_sh_autograd(on_host):
    """GaussianRasterizer.forward(dc=..., shs=rest): gradients come back shaped like dc and rest (rest may be empty), equal to
    the joint call's; the argument checks keep their messages."""
    dgr = on_host
    wc = torch.randn(3, 32, 48, generator=torch.Generator().manual_seed(3))
    for M in (4, 1):
        cam = TO.make_camera(48, 32, sh_degree=1 if M == 4 else 0, bg=(0.2, 0.2, 0.2))
        rast = dgr.GaussianRasterizer(U.settings_to(cam, "cpu"))
        scene = TO.make_scene(120, seed=5, sh_coeffs=M, log_scale_mean=-2.2)
        leaf = lambda t: t.detach().clone().requires_grad_(True)
        kw = dict(opacities=scene["opacities"], scales=scene["scales"], rotations=scene["rotations"])
        joint = leaf(scene["shs"])
        img_j = rast(means3D=scene["means3D"], means2D=torch.zeros(120, 3), shs=joint, **kw)[0]
        (img_j * wc).sum().backward()
        dc, rest = leaf(scene["shs"][:, :1]), leaf(scene["shs"][:, 1:])
        img_s = rast(means3D=scene["means3D"], means2D=torch.zeros(120, 3), shs=rest, dc=dc, **kw)[0]
        (img_s * wc).sum().backward()
        assert torch.equal(img_j, img_s)
        assert dc.grad.shape == (120, 1, 3) and rest.grad.shape == (120, M - 1, 3)
        bar = GRAD_BAR * float(joint.grad.abs().max())
        assert float((dc.grad - joint.grad[:, :1]).abs().max()) <= bar
        assert M == 1 or float((rest.grad - joint.grad[:, 1:]).abs().max()) <= bar
    with pytest.raises(Exception, match="SHs or precomputed colors"):
        rast(means3D=scene["means3D"], means2D=torch.zeros(120, 3), dc=dc, **kw)
    with pytest.raises(Exception, match="not with precomputed colors"):
        rast(means3D=scene["means3D"], means2D=torch.zeros(120, 3), colors_precomp=torch.rand(120, 3), dc=dc, **kw)


def test_abi_rejects_inconsistent_split_input(on_host):
    """check_inputs: dc with colors_precomp, a rest pointer with sh_coeffs == 1, in->shs next to the split input."""
    dgr = on_host
    scene = TO.make_scene(10, seed=1, sh_coeffs=4)
    rs = U.settings_to(TO.make_camera(16, 16, sh_degree=0), "cpu")
    keep = []
    P = 10
    dc, rest = scene["shs"][:, :1].contiguous(), scene["shs"][:, 1:].contiguous()
    args = (scene["means3D"], scene["opacities"].reshape(-1).contiguous(), scene["scales"], scene["rotations"])

    def call(M, shs, colors, sp_dc, sp_rest):
        cs = dgr._c_settings(rs, M, keep)
        ci = dgr._c_inputs(P, args[0], shs, colors, args[1], args[2], args[3], None)
        sp = dgr._split_sh(sp_dc, sp_rest)
        arena = dgr._Arena(scene["means3D"].device)
        out = (torch.empty(3, 16, 16), torch.empty(P, dtype=torch.int32), torch.empty(1, 16, 16))
        rc = dgr._C.gsb_forward_split_sh(dgr.byref(cs), dgr.byref(ci), dgr.byref(sp), out[0].data_ptr(), out[1].data_ptr(),
                                         out[2].data_ptr(), 0, arena.cb, None, dgr.byref(dgr._State()), None)
        return rc, dgr._C.gsb_last_error().decode()

    rc, msg = call(4, None, torch.rand(P, 3), dc, rest)
    assert rc != 0 and "colors_precomp" in msg
    rc, msg = call(1, None, None, dc, rest)
    assert rc != 0 and "sh_coeffs == 1" in msg
    rc, msg = call(4, scene["shs"], None, dc, rest)
    assert rc != 0 and "in->shs must be NULL" in msg
    assert call(4, None, None, dc, rest)[0] == 0 and call(1, None, None, dc, None)[0] == 0


def test_render_separate_sh_matches_joint(on_host):
    """gaussian_renderer.render(separate_sh=True) hands dc / rest to the rasterizer: same image and gradients as
    separate_sh=False on a model whose dc and rest are separate leaves."""
    import bench
    from gaussian_renderer import render
    scene = TO.make_scene(150, seed=8, log_scale_mean=-2.4)
    cam = bench.BenchCamera(48, 32, 1.0, *bench.view_pose(0, 3.0), "cpu")
    out = {}
    for sep in (False, True):
        pc = RefShaped(scene)
        pkg = render(cam, pc, bench.Pipe(), torch.tensor([0.1, 0.2, 0.3]), separate_sh=sep)
        (pkg["render"] * torch.linspace(-1, 1, 3 * 32 * 48).view(3, 32, 48)).sum().backward()
        out[sep] = (pkg["render"].detach(), {n: p.grad.clone() for n, p in pc.named().items()})
    assert torch.equal(out[False][0], out[True][0])
    for n, ref in out[False][1].items():
        assert float((ref - out[True][1][n]).abs().max()) <= GRAD_BAR * float(ref.abs().max()), n


class RefShaped:
    """The reference scene.GaussianModel's six raw leaves and activations (scene/gaussian_model.py:102-130)."""

    def __init__(self, scene, dev="cpu"):
        leaf = lambda t: torch.nn.Parameter(t.detach().to(dev).contiguous().clone())
        self._xyz, self._features_dc, self._features_rest = leaf(scene["means3D"]), leaf(scene["shs"][:, :1]), leaf(scene["shs"][:, 1:])
        self._opacity = leaf(torch.log(scene["opacities"] / (1 - scene["opacities"])))
        self._scaling, self._rotation = leaf(torch.log(scene["scales"])), leaf(scene["rotations"])
        self.active_sh_degree = self.max_sh_degree = 3

    def named(self):
        return {"xyz": self._xyz, "f_dc": self._features_dc, "f_rest": self._features_rest, "opacity": self._opacity,
                "scaling": self._scaling, "rotation": self._rotation}

    get_xyz = property(lambda self: self._xyz)
    get_features = property(lambda self: torch.cat((self._features_dc, self._features_rest), 1))
    get_features_dc = property(lambda self: self._features_dc)
    get_features_rest = property(lambda self: self._features_rest)
    get_opacity = property(lambda self: torch.sigmoid(self._opacity))
    get_scaling = property(lambda self: torch.exp(self._scaling))
    get_rotation = property(lambda self: torch.nn.functional.normalize(self._rotation))


def make_groups(P, seed, dev="cpu"):
    g = torch.Generator().manual_seed(seed)
    return {n: torch.randn(P, *SHAPES[n], generator=g).to(dev) for n in GROUPS}


def optimizers(cls_a, cls_b, init):
    """cls_a over parameters on init's device, cls_b (the oracle) over CPU copies."""
    pa = {n: torch.nn.Parameter(init[n].clone()) for n in GROUPS}
    pb = {n: torch.nn.Parameter(init[n].cpu().clone()) for n in GROUPS}
    oa = cls_a([{"params": [pa[n]], "lr": LRS[n], "name": n} for n in GROUPS], lr=0.0, eps=1e-15)
    ob = cls_b([{"params": [pb[n]], "lr": LRS[n], "name": n} for n in GROUPS], lr=0.0, eps=1e-15)
    return pa, oa, pb, ob


def run_sparse_adam_against_oracle(P, dev, steps=3, seed=0):
    """Both optimizers stepped with the same gradients and masks; f_rest has no gradient in step 1.  Checks the invariants
    and bars of the issue: invisible rows bit-unchanged, visible rows within 2e-6 (params) / 1e-4 rel (moments), a group
    without gradient untouched, step never advanced, torch.optim.Adam's state keys."""
    from diff_gaussian_rasterization.sparse_adam import SparseGaussianAdam
    pa, oa, pb, ob = optimizers(SparseGaussianAdam, SparseGaussianAdamOracle, make_groups(P, seed, dev))
    g = torch.Generator().manual_seed(seed + 100)
    for it in range(steps):
        vis = (torch.rand(P, generator=g) < 0.5).to(dev)
        if P == 1:
            vis[:] = it % 2 == 0
        for n in GROUPS:
            gr = (torch.randn(P, *SHAPES[n], generator=g) * 1e-2).to(dev)
            skip = it == 1 and n == "f_rest"
            pa[n].grad = None if skip else gr.clone()
            pb[n].grad = None if skip else gr.cpu().clone()
        before = {n: (pa[n].detach().clone(), {k: v.clone() for k, v in oa.state[pa[n]].items() if k != "step"}) for n in GROUPS}
        oa.step(vis, P)
        ob.step(vis.cpu(), P)
        for n in GROUPS:
            st_a, st_b = oa.state[pa[n]], ob.state[pb[n]]
            p0, mom0 = before[n]
            if it == 1 and n == "f_rest":
                assert torch.equal(pa[n].detach(), p0) and all(torch.equal(st_a[k], mom0[k]) for k in mom0), n
                continue
            assert sorted(st_a) == ["exp_avg", "exp_avg_sq", "step"] and float(st_a["step"]) == 0.0
            inv = ~vis
            assert torch.equal(pa[n].detach()[inv], p0[inv]), n
            for k in ("exp_avg", "exp_avg_sq"):
                prev = mom0[k][inv] if k in mom0 else torch.zeros_like(st_a[k][inv])
                assert torch.equal(st_a[k][inv], prev), (n, k)
                torch.testing.assert_close(st_a[k].cpu(), st_b[k], rtol=1e-4, atol=1e-9 if k == "exp_avg" else 1e-13,
                                           msg=lambda s: f"{n} {k}: {s}")
            torch.testing.assert_close(pa[n].detach().cpu(), pb[n].detach(), rtol=0, atol=2e-6, msg=lambda s: f"{n}: {s}")
            assert not torch.equal(pa[n].detach()[vis], p0[vis]) or int(vis.sum()) == 0, n
        oa.zero_grad(set_to_none=True)
        ob.zero_grad(set_to_none=True)
    return oa


@pytest.mark.parametrize("P", [1, 33, 2011])
def test_sparse_adam_source_matches_oracle(on_host, P):
    dgr = on_host
    dgr.reset_launch_count()
    run_sparse_adam_against_oracle(P, "cpu")
    assert dgr.launch_count() == 3                     # one launch per step, every group in it


def test_sparse_adam_argument_errors(on_host):
    from diff_gaussian_rasterization.sparse_adam import SparseGaussianAdam
    P = 20
    p = {n: torch.nn.Parameter(t) for n, t in make_groups(P, 1).items()}
    opt = SparseGaussianAdam([{"params": [p[n]], "lr": LRS[n], "name": n} for n in GROUPS], lr=0.0, eps=1e-15)
    for n in GROUPS:
        p[n].grad = torch.ones_like(p[n])
    vis = torch.ones(P, dtype=torch.bool)
    with pytest.raises(ValueError, match="visibility"):
        opt.step(vis[:-1], P)
    with pytest.raises(ValueError, match="expected"):
        opt.step(torch.ones(P + 1, dtype=torch.bool), P + 1)
    q = torch.nn.Parameter(torch.randn(3, P).t())                   # [P,3], not contiguous
    q.grad = torch.ones(P, 3)
    with pytest.raises(ValueError, match="contiguous"):
        SparseGaussianAdam([q], lr=0.1, eps=1e-15).step(vis, P)
    two = SparseGaussianAdam([{"params": [p["xyz"], p["scaling"]]}], lr=0.1, eps=1e-15)
    with pytest.raises(ValueError, match="exactly one tensor"):
        two.step(vis, P)


def test_sparse_adam_refuses_cpu_tensors(host_lib):
    """Outside the host-build fixture the product layer refuses CPU tensors: no CPU path."""
    from diff_gaussian_rasterization.sparse_adam import SparseGaussianAdam
    x = torch.nn.Parameter(torch.zeros(4, 3))
    x.grad = torch.ones(4, 3)
    with pytest.raises(RuntimeError, match="no CPU"):
        SparseGaussianAdam([x], lr=0.1, eps=1e-15).step(torch.ones(4, dtype=torch.bool), 4)


def test_sparse_adam_equals_store_sparse_mode(on_host):
    """The flat store's optimizer_type="sparse_adam" and SparseGaussianAdam run the same device function with the same
    arguments: on the identity-activated groups (xyz, f_dc, f_rest) they agree bit for bit."""
    from diff_gaussian_rasterization.sparse_adam import SparseGaussianAdam
    from gaussian_store import GaussianModel, store_offsets
    P, M = 257, 16
    init = make_groups(P, 4)
    m = GaussianModel(3, optimizer_type="sparse_adam").create_from_tensors(init["xyz"], init["f_dc"], init["f_rest"], init["scaling"],
                                                                          init["rotation"], init["opacity"], 2.0)
    m.training_setup(SimpleNamespace(position_lr_init=1.6e-4, position_lr_final=1.6e-6, position_lr_delay_mult=0.01,
                                     position_lr_max_steps=30000, feature_lr=2.5e-3, opacity_lr=0.025, scaling_lr=5e-3,
                                     rotation_lr=1e-3, percent_dense=0.01))
    names = ("xyz", "f_dc", "f_rest")
    p = {n: torch.nn.Parameter(init[n].clone()) for n in names}
    opt = SparseGaussianAdam([{"params": [p[n]], "lr": m.lr[n], "name": n} for n in names], lr=0.0, eps=m.eps)
    g = torch.Generator().manual_seed(5)
    o = store_offsets(P, M)
    for _ in range(3):
        m.grad.copy_(torch.randn(m.grad.shape, generator=g) * 1e-2)
        m.gradients_ready()
        feat = m.grad[o["features"]:o["opacity"]].view(P, M, 3)
        grads = {"xyz": m.grad[:3 * P].view(P, 3), "f_dc": feat[:, :1], "f_rest": feat[:, 1:]}
        for n in names:
            p[n].grad = grads[n].contiguous().clone()
        vis = torch.rand(P, generator=g) < 0.5
        m.optimizer_step(visible=vis)
        opt.step(vis, P)
        views = {"p": m._group_views(m.store), "exp_avg": m._group_views(m.exp_avg), "exp_avg_sq": m._group_views(m.exp_avg_sq)}
        for n in names:
            assert torch.equal(p[n].detach(), views["p"][n].reshape(p[n].shape)), n
            for k in ("exp_avg", "exp_avg_sq"):
                assert torch.equal(opt.state[p[n]][k], views[k][n].reshape(p[n].shape)), (n, k)


class SparseReplay:
    """SparseModelOracle (the reference class's training state with a sparse optimizer) driven by the fixture recorded from
    the reference class itself (make_golden_sparse.py): row counts and order, state keys and step counts after every stage,
    parameters and moments after the stages the fixture holds them for."""

    def __init__(self, optimizer_cls, dev="cpu"):
        self.gold = {k: v for k, v in np.load(GOLD).items()}
        self.cls, self.dev = optimizer_cls, dev
        gold = self.gold
        t = lambda k: torch.from_numpy(gold["init" + RAW_KEY[k]]).to(dev)
        opt = {str(k): float(v) for k, v in zip(gold["opt_names"], gold["opt_values"])}
        self.opt = opt
        self.m = SparseModelOracle(t("xyz"), t("f_dc"), t("f_rest"), t("opacity"), t("scaling"), t("rotation"), opt,
                                   float(gold["dens_extent"]), optimizer_cls=optimizer_cls)
        self.it = 0

    def backward(self):
        self.it += 1
        m, gold = self.m, self.gold
        act = m.activated()
        P = act["xyz"].shape[0]
        grads = {n: torch.from_numpy(gold["w_" + n][:P]).to(self.dev) + torch.from_numpy(gold["u_" + n][:P]).to(self.dev) * act[n].detach()
                 for n in ACT}
        m.backward(self.it, grads)

    def step(self, tag):
        self.m.optimizer_step(torch.from_numpy(self.gold[f"{tag}_vis"]).to(self.dev))

    def check(self, tag, param_tol=2e-6, moment_rtol=1e-4):
        m, gold = self.m, self.gold
        mom = m.moments()
        assert m.P == int(gold[f"{tag}_P"]), (tag, m.P)
        for k, grp in enumerate(m.adam.param_groups):
            n = grp["name"]
            assert n == GROUPS[k]
            st = m.adam.state.get(grp["params"][0])
            assert (",".join(sorted(st)) if st is not None else "") == str(gold[f"{tag}_keys"][k]), (tag, n)
            if st is not None:
                assert float(st["step"]) == float(gold[f"{tag}_steps"][k]), (tag, n)
            if tag + RAW_KEY[n] not in gold:
                continue
            ref = torch.from_numpy(gold[tag + RAW_KEY[n]])
            assert tuple(m.p[n].shape) == tuple(ref.shape), (tag, n)
            torch.testing.assert_close(m.p[n].detach().cpu(), ref, rtol=param_tol, atol=param_tol, msg=lambda s: f"{tag} {n}: {s}")
            for kind, atol in (("m", 1e-9), ("v", 1e-13)):
                torch.testing.assert_close(mom[n][kind].cpu(), torch.from_numpy(gold[f"{tag}_{kind}_{n}"]), rtol=moment_rtol, atol=atol,
                                           msg=lambda s: f"{tag} {kind} {n}: {s}")

    def run(self):
        m, gold = self.m, self.gold
        for tag in ("s1", "s2", "s3"):
            self.backward()
            self.step(tag)
            self.check(tag)
        self.backward()
        m.grad_accum = torch.from_numpy(gold["dens_accum"]).to(self.dev)
        m.denom = torch.from_numpy(gold["dens_denom"]).to(self.dev)
        m.max_radii2D = torch.from_numpy(gold["dens_max_radii2D"]).to(self.dev)
        torch.manual_seed(int(gold["dens_seed"]))
        info = m.densify_and_prune(self.opt["densify_grad_threshold"], 0.005, float(gold["dens_extent"]), 20)
        assert info["P"] == int(gold["d_P"]) and info["n_clone"] > 0 and info["n_split"] > 0 and info["n_pruned"] > 0, info
        self.step("d")                                   # every parameter was replaced: a no-op
        self.check("d")
        self.backward()
        self.step("s5")
        self.check("s5")
        self.backward()
        m.reset_opacity()
        self.step("r6")
        self.check("r6")
        self.backward()
        self.step("s7")
        self.check("s7")
        # capture() / restore(): the optimizer's state_dict into a fresh instance over the same parameters
        sd = m.adam.state_dict()
        before = {n: {k: v.clone() for k, v in m.adam.state[m.p[n]].items()} for n in GROUPS}
        m.adam = self.cls([{"params": [m.p[n]], "lr": 0.0, "name": n} for n in GROUPS], lr=0.0, eps=1e-15)
        m.adam.load_state_dict(sd)
        for n in GROUPS:
            st = m.adam.state[m.p[n]]
            assert sorted(st) == sorted(before[n]) and all(torch.equal(st[k].cpu(), before[n][k].cpu()) for k in st), n
        self.check("c")
        self.backward()
        self.step("s8")
        self.check("s8")


def test_sparse_adam_source_replays_reference_class_fixture(on_host):
    from diff_gaussian_rasterization.sparse_adam import SparseGaussianAdam
    SparseReplay(SparseGaussianAdam).run()


def test_oracle_replays_reference_class_fixture():
    SparseReplay(SparseGaussianAdamOracle).run()


@pytest.mark.parametrize("value,expected", [(None, False), ("1", True)])
def test_sparse_adam_export_gate(host_lib, value, expected):
    """SparseGaussianAdam is a package attribute only with GSB_SPARSE_ADAM=1 set at import (it flips separate_sh in the
    reference scripts)."""
    env = {k: v for k, v in os.environ.items() if k != "GSB_SPARSE_ADAM"}
    if value is not None:
        env["GSB_SPARSE_ADAM"] = value
    code = f"import sys; sys.path.insert(0, {PKG!r}); import diff_gaussian_rasterization as d; print(hasattr(d, 'SparseGaussianAdam'))"
    r = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, check=True)
    assert r.stdout.strip() == str(expected)
