"""GaussianModel.prune_points against the reference class: tests/golden/reference_prune.npz (tests/golden/make_golden_prune.py,
the reference's own scene/gaussian_model.py on the CPU) replayed on the store, run from the kernel SOURCES on the CPU
(tests/host_emul).  Both optimizer modes; train.py's order (backward, prune, a skipped optimizer.step()); the edge masks none,
all, first row and last row.  Bars: parameters 2e-6, moments 1e-4 relative, step counts and densification tensors exact."""
import os
from types import SimpleNamespace

import numpy as np
import pytest
import torch

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_prune.npz")
GROUPS = ("xyz", "f_dc", "f_rest", "opacity", "scaling", "rotation")
RAW_KEY = {"xyz": "_xyz", "f_dc": "_features_dc", "f_rest": "_features_rest", "opacity": "_opacity", "scaling": "_scaling",
           "rotation": "_rotation"}
ACT = ("xyz", "features", "opacity", "scaling", "rotation")
MODES = {"default": "a_", "sparse_adam": "s_"}


@pytest.fixture(scope="module")
def gold():
    return {k: v for k, v in np.load(GOLD).items()}


class Replay:
    def __init__(self, gold, mode):
        from gaussian_store import GaussianModel
        self.g, self.mode, self.pre = gold, mode, MODES[mode]
        t = lambda k: torch.from_numpy(gold[self.pre + "init" + RAW_KEY[k]])
        opt = {k[4:]: float(v) for k, v in gold.items() if k.startswith("opt_")}
        self.m = GaussianModel(3, mode).create_from_tensors(t("xyz"), t("f_dc"), t("f_rest"), t("scaling"), t("rotation"),
                                                            t("opacity"), 4.0)
        self.m.training_setup(SimpleNamespace(**opt))
        self.m.active_sh_degree = 3

    def backward(self, it):
        m = self.m
        m.update_learning_rate(it)
        act = {"xyz": m.get_xyz, "features": m.get_features, "opacity": m.get_opacity, "scaling": m.get_scaling,
               "rotation": m.get_rotation}
        P = m.P
        for n in ACT:
            w = torch.from_numpy(self.g[self.pre + "w_" + n][:P])
            u = torch.from_numpy(self.g[self.pre + "u_" + n][:P])
            act[n].grad.copy_((w + u * act[n].detach()).view_as(act[n]))
        m.gradients_ready()

    def step(self, tag):
        if self.mode == "sparse_adam":
            self.m.optimizer_step(torch.from_numpy(self.g[f"{self.pre}{tag}_vis"]))
        else:
            self.m.optimizer_step()

    def prune(self, tag, mask_key=None):
        m, g, pre = self.m, self.g, self.pre
        m.xyz_gradient_accum = torch.from_numpy(g[f"{pre}{tag}_in_accum"]).clone()
        m.denom = torch.from_numpy(g[f"{pre}{tag}_in_denom"]).clone()
        m.max_radii2D = torch.from_numpy(g[f"{pre}{tag}_in_max_radii2D"]).clone()
        steps = dict(m.group_steps)
        P_new = m.prune_points(torch.from_numpy(g[f"{pre}{mask_key or tag}_mask"]))
        assert P_new == m.P and m.group_steps == steps and m._skip_next == set(GROUPS)
        assert float(m.grad.abs().sum()) == 0.0

    def check(self, tag):
        from gaussian_store import store_offsets
        m, g, t = self.m, self.g, self.pre + tag
        assert m.P == int(g[t + "_P"]), (tag, m.P)
        raw = m._group_views(m.store)
        for n in GROUPS:
            ref = torch.from_numpy(g[t + RAW_KEY[n]])
            assert tuple(raw[n].shape) == tuple(ref.shape), (tag, n)
            torch.testing.assert_close(raw[n], ref, rtol=2e-6, atol=2e-6, msg=lambda s: f"{tag} {n}: {s}")
        for kind, buf in (("m", m.exp_avg), ("v", m.exp_avg_sq)):
            got = m._group_views(buf)
            for n in GROUPS:
                torch.testing.assert_close(got[n], torch.from_numpy(g[f"{t}_{kind}_{n}"]), rtol=1e-4,
                                           atol=1e-9 if kind == "m" else 1e-13, msg=lambda s: f"{tag} {kind} {n}: {s}")
        if self.mode == "default":        # the sparse optimizer never advances its step (tests/sparse_adam_oracle.py)
            for n in GROUPS:
                assert m.group_steps[n] == int(g[f"{t}_step_{n}"]), (tag, n, m.group_steps)
        for name, got in (("accum", m.xyz_gradient_accum), ("denom", m.denom), ("max_radii2D", m.max_radii2D)):
            ref = torch.from_numpy(g[f"{t}_{name}"])
            assert tuple(got.shape) == tuple(ref.shape) and torch.equal(got, ref), (tag, name)
        assert store_offsets(m.P, 16)["total"] == m.store.numel() == m.grad.numel() == m.exp_avg.numel()
        assert m.act.numel() == 8 * m.P


def _to_s5(gold, mode):
    r = Replay(gold, mode)
    for it in (1, 2):
        r.backward(it)
        r.step(f"s{it}")
    r.backward(3)
    r.prune("p1")
    r.step("p1")                        # skipped: every parameter was just replaced
    r.check("p1")
    r.backward(4)
    r.step("s4")
    r.check("s4")
    r.prune("p2")
    r.check("p2")
    r.backward(5)
    r.step("s5")
    r.check("s5")
    return r


@pytest.mark.parametrize("mode", list(MODES))
def test_prune_points_replays_the_reference(on_host, gold, mode):
    _to_s5(gold, mode)


@pytest.mark.parametrize("edge", ["none", "all", "first", "last"])
@pytest.mark.parametrize("mode", list(MODES))
def test_prune_points_edge_masks(on_host, gold, mode, edge):
    r = _to_s5(gold, mode)
    r.prune("e", mask_key=f"e_{edge}")
    r.check(f"e_{edge}")
    if edge == "all":
        assert r.m.P == 0 and r.m.store.numel() == 0
    r.m.optimizer_step()                # skipped, also on an empty store
    assert r.m._skip_next == set()


def test_prune_points_argument_errors(on_host, gold):
    r = Replay(gold, "default")
    for bad in (torch.zeros(39, dtype=torch.bool), torch.zeros(40, dtype=torch.uint8), torch.zeros(40, 1, dtype=torch.bool),
                torch.zeros(40, dtype=torch.bool, device="meta")):
        with pytest.raises(ValueError):
            r.m.prune_points(bad)
    assert r.m.P == 40
