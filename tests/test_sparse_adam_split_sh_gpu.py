"""Split SH input and SparseGaussianAdam on the H100: the CPU file's checks (tests/test_sparse_adam_split_sh_on_host.py) at
GPU sizes.  The forward pass is bit-equal between the split and the joint input; gradients are compared at the blend
kernel's atomics bar (1e-4 x max, as test_ab_options_keep_results), because its float atomics reorder sums."""
import math

import pytest
import torch

import test_sparse_adam_split_sh_on_host as H
from oracle.model_oracle import GROUPS
from sparse_adam_oracle import SparseGaussianAdamOracle

pytestmark = pytest.mark.gpu
BAR = 1e-4


@pytest.fixture(scope="module")
def dgr():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    import diff_gaussian_rasterization as d
    return d


def _compare(j, s, what):
    for k in ("color", "radii", "invdepth"):
        assert torch.equal(j[k], s[k]), f"{k}: {what}"
    for k, v in j["grads"].items():
        w = s["grads"][k]
        assert not torch.isnan(v).any() and not torch.isnan(w).any(), f"grad {k} not written: {what}"
        assert float((v - w).abs().max()) <= BAR * float(v.abs().max()), f"grad {k}: {what}"


@pytest.mark.parametrize("deg,M", [(0, 1), (0, 16), (1, 4), (2, 9), (3, 16)])
@pytest.mark.parametrize("aa", [False, True])
def test_split_sh_matches_joint_20k(dgr, deg, M, aa):
    for tma in (0, 1):
        dgr.set_option("pre_tma", tma)
        try:
            for acc in (False, True):
                j, s = H.raster_split_vs_joint(dgr, 20000, M, deg, aa, 250, 141, acc, seed=deg * 7 + M, dev="cuda",
                                               log_scale_mean=-4.0)
                assert int((j["radii"] > 0).sum()) > 1000
                _compare(j, s, f"deg {deg} M {M} aa {aa} pre_tma {tma} accumulate {acc}")
        finally:
            dgr.set_option("pre_tma", 1)


@pytest.mark.parametrize("tma", [0, 1])
def test_split_sh_matches_joint_1m_1080p(dgr, tma):
    """configs[2]: 1 M gaussians, 1920 x 1080, SH degree 3."""
    dgr.set_option("pre_tma", tma)
    try:
        for acc in (False, True):
            j, s = H.raster_split_vs_joint(dgr, 1_000_000, 16, 3, False, 1920, 1080, acc, seed=3, dev="cuda", log_scale_mean=-5.3)
            _compare(j, s, f"1M pre_tma {tma} accumulate {acc}")
    finally:
        dgr.set_option("pre_tma", 1)


def test_render_separate_sh_matches_joint(dgr):
    import bench
    from gaussian_renderer import render
    from oracle import torch_oracle as TO
    scene = TO.make_scene(50000, seed=8, log_scale_mean=-4.0)
    cam = bench.BenchCamera(640, 360, math.radians(60.0), *bench.view_pose(0, 3.0), "cuda")
    w = torch.linspace(-1, 1, 3 * 360 * 640, device="cuda").view(3, 360, 640)
    out = {}
    for sep in (False, True):
        pc = H.RefShaped(scene, "cuda")
        pkg = render(cam, pc, bench.Pipe(), torch.tensor([0.1, 0.2, 0.3], device="cuda"), separate_sh=sep)
        (pkg["render"] * w).sum().backward()
        out[sep] = (pkg["render"].detach(), pkg["radii"], {n: p.grad.clone() for n, p in pc.named().items()})
    assert torch.equal(out[False][0], out[True][0]) and torch.equal(out[False][1], out[True][1])
    for n, ref in out[False][2].items():
        assert float((ref - out[True][2][n]).abs().max()) <= BAR * float(ref.abs().max()), n


@pytest.mark.parametrize("P", [1, 33, 2011])
def test_sparse_adam_matches_oracle(dgr, P):
    dgr.reset_launch_count()
    H.run_sparse_adam_against_oracle(P, "cuda")
    assert dgr.launch_count() == 3


def test_sparse_adam_1m_six_groups_one_launch(dgr):
    from diff_gaussian_rasterization.sparse_adam import SparseGaussianAdam
    P = 1_000_000
    init = H.make_groups(P, 2, "cuda")
    p = {n: torch.nn.Parameter(init[n].clone()) for n in GROUPS}
    opt = SparseGaussianAdam([{"params": [p[n]], "lr": H.LRS[n], "name": n} for n in GROUPS], lr=0.0, eps=1e-15)
    g = torch.Generator(device="cuda").manual_seed(3)
    for n in GROUPS:
        p[n].grad = torch.randn(p[n].shape, generator=g, device="cuda") * 1e-2
    vis = torch.rand(P, generator=g, device="cuda") < 0.5
    dgr.reset_launch_count()
    opt.step(vis, P)
    assert dgr.launch_count() == 1
    ref = {n: torch.nn.Parameter(init[n].cpu().clone()) for n in GROUPS}
    ro = SparseGaussianAdamOracle([{"params": [ref[n]], "lr": H.LRS[n], "name": n} for n in GROUPS], lr=0.0, eps=1e-15)
    for n in GROUPS:
        ref[n].grad = p[n].grad.cpu()
    ro.step(vis.cpu(), P)
    for n in GROUPS:
        got = p[n].detach().cpu()
        assert torch.equal(got[~vis.cpu()], init[n].cpu()[~vis.cpu()]), n
        torch.testing.assert_close(got, ref[n].detach(), rtol=0, atol=2e-6)
        for k, atol in (("exp_avg", 1e-9), ("exp_avg_sq", 1e-13)):
            torch.testing.assert_close(opt.state[p[n]][k].cpu(), ro.state[ref[n]][k], rtol=1e-4, atol=atol)


def test_training_loop_render_split_sh_with_sparse_adam(dgr):
    """15 iterations of render(separate_sh=True) -> L1 -> backward -> SparseGaussianAdam.step(radii > 0) on a reference-shaped
    model; every step is repeated by the oracle optimizer on a copy of the parameters and moments with the same gradients
    and mask, and the two results must agree (parameters 2e-6, moments 1e-4 rel).  Lockstep, not two free-running loops:
    without bias correction the first visible step of a row moves it by ~3 lr whatever the gradient's size, so a gradient
    entry near zero, whose sign the blend kernel's float atomics decide differently from run to run, sends two otherwise
    identical loops apart by O(lr) in a few entries (1.4e-4 relative L2 on f_dc after 15 steps, measured on an H100)."""
    import bench
    from diff_gaussian_rasterization.sparse_adam import SparseGaussianAdam
    from gaussian_renderer import render
    from oracle import torch_oracle as TO
    scene = TO.make_scene(20000, seed=12, log_scale_mean=-4.0)
    W_, H_ = 320, 180
    cams = [bench.BenchCamera(W_, H_, math.radians(60.0), *bench.view_pose(i, 3.0), "cuda") for i in range(4)]
    gts = [torch.rand(3, H_, W_, generator=torch.Generator().manual_seed(i)).cuda() for i in range(4)]
    bg = torch.zeros(3, device="cuda")
    pc = H.RefShaped(scene, "cuda")
    named = pc.named()
    opt = SparseGaussianAdam([{"params": [t], "lr": H.LRS[n], "name": n} for n, t in named.items()], lr=0.0, eps=1e-15)
    start = {n: t.detach().clone() for n, t in named.items()}
    for it in range(15):
        pkg = render(cams[it % 4], pc, bench.Pipe(), bg, separate_sh=True)
        (pkg["render"] - gts[it % 4]).abs().mean().backward()
        vis = pkg["radii"] > 0
        assert 0 < int(vis.sum()) < vis.numel()
        shadow = {n: torch.nn.Parameter(t.detach().clone()) for n, t in named.items()}
        for n, t in named.items():
            assert t.grad is not None and t.grad.shape == t.shape, n
            shadow[n].grad = t.grad.clone()
        so = SparseGaussianAdamOracle([{"params": [shadow[n]], "lr": H.LRS[n], "name": n} for n in named], lr=0.0, eps=1e-15)
        for n, t in named.items():
            if len(opt.state[t]):
                so.state[shadow[n]] = {k: v.clone() for k, v in opt.state[t].items()}
        opt.step(vis, vis.shape[0])
        so.step(vis, vis.shape[0])
        opt.zero_grad(set_to_none=True)
        for n, t in named.items():
            torch.testing.assert_close(t.detach(), shadow[n].detach(), rtol=0, atol=2e-6, msg=lambda m: f"step {it} {n}: {m}")
            for k, atol in (("exp_avg", 1e-9), ("exp_avg_sq", 1e-13)):
                torch.testing.assert_close(opt.state[t][k], so.state[shadow[n]][k], rtol=1e-4, atol=atol,
                                           msg=lambda m: f"step {it} {n} {k}: {m}")
    for n, t in named.items():
        assert not torch.equal(t.detach(), start[n]), n
