"""Tile binning at the bench size on the GPU (1 M gaussians, 1080p, SH 3, 8 views): every view's point_list and ranges against a
torch.sort(stable=True) of the (tile, depth) pairs read off the ranges, and the sync and async batch entry points (same kernels,
one reading the counts back, one not) bit-equal in images, n_contrib and final_T."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

V, W, H, P, DEG = 8, 1920, 1080, 1_000_000, 3


@pytest.fixture(scope="module")
def setup():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    import bench
    import diff_gaussian_rasterization as dgr
    from gaussian_renderer.synthetic import make_scene
    dev = torch.device("cuda:0")
    scene = {k: v.to(dev) for k, v in make_scene(P, seed=0, log_scale_mean=bench.LOG_SCALE_MEAN).items()}
    cams = [bench.BenchCamera(W, H, math.radians(60.0), *bench.view_pose(i, 3.0), dev) for i in range(V)]
    rs = [dgr.GaussianRasterizationSettings(H, W, math.tan(c.FoVx * 0.5), math.tan(c.FoVy * 0.5), torch.zeros(3, device=dev), 1.0,
                                            c.world_view_transform, c.full_proj_transform, DEG, c.camera_center, False, False, False)
          for c in cams]
    args = (scene["means3D"], scene["shs"][:, :(DEG + 1) ** 2].contiguous(), scene["opacities"].reshape(-1).contiguous(),
            scene["scales"], scene["rotations"], rs)
    return dgr, scene, cams, args


def _words(buf, ptr, n):
    off = (ptr - buf.data_ptr()) // 4
    return buf.view(torch.int32)[off:off + n]


def test_lists_are_the_stable_tile_sort_of_depth_ordered_instances(setup):
    dgr, scene, cams, args = setup
    _, radii, _, pack = dgr._forward_batch_impl(*args)
    for v in range(V):
        st = pack["states"][v]
        nt, D = int(st.num_tiles), pack["num_rendered"][v]
        pl = _words(pack["binning"], st.point_list, D).long()
        ranges = _words(pack["binning"], st.ranges, 2 * nt).view(nt, 2).long()
        assert D > 1_000_000
        lens = ranges[:, 1] - ranges[:, 0]
        assert int(lens.sum()) == D and bool((lens >= 0).all())
        assert bool((ranges[lens == 0] == 0).all()), "empty tiles must read {0, 0}"
        nz = lens > 0
        assert bool((ranges[nz, 0] == (torch.cumsum(lens, 0) - lens)[nz]).all()), "ranges not contiguous in tile order"
        assert bool((radii[v][pl] > 0).all())
        tile = torch.repeat_interleave(torch.arange(nt, device=pl.device), lens)
        # expected: the pairs sorted stably on depth, then stably on tile
        wv = cams[v].world_view_transform.double()
        z = scene["means3D"].double() @ wv[:3, 2] + wv[3, 2]
        o1 = torch.sort(z[pl], stable=True).indices
        o2 = torch.sort(tile[o1], stable=True).indices
        expected = pl[o1][o2]
        # the kernels order by the float32 depth (ties by index): neighbours within a few ulp may come in either order
        i = torch.nonzero(expected != pl).flatten()
        assert i.numel() < D // 1000
        assert bool((torch.abs(z[expected[i]] - z[pl[i]]) <= 1e-6 * z[pl[i]].abs()).all()), "list not in depth order"


def test_sync_and_async_batch_are_bit_equal(setup):
    dgr, scene, cams, args = setup
    color_s, radii_s, invd_s, pack_s = dgr._forward_batch_impl(*args)
    counts = torch.zeros(dgr.COUNT_SLOTS, dtype=torch.int64, device=color_s.device)
    cap = dgr.capacity_for(max(pack_s["num_rendered"]))
    color_a, radii_a, invd_a, pack_a = dgr._forward_batch_impl(*args, async_counts=counts, capacity=cap)
    torch.cuda.synchronize()
    assert counts[:V].tolist() == pack_s["num_rendered"]
    assert torch.equal(color_s, color_a) and torch.equal(invd_s, invd_a) and torch.equal(radii_s, radii_a)
    for v in range(V):
        ss, sa = pack_s["states"][v], pack_a["states"][v]
        D, nt = pack_s["num_rendered"][v], int(ss.num_tiles)
        assert torch.equal(_words(pack_s["binning"], ss.point_list, D), _words(pack_a["binning"], sa.point_list, D))
        assert torch.equal(_words(pack_s["binning"], ss.ranges, 2 * nt), _words(pack_a["binning"], sa.ranges, 2 * nt))
        for f in ("final_T", "n_contrib"):
            assert torch.equal(_words(pack_s["image"], getattr(ss, f), H * W), _words(pack_a["image"], getattr(sa, f), H * W)), f
