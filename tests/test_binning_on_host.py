"""Tile binning (binning.cu tile_scan / emit, radix_sort.cu tile sort) executed on the CPU through tests/host_emul: every view's
point_list and ranges against a numpy stable sort of the (tile, depth rank) pairs, and tile_order against the list lengths.

The instances are taken from the output itself (tile t holds the gaussians point_list[ranges[t].x:ranges[t].y]); what is
checked is how they are laid out: tiles in ascending order, contiguous, each list in depth order (ties by gaussian index,
the stable depth sort's order), empty tiles {0, 0}.  A truncated run (async capacity below the count) must hold exactly the
first `capacity` instances in emission order -- gaussians by depth rank, each one's tiles in ascending id -- sorted by tile."""
import ctypes
import math

import numpy as np
import pytest
import torch

from oracle import torch_oracle as TO


def _u32(ptr, n):
    if n == 0:
        return np.zeros(0, dtype=np.uint32)
    return np.ctypeslib.as_array((ctypes.c_uint32 * n).from_address(ptr)).copy()


def _cams(V, W, H):
    import bench
    return [bench.BenchCamera(W, H, math.radians(60.0), *bench.view_pose(i, 3.0), "cpu") for i in range(V)]


def _settings(dgr, cam, deg):
    return dgr.GaussianRasterizationSettings(cam.image_height, cam.image_width, math.tan(cam.FoVx * 0.5), math.tan(cam.FoVy * 0.5),
                                             torch.zeros(3), 1.0, cam.world_view_transform, cam.full_proj_transform, deg,
                                             cam.camera_center, False, False, False)


def _depth_rank(scene, cam):
    """Position of every gaussian in the depth order (view-space z ascending, ties by index)."""
    p = scene["means3D"].double().numpy()
    z = (np.concatenate([p, np.ones((len(p), 1))], 1) @ cam.world_view_transform.double().numpy())[:, 2]
    order = np.argsort(z, kind="stable")
    zs = z[order]
    assert len(zs) < 2 or np.min(np.diff(zs)) > 1e-6, "depths too close to fix the order in float32"
    rank = np.empty(len(z), dtype=np.int64)
    rank[order] = np.arange(len(z))
    return rank


def _forward(dgr, scene, cams, deg, capacity=None):
    V = len(cams)
    args = (scene["means3D"], scene["shs"][:, :(deg + 1) ** 2].contiguous(), scene["opacities"].reshape(-1), scene["scales"],
            scene["rotations"], [_settings(dgr, c, deg) for c in cams])
    if capacity is None:
        _, radii, _, pack = dgr._forward_batch_impl(*args)
        counts = pack["num_rendered"]
    else:
        ac = torch.zeros(dgr.COUNT_SLOTS, dtype=torch.int64)
        _, radii, _, pack = dgr._forward_batch_impl(*args, async_counts=ac, capacity=capacity)
        counts = [int(c) for c in ac[:V]]
    out = []
    for v in range(V):
        st = pack["states"][v]
        nt = int(st.num_tiles)
        d = counts[v] if capacity is None else min(counts[v], capacity)
        ranges = _u32(st.ranges, 2 * nt).reshape(nt, 2)
        order = _u32(st.tile_order, nt) if st.tile_order else None
        out.append(dict(count=counts[v], point_list=_u32(st.point_list, d), ranges=ranges, tile_order=order))
    return out, radii


def _pairs(view):
    """(tile, gaussian) of every instance, read off the ranges."""
    t = np.concatenate([np.full(int(y - x), i, dtype=np.int64) for i, (x, y) in enumerate(view["ranges"])] + [np.zeros(0, np.int64)])
    g = np.concatenate([view["point_list"][x:y] for x, y in view["ranges"]] + [np.zeros(0, np.uint32)]).astype(np.int64)
    return t, g


def _expected(tile, gauss, rank, num_tiles):
    o = np.lexsort((rank[gauss], tile))          # stable sort on (tile, depth rank)
    pl = gauss[o].astype(np.uint32)
    ts = tile[o]
    ranges = np.zeros((num_tiles, 2), dtype=np.uint32)
    if len(ts):
        u, first = np.unique(ts, return_index=True)
        last = np.r_[first[1:], len(ts)]
        ranges[u, 0], ranges[u, 1] = first, last
    return pl, ranges


def _check_view(view, rank):
    nt = len(view["ranges"])
    tile, gauss = _pairs(view)
    assert len(tile) == len(view["point_list"]) == view["count"], "ranges do not cover the list"
    pl, ranges = _expected(tile, gauss, rank, nt)
    assert np.array_equal(view["ranges"], ranges)
    assert np.array_equal(view["point_list"], pl)
    if view["tile_order"] is not None:
        order = view["tile_order"]
        assert np.array_equal(np.sort(order), np.arange(nt)), "tile_order is not a permutation"
        lens = (view["ranges"][:, 1] - view["ranges"][:, 0]).astype(np.int64)[order]
        bins = np.where(lens < 2048, lens >> 4, np.minimum(255, 128 + ((lens - 2048) >> 7)))   # render.cu tile_order_kernel
        assert np.all(np.diff(bins) <= 0), "tile_order not in descending bin order"


def _run(dgr, scene, V, W, H, deg=1):
    cams = _cams(V, W, H)
    views, radii = _forward(dgr, scene, cams, deg)
    for v, view in enumerate(views):
        rank = _depth_rank(scene, cams[v]) if view["count"] else np.zeros(len(radii[v]), dtype=np.int64)
        assert set(view["point_list"].tolist()) <= set(np.nonzero(radii[v].numpy() > 0)[0].tolist())
        _check_view(view, rank)
    return cams, views


@pytest.mark.parametrize("V", [1, 5, 16])
def test_views(on_host, V):
    scene = TO.make_scene(300, seed=60 + V, log_scale_mean=-2.6)
    _, views = _run(on_host, scene, V, 64, 48)
    assert all(v["count"] > 0 for v in views)


def test_fully_culled(on_host):
    scene = TO.make_scene(80, seed=3, sh_coeffs=4)
    scene["means3D"] = scene["means3D"] * 0.01 + 100.0       # far behind every camera's near plane or outside the frustum
    _, views = _run(on_host, scene, 2, 48, 32)
    assert all(v["count"] == 0 and not v["ranges"].any() for v in views)


def test_image_smaller_than_a_tile(on_host):
    scene = TO.make_scene(120, seed=4, log_scale_mean=-2.4)
    _, views = _run(on_host, scene, 3, 12, 10)
    assert len(views[0]["ranges"]) == 1


def test_many_tile_gaussians(on_host):
    """Gaussians covering tens of tiles: one warp's instances span several staging windows of emit."""
    scene = TO.make_scene(150, seed=5, log_scale_mean=-0.9, log_scale_std=0.6)
    _, views = _run(on_host, scene, 2, 160, 128)
    tile, gauss = _pairs(views[0])
    assert len(tile) > 8 * len(np.unique(gauss))          # 32 gaussians of a warp: more than one 256-slot window


def test_culling_off(on_host):
    dgr = on_host
    scene = TO.make_scene(200, seed=6, log_scale_mean=-2.0)
    dgr.set_option("cull", 0)
    try:
        _, off = _run(dgr, scene, 2, 80, 48)
    finally:
        dgr.set_option("cull", 1)
    _, on = _run(dgr, scene, 2, 80, 48)
    assert off[0]["count"] > on[0]["count"]


@pytest.mark.parametrize("frac", [0.0, 0.37, 0.999])
def test_async_capacity_truncation(on_host, frac):
    """Capacity below the count: the first `capacity` instances in emission order, sorted by tile; counts stay exact."""
    dgr = on_host
    scene = TO.make_scene(250, seed=7, log_scale_mean=-2.2)
    cams = _cams(2, 64, 48)
    full, _ = _forward(dgr, scene, cams, 1)
    cap = max(1, int(frac * min(v["count"] for v in full)))
    cut, _ = _forward(dgr, scene, cams, 1, capacity=cap)
    for v in range(2):
        rank = _depth_rank(scene, cams[v])
        assert cut[v]["count"] == full[v]["count"]
        tile, gauss = _pairs(full[v])
        emitted = np.lexsort((tile, rank[gauss]))[:cap]
        pl, ranges = _expected(tile[emitted], gauss[emitted], rank, len(full[v]["ranges"]))
        assert np.array_equal(cut[v]["point_list"], pl)
        assert np.array_equal(cut[v]["ranges"], ranges)
