"""Growth of the dreamed point cloud on the device (pcd.grow_view) against the host restatement of the reference's
dreaming-loop body (tests/grow_host.py), which tests/test_grow_cpu.py pins to the reference's own digests."""
import numpy as np
import pytest
import torch

import grow_host
import grow_inputs
import pcd_cases
import pcd_host
from luciddreamer_b200 import pcd

pytestmark = pytest.mark.gpu


def same_bits(a, b):
    """Elementwise: the same float bits (signed zeros told apart), or both NaN."""
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    u = np.uint64 if a.dtype == np.float64 else np.uint32
    return (a.view(u) == b.view(u)) | (np.isnan(a) & np.isnan(b))


def perturb(d, rng):
    """new_depth moved by a relative 1e-12, plus 1e-12 of its largest magnitude: the barycentric sums round off at
    that absolute scale, which a relative move alone misses where the corrections cancel to nearly 0."""
    scale = np.abs(d[np.isfinite(d)]).max(initial=0.0)
    return d * (1.0 + 1e-12 * rng.uniform(-1, 1, d.shape)) + 1e-12 * scale * rng.uniform(-1, 1, d.shape)


def grow(inp, **kw):
    return pcd.grow_view(inp["pts"], inp["colors"], inp["R"], inp["T"], inp["K"], inp["mask2"], inp["valid_idx"],
                         inp["coords"], inp["rnd"], inp["image"], inp["depth"], return_details=True, **kw)


def check(inp, out=None, seeds=3):
    """Device against host for one view: border points, count, colours and old points bit-identical; a new
    coordinate may differ only where a 1e-12 perturbation of the host's interpolated correction (`perturb`) changes
    the host's coordinate too, and in views with 1000 or more new points such points are fewer than 1e-3 of them."""
    pts, cols, border, new_depth = grow(inp) if out is None else out
    h_pts, h_cols, h_border, h_depth = grow_host.grow_view_host(**inp)
    n = inp["pts"].shape[1]
    M = h_pts.shape[1] - n
    assert pts.dtype == np.float64 and cols.dtype == np.float32 and pts.shape == h_pts.shape
    np.testing.assert_array_equal(border, h_border)
    assert cols.tobytes() == h_cols.tobytes()
    assert pts[:, :n].tobytes() == np.asarray(inp["pts"], np.float64).tobytes()
    np.testing.assert_allclose(new_depth, h_depth, rtol=1e-12, atol=1e-12, equal_nan=True)
    diff = ~same_bits(pts[:, n:], h_pts[:, n:]).all(0)
    if diff.any():
        unstable = np.zeros(M, bool)
        for s in range(seeds):
            rng = np.random.default_rng(100 + s)
            alt = grow_host.grow_view_host(**inp, perturb=lambda d: perturb(d, rng))
            unstable |= ~same_bits(alt[0][:, n:], h_pts[:, n:]).all(0)
        print(f"{diff.sum()} of {M} new points differ, {unstable.sum()} round-off-sensitive")
        bad = np.where(diff & ~unstable)[0]
        assert not len(bad), (bad[:4], new_depth[bad[:4]], h_depth[bad[:4]], pts[:, n + bad[:4]], h_pts[:, n + bad[:4]])
        if M >= 1000:                                      # the synthetic views below are smaller
            assert diff.sum() < 1e-3 * M
    return pts, cols


def test_golden_cases_match_the_reference_growth():
    for c, inp, _ in grow_inputs.golden_cases():
        pts, cols, border, _ = grow(inp)
        assert len(border) == c["n_border"]
        check(inp, (pts, cols, border, _))


def seeded_case(seed, n, H, W, f32):
    pts, cols = pcd_cases.depth_cloud(seed, H, W, extra=max(n - H * W, 0))
    pts = pts if f32 else pts.astype(np.float64)
    K = pcd_cases.intrinsics(H, W).astype(np.float32)
    R, T = pcd_cases.random_pose(seed)
    _, mask2, valid, coords, rnd = pcd.warp_view(pts, cols, R, T, K, H, W)
    return dict(pts=pts, colors=cols, R=R, T=T, K=K, mask2=mask2, valid_idx=valid, coords=coords, rnd=rnd,
                image=grow_host.stub_image(seed + 1, H, W), depth=grow_host.stub_depth(seed + 2, H, W))


@pytest.mark.parametrize("seed,n,H,W,f32", [(0, 262_144, 96, 128, True), (1, 1_000_000, 192, 256, False),
                                            (2, 2_000_000, 512, 512, False)])
def test_seeded_clouds_match_the_host_restatement(seed, n, H, W, f32):
    inp = seeded_case(seed, n, H, W, f32)
    assert (inp["mask2"] != 1).any() and len(inp["valid_idx"]) > 0
    check(inp)


def test_three_view_dreaming_loop_and_aligning_stage():
    H, W = 96, 128
    K = pcd_cases.intrinsics(H, W).astype(np.float32)
    pts, cols = pcd_cases.depth_cloud(4, H, W)
    for i in (1, 2, 3):
        R, T = pcd_cases.random_pose(10 + i)
        _, mask2, valid, coords, rnd = pcd.warp_view(pts, cols, R, T, K, H, W)
        _, h_mask2, h_valid, _, h_rnd = pcd_host.warp_view_host(pts, cols, R, T, K, H, W)
        np.testing.assert_array_equal(mask2, h_mask2)
        np.testing.assert_array_equal(valid, h_valid)
        np.testing.assert_array_equal(rnd, h_rnd)
        inp = dict(pts=pts, colors=cols, R=R, T=T, K=K, mask2=mask2, valid_idx=valid, coords=coords, rnd=rnd,
                   image=grow_host.stub_image(20 + i, H, W), depth=grow_host.stub_depth(30 + i, H, W))
        pts, cols = check(inp)
        assert pts.dtype == np.float64
    rp = np.concatenate([pcd_cases.rotate360(1), np.concatenate(pcd_cases.random_pose(11), 1)[None]])
    hemi = pcd_cases.hemisphere(2.0)
    frames, mats = pcd.align_frames(pts, cols, rp, hemi, K, H, W)
    ref, _ = pcd_host.align_frames_host(pts, cols, rp, hemi, K, H, W)
    assert len(frames) == len(ref)
    unstable = np.zeros(ref.shape[:3], bool)
    for s in range(3):
        rng = np.random.default_rng(100 + s)
        alt, _ = pcd_host.align_frames_host(pts, cols, rp, hemi, K, H, W,
                                            perturb=lambda c: c * (1.0 + 1e-12 * rng.uniform(-1, 1, c.shape)))
        unstable |= (alt != ref).any(-1)
    diff = (frames != ref).any(-1)
    assert not (diff & ~unstable).any()
    assert unstable.sum() < 1e-3 * unstable.size


def synthetic(seed, H, W, dup=False, corner=False):
    """Warp outputs made up directly: mask2 1 on a random half-plane, valid points scattered over the view with
    their round coordinates, the cloud 2 units along each point's ray."""
    rng = np.random.default_rng(seed)
    K = np.array([[64.0, 0.0, W / 2.0], [0.0, 64.0, H / 2.0], [0.0, 0.0, 1.0]], np.float32)
    yy, xx = np.mgrid[0:H, 0:W]
    mask2 = ((xx - W / 2.0) * rng.uniform(-1, 1) + (yy - H / 2.0) * rng.uniform(-1, 1) >= 0).astype(np.int64)
    nv = max(4, H * W // 2)
    coords = np.stack([rng.uniform(0, W - 1, nv), rng.uniform(0, H - 1, nv)])
    if corner:                                             # a border point exactly on the corner (0, 0)
        mask2[0, 0], mask2[1, 0], mask2[0, 1] = 1, 0, 0
        coords[:, 0] = 0.0
    z = rng.uniform(1.5, 2.5, nv)
    pts = np.stack([(coords[0] - W / 2.0) / 64.0 * z, (coords[1] - H / 2.0) / 64.0 * z, z])
    if corner:
        pts[:, 0] = [-W / 128.0, -H / 128.0, 1.0]          # on the corner's ray at the depth map's depth
    if dup:                                                # every point twice: duplicate border points
        coords, pts = np.concatenate([coords, coords], 1), np.concatenate([pts, pts], 1)
        order = np.argsort(np.concatenate([np.arange(nv), np.arange(nv)]), kind="stable")
        coords, pts = coords[:, order], pts[:, order]
    valid = np.arange(pts.shape[1], dtype=np.int64)
    depth = grow_host.stub_depth(seed, H, W)
    depth[0, 0] = 1.0
    return dict(pts=pts, colors=rng.random((pts.shape[1], 3)).astype(np.float32), R=np.eye(3), T=np.zeros((3, 1)),
                K=K, mask2=mask2, valid_idx=valid, coords=coords, rnd=np.round(coords).astype(np.int32),
                image=grow_host.stub_image(seed, H, W), depth=depth)


def test_duplicate_border_points_and_a_border_point_on_a_corner():
    inp = synthetic(3, 24, 32, dup=True)
    _, _, border, _ = grow(inp)
    assert len(border) > 0 and (inp["coords"][:, border[0::2]] == inp["coords"][:, border[1::2]]).all()
    check(inp)
    inp = synthetic(4, 24, 32, corner=True)
    _, _, border, _ = grow(inp)
    assert border[0] == 0
    check(inp)


@pytest.mark.parametrize("H,W", [(3, 3), (3, 4), (4, 3), (5, 6), (7, 7), (8, 9), (16, 15)])
def test_odd_and_even_sizes(H, W):
    check(synthetic(H * 100 + W, H, W))


def test_deterministic_and_same_bytes_for_tensor_inputs():
    inp = seeded_case(5, 50_000, 96, 128, False)
    a = grow(inp)
    b = grow(inp)
    dev = torch.device("cuda")
    c = pcd.grow_view(torch.from_numpy(inp["pts"]).to(dev), torch.from_numpy(inp["colors"]).to(dev), inp["R"],
                      inp["T"], inp["K"], inp["mask2"], inp["valid_idx"], inp["coords"], inp["rnd"],
                      torch.from_numpy(inp["image"]).to(dev), torch.from_numpy(inp["depth"]).to(dev),
                      return_details=True)
    from PIL import Image
    d = pcd.grow_view(inp["pts"], inp["colors"], inp["R"], inp["T"], inp["K"], inp["mask2"], inp["valid_idx"],
                      inp["coords"], inp["rnd"], Image.fromarray(inp["image"]), inp["depth"], return_details=True)
    for other in (b, c, d):
        for x, y in zip(a, other):
            assert x.dtype == y.dtype and x.tobytes() == y.tobytes()
