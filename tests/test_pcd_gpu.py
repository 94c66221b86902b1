"""Point-cloud warp on the device (luciddreamer_b200.pcd) against the host restatement of generate_pcd's loops
and the digests of the reference's own loops."""
import ctypes as C
import hashlib
import json
import os

import numpy as np
import pytest
import torch

import pcd_cases
import pcd_host
from luciddreamer_b200 import pcd

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = json.load(open(os.path.join(ROOT, "tests", "golden", "pcd_golden.json")))


def digest(a):
    a = np.ascontiguousarray(a)
    return {"shape": list(a.shape), "dtype": str(a.dtype), "sha256": hashlib.sha256(a.tobytes()).hexdigest()}


def golden_inputs():
    g = GOLDEN
    pts, cols = pcd_cases.depth_cloud(g["cloud"]["seed"], g["H"], g["W"], extra=g["cloud"]["extra"])
    return pts, cols, np.array(g["K"]), g["H"], g["W"]


def check_view(pts, cols, R, T, K, H, W):
    img, mask, valid, coords, rnd = pcd.warp_view(pts, cols, R, T, K, H, W)
    h_img, h_mask, h_valid, h_coords, h_rnd = pcd_host.warp_view_host(pts, cols, R, T, K, H, W)
    assert mask.dtype == h_mask.dtype and valid.dtype == h_valid.dtype and rnd.dtype == h_rnd.dtype
    np.testing.assert_array_equal(valid, h_valid)
    np.testing.assert_array_equal(rnd, h_rnd)
    np.testing.assert_allclose(coords, h_coords, rtol=1e-15, atol=0)
    np.testing.assert_array_equal(mask, h_mask)
    assert np.abs(img - h_img).max(initial=0.0) <= 1e-12
    return img, mask


def roundoff_sensitive(pts, cols, rp, hemi, K, H, W, seeds=3):
    """Pixels of the host frames that change when the projected coordinates move by a relative 1e-12."""
    ref, _ = pcd_host.align_frames_host(pts, cols, rp, hemi, K, H, W)
    unstable = np.zeros(ref.shape[:3], bool)
    for s in range(seeds):
        rng = np.random.default_rng(100 + s)
        alt, _ = pcd_host.align_frames_host(pts, cols, rp, hemi, K, H, W,
                                            perturb=lambda c: c * (1.0 + 1e-12 * rng.uniform(-1, 1, c.shape)))
        unstable |= (alt != ref).any(-1)
    return ref, unstable


def test_aligning_stage_matches_the_reference_digests():
    """Frames equal the reference's bytes, except in views whose points sit on the pixel lattice (the identity
    view of the depth-map cloud), where Qhull's choice between cocircular diagonals is arbitrary: there the
    differences must lie where 1e-12 of round-off changes the reference too."""
    pts, cols, K, H, W = golden_inputs()
    rp, hemi = np.array(GOLDEN["render_poses"]), np.array(GOLDEN["internal_poses"])
    frames, mats = pcd.align_frames(pts, cols, rp, hemi, K, H, W)
    assert len(frames) == len(GOLDEN["align_frames"])
    ref, unstable = roundoff_sensitive(pts, cols, rp, hemi, K, H, W)
    exact = 0
    for k, (f, m, g) in enumerate(zip(frames, mats, GOLDEN["align_frames"])):
        assert digest(ref[k]) == g["image"]
        assert m.tolist() == g["transform_matrix"]
        if digest(f) == g["image"]:
            exact += 1
            continue
        diff = (f != ref[k]).any(-1)
        print(f"frame {k}: {diff.sum()} differing pixels, {unstable[k].sum()} round-off-sensitive")
        assert not (diff & ~unstable[k]).any()
        assert unstable[k].sum() < 1e-3 * H * W
    print(f"{exact} of {len(frames)} frames byte-identical to the reference")


def test_dreaming_warp_matches_the_reference():
    pts, cols, K, H, W = golden_inputs()
    P = np.array(GOLDEN["dream_poses"])
    for g in GOLDEN["dream"]:
        img, mask = check_view(pts, cols, P[g["pose"], :3, :3], P[g["pose"], :3, 3:4], K, H, W)
        assert digest(mask) == g["mask2"]


@pytest.mark.parametrize("seed,n,H,W", [(0, 20_000, 96, 128), (1, 262_144, 256, 256), (2, 1_000_000, 512, 512)])
def test_generic_clouds_match_the_host_restatement(seed, n, H, W):
    pts, cols = pcd_cases.random_cloud(seed, n, H, W)
    K = pcd_cases.intrinsics(H, W)
    R, T = pcd_cases.random_pose(seed)
    check_view(pts, cols, R, T, K, H, W)
    internal = pcd_cases.hemisphere(2.0)[:2] if n > 500_000 else pcd_cases.hemisphere(2.0)   # scipy: ~12 s a view
    rp = np.concatenate([np.concatenate([R, T], 1)[None], pcd_cases.rotate360(1)])
    frames, mats = pcd.align_frames(pts, cols, rp, internal, K, H, W)
    h_frames, h_mats = pcd_host.align_frames_host(pts, cols, rp, internal, K, H, W)
    np.testing.assert_array_equal(frames, h_frames)
    assert [m.tolist() for m in mats] == [m.tolist() for m in h_mats]


def test_luciddreamer_shaped_identity_view_differs_only_where_round_off_decides():
    H, W = 96, 128
    pts, cols = pcd_cases.depth_cloud(3, H, W)
    K = pcd_cases.intrinsics(H, W)
    hemi = pcd_cases.hemisphere(2.0)
    rp = pcd_cases.rotate360(1)
    frames, _ = pcd.align_frames(pts, cols, rp, hemi[2:3], K, H, W)        # hemisphere view 2 is the identity
    ref, _ = pcd_host.align_frames_host(pts, cols, rp, hemi[2:3], K, H, W)
    _, mask = check_view_masks(pts, cols, K, H, W)
    unstable = np.zeros((H, W), bool)
    for s in range(3):
        rng = np.random.default_rng(100 + s)
        pert = lambda c: c * (1.0 + 1e-12 * rng.uniform(-1, 1, c.shape))
        alt, _ = pcd_host.align_frames_host(pts, cols, rp, hemi[2:3], K, H, W, perturb=pert)
        unstable |= (alt[0] != ref[0]).any(-1)
    diff = (frames[0] != ref[0]).any(-1)
    print(f"identity view: {diff.sum()} device/host differences, {unstable.sum()} round-off-sensitive pixels of "
          f"{mask.sum()} in the mask")
    assert not (diff & ~unstable).any()
    assert unstable.sum() < 1e-3 * mask.sum()


def check_view_masks(pts, cols, K, H, W):
    img, mask, *_ = pcd.warp_view(pts, cols, np.eye(3), np.zeros((3, 1)), K, H, W)
    h_img, h_mask, *_ = pcd_host.warp_view_host(pts, cols, np.eye(3), np.zeros((3, 1)), K, H, W)
    np.testing.assert_array_equal(mask, h_mask)
    return img, mask


def test_run_to_run_and_graph_replay_are_identical():
    pts, cols, K, H, W = golden_inputs()
    rp, hemi = np.array(GOLDEN["render_poses"]), np.array(GOLDEN["internal_poses"])
    a, _ = pcd.align_frames(pts, cols, rp, hemi, K, H, W)
    b, _ = pcd.align_frames(torch.from_numpy(pts).cuda(), torch.from_numpy(cols).cuda(), rp, hemi, K, H, W)
    np.testing.assert_array_equal(a, b)
    # the library call captured into a CUDA graph and replayed
    dev = torch.device("cuda")
    L = pcd.lib()
    p = torch.from_numpy(pts).to(dev, torch.float64)
    c = torch.from_numpy(cols).to(dev)
    views = pcd.compose_poses(rp, hemi)
    poses = np.ascontiguousarray(np.stack([pcd._pose12(R, T) for R, T, _ in views]))
    Kc = np.ascontiguousarray(K, np.float64)
    nb = C.c_uint64()
    assert L.gspcd_scratch_bytes(p.shape[1], H, W, C.byref(nb)) == 0
    scratch = torch.empty(nb.value, dtype=torch.uint8, device=dev)
    frames = torch.zeros((len(views), H, W, 3), dtype=torch.uint8, device=dev)
    small = torch.zeros(len(views) + 1, dtype=torch.int32, device=dev)
    s = torch.cuda.Stream()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        rc = L.gspcd_align(p.data_ptr(), c.data_ptr(), p.shape[1], poses.ctypes.data, Kc.ctypes.data, len(views), H,
                           W, frames.data_ptr(), small.data_ptr(), small.data_ptr() + 4 * len(views),
                           scratch.data_ptr(), nb.value, C.c_void_p(s.cuda_stream))
    assert rc == 0
    frames.zero_()
    g.replay()
    torch.cuda.synchronize()
    keep = [k for k in range(len(views)) if small[k].item() > 0]
    assert small[-1].item() == 0
    np.testing.assert_array_equal(frames[keep].cpu().numpy(), a)


def test_colours_must_be_float32():
    pts, cols = pcd_cases.random_cloud(0, 100, 24, 32)
    with pytest.raises(TypeError):
        pcd.warp_view(pts, cols.astype(np.float64), np.eye(3), np.zeros((3, 1)), pcd_cases.intrinsics(24, 32), 24, 32)


def test_empty_duplicate_and_border_points():
    H, W = 24, 32
    K = pcd_cases.intrinsics(H, W)
    R, T = np.eye(3), np.zeros((3, 1))
    img, mask, valid, coords, rnd = pcd.warp_view(np.zeros((3, 0)), np.zeros((0, 3), np.float32), R, T, K, H, W)
    assert not img.any() and not mask.any() and valid.size == 0
    frames, mats = pcd.align_frames(np.zeros((3, 0)), np.zeros((0, 3), np.float32), pcd_cases.rotate360(1),
                                    pcd_cases.hemisphere(1.0), K, H, W)
    assert frames.shape == (0, H, W, 3) and mats == []
    # points exactly on the W-1 / H-1 borders, and every point twice with the same colour
    rng = np.random.default_rng(5)
    u = np.concatenate([rng.uniform(0, W - 1, 300), np.full(20, W - 1.0), rng.uniform(0, W - 1, 20)])
    v = np.concatenate([rng.uniform(0, H - 1, 300), rng.uniform(0, H - 1, 20), np.full(20, H - 1.0)])
    z = np.full(u.shape, 2.0)
    pts = np.stack([(u - K[0, 2]) / K[0, 0] * z, (v - K[1, 2]) / K[1, 1] * z, z])
    cols = rng.random((len(u), 3)).astype(np.float32)
    pts2, cols2 = np.concatenate([pts, pts], 1), np.concatenate([cols, cols])
    check_view(pts, cols, R, T, K, H, W)
    check_view(pts2, cols2, R, T, K, H, W)


@pytest.mark.parametrize("H,W", [(4, 5), (6, 4), (9, 7), (12, 10)])
def test_filters_at_sizes_smaller_than_the_window(H, W):
    pts, cols = pcd_cases.random_cloud(11, 200, H, W)
    check_view(pts, cols, np.eye(3), np.zeros((3, 1)), pcd_cases.intrinsics(H, W), H, W)


def test_too_few_or_collinear_points_interpolate_to_the_fill_value():
    """Where griddata raises QhullError (the reference aborts), the device writes 0 and the masks still apply."""
    H, W = 24, 32
    K = pcd_cases.intrinsics(H, W)
    for u, v in (([10.3], [7.7]), ([10.3, 12.1], [7.7, 8.2]), ([4.0, 8.0, 12.0, 16.0], [3.0, 6.0, 9.0, 12.0])):
        u, v = np.array(u), np.array(v)
        z = np.full(u.shape, 2.0)
        pts = np.stack([(u - K[0, 2]) / K[0, 0] * z, (v - K[1, 2]) / K[1, 1] * z, z])
        cols = np.full((len(u), 3), 0.5, np.float32)
        img, mask, valid, *_ = pcd.warp_view(pts, cols, np.eye(3), np.zeros((3, 1)), K, H, W)
        assert len(valid) == len(u) and mask.dtype == np.int64
        assert not img.any()             # 0 inside the 9x9 mask, -1 outside it, and the 11x11 mask then zeroes all
