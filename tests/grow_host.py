"""Growth of the dreamed cloud (luciddreamer_b200.pcd.grow_view), host side: the numpy + torch + scipy restatement
of LucidDreamer.generate_pcd's growth step, the oracle of the device path, and the seeded stand-ins for the
inpainting and depth models and the sparse cloud its tests use."""
from __future__ import annotations

import numpy as np
from scipy.interpolate import griddata

import pcd_cases


def stub_image(seed, H, W):
    """A seeded stand-in for the inpainting model's output: uint8 [H, W, 3]."""
    return np.random.default_rng(seed).integers(0, 256, (H, W, 3)).astype(np.uint8)


def stub_depth(seed, H, W, zero_rows=()):
    """A seeded stand-in for the depth model's output: float32 [H, W], positive, with the rows `zero_rows` set to 0."""
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:H, 0:W].astype(np.float32)
    d = (2.1 + 0.4 * np.cos(xx / 11.0) * np.sin(yy / 13.0) + 0.05 * rng.random((H, W))).astype(np.float32)
    d[list(zero_rows), :] = 0.0
    return d


def sparse_cloud(seed, H, W, step=16):
    """One float64 point near each node of a `step`-pixel lattice at depth 2: far enough apart that the 9x9 maximum
    and 11x11 minimum filters of the dreaming stage leave `mask2` all zero, so no point lies on its border."""
    rng = np.random.default_rng(seed)
    K = pcd_cases.intrinsics(H, W)
    gu, gv = np.meshgrid(np.arange(3.0, W - 1, step), np.arange(3.0, H - 1, step))
    u, v = gu.ravel() + rng.uniform(-0.4, 0.4, gu.size), gv.ravel() + rng.uniform(-0.4, 0.4, gv.size)
    z = np.full(u.shape, 2.0)
    pts = np.stack([(u - K[0, 2]) / K[0, 0] * z, (v - K[1, 2]) / K[1, 1] * z, z])
    return pts, rng.random((u.size, 3)).astype(np.float32)


def grow_view_host(pts, colors, R, T, K, mask2, valid_idx, coords, rnd, image, depth, perturb=None):
    """The dreaming stage's growth of the cloud (`generate_pcd` after `depth_curr = self.d(image_curr)`), with the
    reference's own numpy / torch expressions, without the scale fit, which leaves `trans3d` the identity.

    `image` is uint8 [H, W, 3] (or a PIL image), `depth` float32 [H, W]; the other inputs are `warp_view`'s. Returns
    (pts [3, N+M] float64, colors [N+M, 3] float32, border_valid_idx, new_depth). `perturb(new_depth) -> new_depth`
    is a test hook applied after the interpolation, to probe how sensitive the new points are to its round-off."""
    import torch
    H, W = mask2.shape
    x, y = np.meshgrid(np.arange(W, dtype=np.float32), np.arange(H, dtype=np.float32), indexing='xy')
    mask_hf = np.abs(mask2[:H - 1, :W - 1] - mask2[1:, :W - 1]) + np.abs(mask2[:H - 1, :W - 1] - mask2[:H - 1, 1:])
    mask_hf = np.pad(mask_hf, ((0, 1), (0, 1)), 'edge')
    mask_hf = np.where(mask_hf < 0.3, 0, 1)
    border_valid_idx = np.where(mask_hf[rnd[1], rnd[0]] == 1)[0]

    t_z2 = torch.tensor(depth)
    trans3d = torch.eye(4)                            # what the reference's fit leaves: sc never receives a gradient
    with torch.no_grad():
        coord_cam2 = torch.matmul(torch.tensor(np.linalg.inv(K)), torch.stack((torch.tensor(x) * t_z2, torch.tensor(y) * t_z2, 1 * t_z2), axis=0)[:, rnd[1, border_valid_idx], rnd[0, border_valid_idx]].reshape(3, -1))
        coord_world2 = (torch.tensor(np.linalg.inv(R)).float().matmul(coord_cam2) - torch.tensor(np.linalg.inv(R)).float().matmul(torch.tensor(T).float()))
        coord_world2_warp = torch.cat((coord_world2, torch.ones((1, border_valid_idx.shape[0]))), dim=0)
        coord_world2_trans = torch.matmul(trans3d, coord_world2_warp)
        coord_world2_trans = coord_world2_trans[:3] / coord_world2_trans[-1]
    trans3d = trans3d.numpy()

    camera_origin_coord_world2 = - np.linalg.inv(R).dot(T).astype(np.float32)
    vector_camorigin_to_campixels = coord_world2_trans.numpy() - camera_origin_coord_world2
    vector_camorigin_to_pcdpixels = pts[:, valid_idx[border_valid_idx]] - camera_origin_coord_world2
    with np.errstate(invalid='ignore', divide='ignore'):
        compensate_depth_coeff = np.sum(vector_camorigin_to_pcdpixels * vector_camorigin_to_campixels, axis=0) / np.sum(vector_camorigin_to_campixels * vector_camorigin_to_campixels, axis=0)
    compensate_pts_coord_world2_correspond = camera_origin_coord_world2 + vector_camorigin_to_campixels * compensate_depth_coeff.reshape(1, -1)
    compensate_coord_cam2_correspond = R.dot(compensate_pts_coord_world2_correspond) + T
    homography_coord_cam2_correspond = R.dot(coord_world2_trans.numpy()) + T
    compensate_depth_correspond = compensate_coord_cam2_correspond[-1] - homography_coord_cam2_correspond[-1]
    compensate_depth = np.concatenate((compensate_depth_correspond, np.zeros(4)), axis=0)
    pixel_cam2_correspond = coords[:, border_valid_idx]
    pixel_cam2_zero = np.array([[0, 0, W - 1, W - 1], [0, H - 1, 0, H - 1]])
    pixel_cam2 = np.concatenate((pixel_cam2_correspond, pixel_cam2_zero), axis=1).transpose(1, 0)

    masked_pixels_xy = np.stack(np.where(1 - mask2), axis=1)[:, [1, 0]]
    new_depth_linear = griddata(pixel_cam2, compensate_depth, masked_pixels_xy)
    new_depth_nearest = griddata(pixel_cam2, compensate_depth, masked_pixels_xy, method='nearest')
    new_depth = np.where(np.isnan(new_depth_linear), new_depth_nearest, new_depth_linear)
    if perturb is not None:
        new_depth = perturb(new_depth)

    sel = np.where(1 - mask2.reshape(-1))[0]
    pts_coord_cam2 = np.matmul(np.linalg.inv(K), np.stack((x * depth, y * depth, 1 * depth), axis=0).reshape(3, -1))[:, sel]
    x_nonmask, y_nonmask = x.reshape(-1)[sel], y.reshape(-1)[sel]
    compensate_pts_coord_cam2 = np.matmul(np.linalg.inv(K), np.stack((x_nonmask * new_depth, y_nonmask * new_depth, 1 * new_depth), axis=0))
    new_warp_pts_coord_cam2 = pts_coord_cam2 + compensate_pts_coord_cam2
    new_pts_coord_world2 = (np.linalg.inv(R).dot(new_warp_pts_coord_cam2) - np.linalg.inv(R).dot(T)).astype(np.float32)
    new_pts_coord_world2_warp = np.concatenate((new_pts_coord_world2, np.ones((1, new_pts_coord_world2.shape[1]))), axis=0)
    with np.errstate(invalid='ignore'):
        new_pts_coord_world2 = np.matmul(trans3d, new_pts_coord_world2_warp)
        new_pts_coord_world2 = new_pts_coord_world2[:3] / new_pts_coord_world2[-1]
    new_pts_colors2 = (np.array(image).reshape(-1, 3).astype(np.float32) / 255.)[sel]
    return (np.concatenate((pts, new_pts_coord_world2), axis=-1), np.concatenate((colors, new_pts_colors2), axis=0),
            border_valid_idx, new_depth)
