"""numpy + scipy restatement of LucidDreamer.generate_pcd's two warp loops: the oracle for luciddreamer_b200.pcd.

`perturb(coords) -> coords` is a test hook applied to the projected float64 coordinates [2, n] before the
interpolation, to probe how sensitive a frame is to round-off in the coordinates."""
from __future__ import annotations

import numpy as np
from scipy.interpolate import griddata
from scipy.ndimage import maximum_filter, minimum_filter

from luciddreamer_b200.pcd import compose_poses


def _edgemask(H, W):
    edgeN = 2
    e = np.ones((H - 2 * edgeN, W - 2 * edgeN))
    return np.pad(e, ((edgeN, edgeN), (edgeN, edgeN)))


def _project(pts, R, T, K, H, W):
    cam = R.dot(pts) + T
    pix = np.matmul(K, cam)
    valid = np.where(np.logical_and.reduce((pix[2] > 0, pix[0] / pix[2] >= 0, pix[0] / pix[2] <= W - 1,
                                            pix[1] / pix[2] >= 0, pix[1] / pix[2] <= H - 1)))[0]
    coords = pix[:2, valid] / pix[-1:, valid]
    return valid, coords, np.round(coords).astype(np.int32)


def _image(coords, rnd, colors, H, W, perturb=None):
    x, y = np.meshgrid(np.arange(W, dtype=np.float32), np.arange(H, dtype=np.float32), indexing='xy')
    grid = np.stack((x, y), axis=-1).reshape(-1, 2)
    c = perturb(coords) if perturb is not None else coords
    img = griddata(c.transpose(1, 0), colors, grid, method='linear', fill_value=0).reshape(H, W, 3)
    e = _edgemask(H, W)
    img = e[..., None] * img + (1 - e[..., None]) * np.pad(img[1:-1, 1:-1], ((1, 1), (1, 1), (0, 0)), mode='edge')
    m = np.zeros((H, W), dtype=np.float32)
    m[rnd[1], rnd[0]] = 1
    m = maximum_filter(m, size=(9, 9), axes=(0, 1))
    img = m[..., None] * img + (1 - m[..., None]) * (-1)
    mask = minimum_filter((img.sum(-1) != -3) * 1, size=(11, 11), axes=(0, 1))
    img = mask[..., None] * img + (1 - mask[..., None]) * 0
    return img, mask


def warp_view_host(pts, colors, R, T, K, H, W, perturb=None):
    """(image2, mask2, valid_idx, coords, round coords) of the dreaming stage for pose (R, T)."""
    valid, coords, rnd = _project(pts, R, T, K, H, W)
    img, mask = _image(coords, rnd, colors[valid], H, W, perturb)
    return img, mask, valid, coords, rnd


def align_frames_host(pts, colors, render_poses, internal_poses, K, H, W, perturb=None):
    """(uint8 frames, Pc2w list) of the aligning stage, views with no valid point skipped."""
    frames, mats = [], []
    for Rw2j, Tw2j, Pc2w in compose_poses(render_poses, internal_poses):
        valid, coords, rnd = _project(pts, Rw2j, Tw2j, K, H, W)
        if len(valid) == 0:
            continue
        img, _ = _image(coords, rnd, colors[valid], H, W, perturb)
        frames.append(np.round(img * 255.).astype(np.uint8))
        mats.append(Pc2w)
    return (np.stack(frames) if frames else np.zeros((0, H, W, 3), np.uint8)), mats
