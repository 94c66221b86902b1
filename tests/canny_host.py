"""Host restatement of what luciddreamer_b200.scene computes for each training frame: the reference's compositing
(`loadCamerasFromData`) and `image2canny`'s `1 - cv2.Canny(u8, 50, 150) / 255` (OpenCV's Canny for 8-bit
three-channel input, aperture 3, L1 norm), written out in numpy so that the golden data and the device can be
checked against something that states every rule."""
from __future__ import annotations

import numpy as np
from scipy import ndimage

TG22 = 13573                      # round(tan(22.5 deg) * 2^15)


def rgba(frames: np.ndarray) -> np.ndarray:
    """[F, H, W, 3 or 4] uint8 -> RGBA, alpha 255 where there is none (what `Image.convert("RGBA")` gives)."""
    if frames.shape[-1] == 4:
        return frames
    a = np.full(frames.shape[:-1] + (1,), 255, np.uint8)
    return np.concatenate([frames, a], axis=-1)


def composite(frames: np.ndarray, white_background: bool) -> np.ndarray:
    """`original_image` [F, 3, H, W] float32: norm = u / 255.0 and rgb * a + bg * (1 - a) in float64, rounded to
    float32, clamped to [0, 1]."""
    norm = rgba(frames) / 255.0
    bg = np.array([1, 1, 1]) if white_background else np.array([0, 0, 0])
    arr = norm[..., :3] * norm[..., 3:4] + bg * (1 - norm[..., 3:4])
    return np.clip(arr.astype(np.float32), 0.0, 1.0).transpose(0, 3, 1, 2).copy()


def canny_input(image: np.ndarray) -> np.ndarray:
    """`(original_image.permute(1, 2, 0) * 255.).astype(np.uint8)` for one [3, H, W] float32 image."""
    return (image.transpose(1, 2, 0) * 255.).astype(np.uint8)


def _sobel(ch: np.ndarray):
    p = np.pad(ch.astype(np.int32), 1, mode="edge")
    dx = (p[:-2, 2:] + 2 * p[1:-1, 2:] + p[2:, 2:]) - (p[:-2, :-2] + 2 * p[1:-1, :-2] + p[2:, :-2])
    dy = (p[2:, :-2] + 2 * p[2:, 1:-1] + p[2:, 2:]) - (p[:-2, :-2] + 2 * p[:-2, 1:-1] + p[:-2, 2:])
    return dx, dy


def gradient(u8: np.ndarray):
    """Per pixel, the 3x3 Sobel (replicated borders) of the channel with the largest |dx| + |dy|, ties to the lowest
    channel: (dx, dy, m) int32 [H, W]."""
    dx, dy = _sobel(u8[..., 0])
    m = np.abs(dx) + np.abs(dy)
    for c in range(1, u8.shape[-1]):
        cx, cy = _sobel(u8[..., c])
        cm = np.abs(cx) + np.abs(cy)
        take = cm > m
        dx, dy, m = np.where(take, cx, dx), np.where(take, cy, dy), np.where(take, cm, m)
    return dx, dy, m


def classify(u8: np.ndarray, low: int = 50, high: int = 150):
    """Candidates (m > low and a local maximum along the gradient) and strong pixels (candidates with m > high).
    The neighbour tests are OpenCV's: the integer tan 22.5 / 67.5 deg sectors, `>` towards the previous pixel and
    `>=` towards the next one in the horizontal and vertical sectors, `>` on both sides in the diagonal ones;
    magnitudes outside the image are 0."""
    dx, dy, m = gradient(u8)
    M = np.pad(m, 1)
    H, W = m.shape
    x = np.abs(dx).astype(np.int64)
    y = np.abs(dy).astype(np.int64) << 15
    tg22x = x * TG22
    tg67x = tg22x + (x << 16)
    horiz = y < tg22x
    vert = ~horiz & (y > tg67x)
    s = np.where((dx ^ dy) < 0, -1, 1)
    ii, jj = np.mgrid[0:H, 0:W]
    ii, jj = ii + 1, jj + 1                                            # indices into the padded M
    nms_h = (m > M[ii, jj - 1]) & (m >= M[ii, jj + 1])
    nms_v = (m > M[ii - 1, jj]) & (m >= M[ii + 1, jj])
    nms_d = (m > M[ii - 1, jj - s]) & (m > M[ii + 1, jj + s])
    nms = np.where(horiz, nms_h, np.where(vert, nms_v, nms_d))
    cand = (m > low) & nms
    return cand, cand & (m > high)


def canny(u8: np.ndarray, low: int = 50, high: int = 150) -> np.ndarray:
    """cv2.Canny(u8, low, high) for [H, W, 3] uint8: the 8-connected closure of the strong pixels through the
    candidates, as 0 / 255 uint8."""
    cand, strong = classify(u8, low, high)
    lab, _ = ndimage.label(cand, structure=np.ones((3, 3), bool))
    keep = np.zeros(lab.max() + 1, bool)
    keep[lab[strong]] = True
    keep[0] = False
    return np.where(keep[lab], 255, 0).astype(np.uint8)


def canny_mask(image: np.ndarray) -> np.ndarray:
    """`canny_mask` [H, W] float32 of one [3, H, W] `original_image`: 1 - Canny / 255."""
    return (1. - canny(canny_input(image)) / 255.).astype(np.float32)


def scene_images(frames: np.ndarray, white_background: bool):
    """(original_image [F, 3, H, W], canny_mask [F, H, W]) for uint8 frames [F, H, W, 3 or 4]."""
    img = composite(frames, white_background)
    return img, np.stack([canny_mask(im) for im in img]) if len(img) else np.zeros((0,) + img.shape[2:], np.float32)
