"""Writes canny_golden.npz: training frames and what the reference's Camera makes of them, computed with the
reference's own expressions and cv2.Canny (OpenCV 4.13), for tests of luciddreamer_b200.scene.

Per case `<name>/`: `frame` [H, W, 3 or 4] uint8, `white` (0 / 1), `canny` [H, W] uint8 = cv2.Canny(u8, 50, 150)
of the composited frame, and, for frames up to 64 x 64, `image` [3, H, W] float32, the composited `original_image`.
The compositing is loadCamerasFromData's (PIL's RGBA conversion, float64 arithmetic, torch.Tensor's rounding to
float32), and u8 is image2canny's `(image.permute(1, 2, 0).numpy() * 255.).astype(np.uint8)`.

The Sobel magnitude |dx| + |dy| is always even (every weight of dx + dy is even), so no pixel can sit at 51 or 151;
the threshold cases put pixels at 50 / 52 and 150 / 152 instead.

Run from the repository root: python tests/golden/make_canny_golden.py
"""
import os

import cv2
import numpy as np
import torch
from PIL import Image

HERE = os.path.dirname(os.path.abspath(__file__))


def reference_camera_images(frame, white):
    """loadCamerasFromData's compositing and image2canny's input, as the reference writes them."""
    im_data = np.array(Image.fromarray(frame).convert("RGBA"))
    bg = np.array([1, 1, 1]) if white else np.array([0, 0, 0])
    norm_data = im_data / 255.0
    arr = norm_data[:, :, :3] * norm_data[:, :, 3:4] + bg * (1 - norm_data[:, :, 3:4])
    image = torch.Tensor(arr).permute(2, 0, 1).clamp(0.0, 1.0)
    u8 = (image.permute(1, 2, 0).numpy() * 255.).astype(np.uint8)
    return image.numpy(), cv2.Canny(u8, 50, 150)


def rgb(*ch):
    return np.ascontiguousarray(np.stack([np.clip(c, 0, 255) for c in ch], -1).astype(np.uint8))


def grey(u):
    return rgb(u, u, u)


def half_plane(H, W, a, b, slope=40.0, lo=40, hi=200):
    """A straight soft edge whose gradient points along (a, b)."""
    yy, xx = np.mgrid[0:H, 0:W].astype(np.float64)
    t = (a * (xx - W / 2) + b * (yy - H / 2)) / np.hypot(a, b)
    return np.clip(np.round(lo + (hi - lo) / (1 + np.exp(-t * slope / (hi - lo)))), 0, 255)


def spiral(H, W, weak=30, strong=200):
    """A one-pixel spiral line (turns four pixels apart) of weak intensity spanning the frame, strong only over its
    last few pixels."""
    u = np.zeros((H, W))
    path = []
    top, left, bottom, right = 1, 1, H - 2, W - 2
    while top <= bottom and left <= right:
        path += [(top, x) for x in range(left, right + 1)]
        path += [(y, right) for y in range(top + 1, bottom + 1)]
        if top < bottom:
            path += [(bottom, x) for x in range(right - 1, left - 1, -1)]
        if left < right:
            path += [(y, left) for y in range(bottom - 1, top, -1)]
        top, left, bottom, right = top + 4, left + 4, bottom - 4, right - 4
    for k, (y, x) in enumerate(path):
        u[y, x] = strong if k >= len(path) - 3 else weak
    return u


def cases():
    rng = np.random.default_rng(20261016)
    out = []
    # seeded frames: noise, smoothed noise (natural-looking edges), blocky colour patches
    for k, (H, W) in enumerate([(24, 32), (37, 29), (64, 64)]):
        out.append((f"noise_{H}x{W}", rng.integers(0, 256, (H, W, 3)).astype(np.uint8), k % 2))
        sm = cv2.GaussianBlur(rng.integers(0, 256, (H, W, 3)).astype(np.uint8), (0, 0), 1.5)
        out.append((f"smooth_{H}x{W}", sm, 0))
        blk = np.kron(rng.integers(0, 4, (H // 4 + 1, W // 4 + 1, 3)) * 70, np.ones((4, 4, 1)))[:H, :W]
        out.append((f"blocks_{H}x{W}", blk.astype(np.uint8), 1))
    # magnitude exactly at and just above each threshold: a single bump of v puts 2v on its eight neighbours
    for v in (25, 26, 75, 76):
        u = np.zeros((9, 11)); u[4, 5] = v
        out.append((f"bump_m{2 * v}", grey(u), 0))
    # ramps: a step of h gives 4h beside it, a linear ramp (a, b) gives 8(|a| + |b|)
    for h in (12, 13, 37, 38):
        u = np.zeros((8, 12)); u[:, 6:] = h
        out.append((f"step_m{4 * h}", grey(u), 0))
    yy, xx = np.mgrid[0:10, 0:12]
    for a, b in ((6, 0), (6, 1), (18, 0), (18, 1), (3, 3), (9, 10)):
        out.append((f"ramp_{a}_{b}", grey(a * xx + b * yy), 0))
    # edges on both sides of the tan 22.5 / tan 67.5 sector boundaries, in all four quadrants
    t22, t67 = np.tan(np.pi / 8), np.tan(3 * np.pi / 8)
    for name, r in (("22lo", t22 * 0.97), ("22hi", t22 * 1.03), ("67lo", t67 * 0.97), ("67hi", t67 * 1.03)):
        for sx, sy in ((1, 1), (-1, 1)):
            for slope in (25.0, 60.0):
                out.append((f"angle_{name}_{sx}{sy}_{int(slope)}", grey(half_plane(33, 41, sx, sy * r, slope)), 0))
    # channel ties: equal magnitudes with different (dx, dy) in different channels
    u = np.zeros((12, 12)); u[:, 6:] = 100
    out.append(("tie_xy", rgb(u, u.T, u), 0))
    out.append(("tie_sign", rgb(u, 255 - u, u.T), 0))
    out.append(("tie_later_wins", rgb(u * 0.5, u.T, u), 0))
    d = half_plane(20, 20, 1, 1, 80.0)
    out.append(("tie_diag", rgb(d, d[:, ::-1], d[::-1]), 0))
    # plateaus where the > / >= asymmetry decides which side of a step is marked
    for name, (H, W) in (("v", (10, 12)), ("h", (12, 10))):
        u = np.zeros((H, W))
        if name == "v":
            u[:, W // 2:] = 120
        else:
            u[H // 2:, :] = 120
        out.append((f"plateau_{name}", grey(u), 0))
        out.append((f"plateau_{name}_down", grey(120 - u), 0))
    u = np.zeros((12, 12)); u[np.add.outer(np.arange(12), np.arange(12)) >= 12] = 120
    out.append(("plateau_diag", grey(u), 0))
    # edges on the first and last rows and columns
    for name, sl in (("col0", np.s_[:, 1:]), ("colN", np.s_[:, -1:]), ("row0", np.s_[1:, :]), ("rowN", np.s_[-1:, :])):
        u = np.zeros((9, 13)); u[sl] = 200
        out.append((f"border_{name}", grey(u), 0))
    # weak chains reaching a strong pixel at one end only
    u = np.zeros((16, 40)); u[8, 2:38] = 30; u[8, 36:38] = 200
    out.append(("chain_line", grey(u), 0))
    out.append(("chain_spiral", grey(spiral(64, 64)), 0))
    out.append(("chain_spiral_512", grey(spiral(512, 512)), 1))
    # tiny sizes and the working size
    out.append(("tiny_3x3", rng.integers(0, 256, (3, 3, 3)).astype(np.uint8), 0))
    out.append(("tiny_5x7", rng.integers(0, 256, (5, 7, 3)).astype(np.uint8), 1))
    big = cv2.GaussianBlur(rng.integers(0, 256, (512, 512, 3)).astype(np.uint8), (0, 0), 2.0)
    out.append(("seeded_512", big, 0))
    # RGBA frames: alpha below 255 over both backgrounds
    for white in (0, 1):
        f = rng.integers(0, 256, (40, 48, 4)).astype(np.uint8)
        f[..., 3] = np.where(rng.random((40, 48)) < 0.3, 255, f[..., 3])
        out.append((f"rgba_{'white' if white else 'black'}", f, white))
        out.append((f"rgba_smooth_{white}", cv2.GaussianBlur(f, (0, 0), 1.2), white))
    return out


def main():
    arrays = {}
    for name, frame, white in cases():
        image, canny = reference_camera_images(frame, white)
        arrays[f"{name}/frame"] = frame
        arrays[f"{name}/white"] = np.int32(white)
        arrays[f"{name}/canny"] = canny
        if frame.shape[0] * frame.shape[1] <= 64 * 64:
            arrays[f"{name}/image"] = image
        print(f"{name:28s} {frame.shape} edges {int((canny > 0).sum())}")
    np.savez_compressed(os.path.join(HERE, "canny_golden.npz"), **arrays)


if __name__ == "__main__":
    main()
