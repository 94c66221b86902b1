"""Seeded point clouds and cameras for the point-cloud warp tests (luciddreamer_b200.pcd)."""
from __future__ import annotations

import numpy as np


def intrinsics(H, W, f=None):
    f = float(max(H, W)) if f is None else f
    return np.array([[f, 0.0, W / 2.0], [0.0, f, H / 2.0], [0.0, 0.0, 1.0]])


def depth_cloud(seed, H, W, extra=0):
    """A depth-map cloud unprojected through the identity pose like generate_pcd's initialisation (float32
    points, float32 colours in [0, 1]), plus `extra` random points in front of the camera."""
    rng = np.random.default_rng(seed)
    K = intrinsics(H, W)
    yy, xx = np.mgrid[0:H, 0:W].astype(np.float32)
    depth = (2.0 + 0.5 * np.sin(xx / 9.0) * np.cos(yy / 7.0) + 0.05 * rng.random((H, W))).astype(np.float32)
    x, y = np.meshgrid(np.arange(W, dtype=np.float32), np.arange(H, dtype=np.float32), indexing='xy')
    cam = np.matmul(np.linalg.inv(K), np.stack((x * depth, y * depth, 1 * depth), axis=0).reshape(3, -1))
    pts = cam.astype(np.float32)
    cols = rng.integers(0, 256, size=(H * W, 3)).astype(np.float32) / 255.
    if extra:
        z = rng.uniform(1.5, 3.0, extra)
        u, v = rng.uniform(-0.1 * W, 1.1 * W, extra), rng.uniform(-0.1 * H, 1.1 * H, extra)
        e = np.stack([(u - W / 2.0) / K[0, 0] * z, (v - H / 2.0) / K[1, 1] * z, z]).astype(np.float32)
        pts = np.concatenate([pts, e], axis=1)
        cols = np.concatenate([cols, rng.integers(0, 256, size=(extra, 3)).astype(np.float32) / 255.])
    return pts, cols


def random_cloud(seed, n, H, W):
    """n generic float64 points in front of the camera, spread a little past the view."""
    rng = np.random.default_rng(seed)
    K = intrinsics(H, W)
    z = rng.uniform(1.0, 4.0, n)
    u, v = rng.uniform(-0.2 * W, 1.2 * W, n), rng.uniform(-0.2 * H, 1.2 * H, n)
    pts = np.stack([(u - W / 2.0) / K[0, 0] * z, (v - H / 2.0) / K[1, 1] * z, z])
    return pts, rng.random((n, 3)).astype(np.float32)


def random_pose(seed, deg=6.0, shift=0.15):
    rng = np.random.default_rng(seed)
    a, b, c = np.deg2rad(rng.uniform(-deg, deg, 3))
    Rx = np.array([[1, 0, 0], [0, np.cos(a), -np.sin(a)], [0, np.sin(a), np.cos(a)]])
    Ry = np.array([[np.cos(b), 0, np.sin(b)], [0, 1, 0], [-np.sin(b), 0, np.cos(b)]])
    Rz = np.array([[np.cos(c), -np.sin(c), 0], [np.sin(c), np.cos(c), 0], [0, 0, 1]])
    return Rz @ Ry @ Rx, rng.uniform(-shift, shift, (3, 1))


def hemisphere(center_depth, degree=5):
    """Five hemisphere views around the scene centre, the third one the identity."""
    th_l, phi_l = np.array([degree, 0, 0, 0, -degree]), np.array([0, -degree, 0, degree, 0])
    P = np.zeros((5, 3, 4))
    for i, (th, phi) in enumerate(zip(th_l, phi_l)):
        t, p = th / 180 * np.pi, phi / 180 * np.pi
        P[i, :3, :3] = np.array([[np.cos(t), 0, -np.sin(t)], [0, 1, 0], [np.sin(t), 0, np.cos(t)]]) @ \
            np.array([[1, 0, 0], [0, np.cos(p), -np.sin(p)], [0, np.sin(p), np.cos(p)]])
        d = center_depth
        P[i, :3, 3:4] = np.array([d * np.sin(t), 0, d - d * np.cos(t)]).reshape(3, 1) + \
            np.array([0, d * np.sin(p), d - d * np.cos(p)]).reshape(3, 1)
    return P


def rotate360(n=10, step_deg=36.0):
    """Generation poses turning about the vertical axis (n of them, the first the identity)."""
    P = np.zeros((n, 3, 4))
    for i in range(n):
        t = np.deg2rad(step_deg * i)
        P[i, :3, :3] = np.array([[np.cos(t), 0, np.sin(t)], [0, 1, 0], [-np.sin(t), 0, np.cos(t)]])
    return P
