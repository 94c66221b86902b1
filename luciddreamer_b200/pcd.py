"""Warp LucidDreamer's generated point cloud into camera views on the device (include/gspcd.h).

`warp_view` replaces the per-pose projection and `griddata` block of `LucidDreamer.generate_pcd`'s dreaming stage,
`align_frames` the whole aligning stage (every generation pose times every hemisphere view, in one call). Both
follow the reference's numpy expressions: the projection in float64, `np.where` order of the valid points,
`np.round` (half to even), linear interpolation in the Delaunay triangulation of the projected points with
fill value 0, the edge ring, and the 9x9 maximum / 11x11 minimum filters with `mode='reflect'`.

One input differs from the reference: with fewer than three valid points, or only collinear ones, scipy's
`griddata` raises `QhullError` and `generate_pcd` aborts. Here the interpolated value is then the fill value 0
and the masks still apply.

There is no CPU path: the inputs are numpy arrays or CUDA tensors, and the work runs on the current CUDA device.
Points may be float32 or float64 (widened exactly); colours must be float32, as generate_pcd makes them.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np
import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "pcd_csrc", "libgspcd.so")

GSPCD_OK = 0
_P = C.c_void_p
SYMBOLS = [
    ("gspcd_abi_version", C.c_int, []),
    ("gspcd_scratch_bytes", C.c_int, [C.c_int64, C.c_int32, C.c_int32, C.POINTER(C.c_uint64)]),
    ("gspcd_align", C.c_int, [_P, _P, C.c_int64, _P, _P, C.c_int32, C.c_int32, C.c_int32, _P, _P, _P, _P,
                              C.c_uint64, _P]),
    ("gspcd_warp_view", C.c_int, [_P, _P, C.c_int64, _P, _P, C.c_int32, C.c_int32, _P, _P, _P, _P, _P, _P, _P, _P,
                                  C.c_uint64, _P]),
]

_lib = None


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(f"{LIB_PATH} is not built; run __graft_entry__.build()")
        L = C.CDLL(LIB_PATH)
        for name, res, args in SYMBOLS:
            f = getattr(L, name)
            f.restype, f.argtypes = res, args
        _lib = L
    return _lib


def _check(rc: int, what: str) -> None:
    if rc != GSPCD_OK:
        raise RuntimeError(f"{what} failed with code {rc}")


def _device() -> torch.device:
    if not torch.cuda.is_available():
        raise RuntimeError("luciddreamer_b200.pcd needs a CUDA device; there is no CPU path")
    return torch.device("cuda", torch.cuda.current_device())


def _as_cuda(a, dtype: torch.dtype, dev: torch.device, name: str) -> torch.Tensor:
    if isinstance(a, np.ndarray):
        return torch.from_numpy(np.ascontiguousarray(a)).to(device=dev, dtype=dtype)
    if isinstance(a, torch.Tensor) and a.is_cuda:
        if a.dtype not in (torch.float32, torch.float64):
            raise TypeError(f"{name} must be float32 or float64, got {a.dtype}")
        return a.to(device=dev, dtype=dtype).contiguous()       # float32 -> float64 widens exactly
    raise TypeError(f"{name} must be a numpy array or a CUDA tensor")


def _cloud(pts, colors, dev):
    p = _as_cuda(pts, torch.float64, dev, "pts")
    # colours stay float32 as generate_pcd makes them; a float64 colour would be interpolated differently there
    if getattr(colors, "dtype", None) not in (np.float32, torch.float32):
        raise TypeError(f"colors must be float32, got {getattr(colors, 'dtype', type(colors))}")
    c = _as_cuda(colors, torch.float32, dev, "colors")
    if p.dim() != 2 or p.shape[0] != 3:
        raise ValueError(f"pts must be [3, N], got {tuple(p.shape)}")
    if c.shape != (p.shape[1], 3):
        raise ValueError(f"colors must be [N, 3] with N = {p.shape[1]}, got {tuple(c.shape)}")
    return p, c


def _scratch(n: int, H: int, W: int, dev) -> torch.Tensor:
    b = C.c_uint64()
    _check(lib().gspcd_scratch_bytes(n, H, W, C.byref(b)), "gspcd_scratch_bytes")
    return torch.empty(b.value, dtype=torch.uint8, device=dev)


def _stream(dev) -> C.c_void_p:
    return C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)


def _K64(K) -> np.ndarray:
    K = np.ascontiguousarray(np.asarray(K, dtype=np.float64))
    if K.shape != (3, 3):
        raise ValueError(f"K must be 3x3, got {K.shape}")
    return K


def _pose12(R, T) -> np.ndarray:
    R = np.asarray(R, dtype=np.float64).reshape(3, 3)
    T = np.asarray(T, dtype=np.float64).reshape(3)
    return np.ascontiguousarray(np.concatenate([R.reshape(-1), T]))


def warp_view(pts, colors, R, T, K, H: int, W: int):
    """The dreaming stage's warp of the cloud into pose (R, T) (`generate_pcd`, `image2` through `mask2`).

    Returns numpy arrays with the reference's dtypes: `image2` [H, W, 3] float64, `mask2` [H, W] int64,
    `valid_idx` [n] int64, the float64 coordinates [2, n] and the round coordinates [2, n] int32."""
    dev = _device()
    p, c = _cloud(pts, colors, dev)
    n = p.shape[1]
    K = _K64(K)
    pose = _pose12(R, T)
    scratch = _scratch(n, H, W, dev)
    image = torch.empty((H, W, 3), dtype=torch.float64, device=dev)
    mask = torch.empty((H, W), dtype=torch.int32, device=dev)
    vidx = torch.empty(max(n, 1), dtype=torch.int32, device=dev)
    coords = torch.empty((2, max(n, 1)), dtype=torch.float64, device=dev)
    rnd = torch.empty((2, max(n, 1)), dtype=torch.int32, device=dev)
    small = torch.zeros(2, dtype=torch.int32, device=dev)         # count, status
    _check(lib().gspcd_warp_view(p.data_ptr(), c.data_ptr(), n, pose.ctypes.data, K.ctypes.data, H, W,
                                 image.data_ptr(), mask.data_ptr(), vidx.data_ptr(), coords.data_ptr(), rnd.data_ptr(),
                                 small.data_ptr(), small.data_ptr() + 4, scratch.data_ptr(), scratch.numel(),
                                 _stream(dev)), "gspcd_warp_view")
    count, status = small.cpu().tolist()
    if status:
        raise RuntimeError(f"gspcd_warp_view: status {status} (exact predicate precision or walk cap exceeded)")
    if n == 0:
        return (image.cpu().numpy(), mask.cpu().numpy().astype(np.int64), np.zeros(0, np.int64),
                np.zeros((2, 0), np.float64), np.zeros((2, 0), np.int32))
    return (image.cpu().numpy(), mask.cpu().numpy().astype(np.int64), vidx[:count].cpu().numpy().astype(np.int64),
            coords[:, :count].cpu().numpy(), rnd[:, :count].cpu().numpy())


def compose_poses(render_poses, internal_poses):
    """World-to-view (Rw2j, Tw2j) and the frame's Pc2w for every (generation pose, hemisphere view), in the
    aligning stage's order, with the reference's own numpy expressions."""
    yz_reverse = np.array([[1, 0, 0], [0, -1, 0], [0, 0, -1]])
    out = []
    for i in range(len(render_poses)):
        for j in range(len(internal_poses)):
            Rw2i = render_poses[i, :3, :3]
            Tw2i = render_poses[i, :3, 3:4]
            Ri2j = internal_poses[j, :3, :3]
            Ti2j = internal_poses[j, :3, 3:4]
            Rw2j = np.matmul(Ri2j, Rw2i)
            Tw2j = np.matmul(Ri2j, Tw2i) + Ti2j
            Rj2w = np.matmul(yz_reverse, Rw2j).T
            Tj2w = -np.matmul(Rj2w, np.matmul(yz_reverse, Tw2j))
            Pc2w = np.concatenate((Rj2w, Tj2w), axis=1)
            Pc2w = np.concatenate((Pc2w, np.array([[0, 0, 0, 1]])), axis=0)
            out.append((Rw2j, Tw2j, Pc2w))
    return out


def align_frames(pts, colors, render_poses, internal_poses, K, H: int, W: int):
    """The aligning stage of `generate_pcd`: every generation pose times every hemisphere view, one device call.

    Returns (frames [n, H, W, 3] uint8, [Pc2w 4x4 float64] * n), skipping views with no valid point like the
    reference's `continue`. `frames[k]` is `np.round(imagej*255.).astype(np.uint8)` of the k-th kept view."""
    dev = _device()
    p, c = _cloud(pts, colors, dev)
    n = p.shape[1]
    K = _K64(K)
    views = compose_poses(np.asarray(render_poses), np.asarray(internal_poses))
    V = len(views)
    poses = np.ascontiguousarray(np.stack([_pose12(R, T) for R, T, _ in views])) if V else np.zeros((0, 12))
    scratch = _scratch(n, H, W, dev)
    frames = torch.empty((max(V, 1), H, W, 3), dtype=torch.uint8, device=dev)
    small = torch.zeros(V + 1, dtype=torch.int32, device=dev)     # counts[V], status
    _check(lib().gspcd_align(p.data_ptr(), c.data_ptr(), n, poses.ctypes.data, K.ctypes.data, V, H, W,
                             frames.data_ptr(), small.data_ptr(), small.data_ptr() + 4 * V, scratch.data_ptr(),
                             scratch.numel(), _stream(dev)), "gspcd_align")
    small_h = small.cpu().numpy()
    if small_h[V]:
        raise RuntimeError(f"gspcd_align: status {small_h[V]} (exact predicate precision or walk cap exceeded)")
    keep = [k for k in range(V) if small_h[k] > 0]
    out = frames[keep].cpu().numpy() if keep else np.zeros((0, H, W, 3), np.uint8)
    return out, [views[k][2] for k in keep]
