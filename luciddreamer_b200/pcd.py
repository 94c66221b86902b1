"""Warp LucidDreamer's generated point cloud into camera views on the device (include/gspcd.h).

`warp_view` replaces the per-pose projection and `griddata` block of `LucidDreamer.generate_pcd`'s dreaming stage,
`grow_view` the same stage's growth of the cloud from the inpainted view, `align_frames` the whole aligning stage (every generation pose times every hemisphere view, in one call). Both
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
    ("gspcd_grow_scratch_bytes", C.c_int, [C.c_int64, C.c_int32, C.c_int32, C.POINTER(C.c_uint64)]),
    ("gspcd_grow_view", C.c_int, [_P, C.c_int64, C.c_int32, _P, _P, _P, C.c_int64, _P, _P, _P, C.c_int32, C.c_int32,
                                  _P, C.c_int64, _P, _P, _P, _P, _P, _P, _P, C.c_uint64, _P]),
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


def align_frames(pts, colors, render_poses, internal_poses, K, H: int, W: int, on_device: bool = False):
    """The aligning stage of `generate_pcd`: every generation pose times every hemisphere view, one device call.

    Returns (frames [n, H, W, 3] uint8, [Pc2w 4x4 float64] * n), skipping views with no valid point like the
    reference's `continue`. `frames[k]` is `np.round(imagej*255.).astype(np.uint8)` of the k-th kept view. With
    `on_device` the frames stay on the device as a uint8 CUDA tensor, ready for `scene.build_scene(frames=...)`."""
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
    if on_device:
        out = frames[:V] if len(keep) == V else frames[keep]
    else:
        out = frames[keep].cpu().numpy() if keep else np.zeros((0, H, W, 3), np.uint8)
    return out, [views[k][2] for k in keep]


def grow_matrices(R, T, K) -> np.ndarray:
    """The 48 host float64 values gspcd_grow_view reads, formed with the reference's own numpy / torch expressions
    (`generate_pcd`, dreaming stage), so that the device never inverts anything."""
    invR = np.linalg.inv(R)
    invR32 = torch.tensor(invR).float()
    invRT32 = invR32.matmul(torch.tensor(T).float())                  # the torch product of the border points
    origin = - np.linalg.inv(R).dot(T).astype(np.float32)              # camera_origin_coord_world2
    parts = [np.linalg.inv(K), invR32.numpy(), invRT32.numpy(), origin, invR, np.linalg.inv(R).dot(T), R, T]
    return np.ascontiguousarray(np.concatenate([np.asarray(a, np.float64).reshape(-1) for a in parts]))


def _as_cuda_exact(a, dtype, dev, name, shape):
    """A numpy array, PIL image or CUDA tensor of exactly `dtype` and `shape`, on the device."""
    if isinstance(a, torch.Tensor):
        if not a.is_cuda:
            raise TypeError(f"{name} must be a numpy array or a CUDA tensor")
        t = a
    else:
        t = np.asarray(a)
        if t.dtype == object:
            raise TypeError(f"{name} must be a numpy array, a PIL image or a CUDA tensor")
        t = torch.from_numpy(np.array(t))                              # a copy: PIL arrays are read-only
    if t.dtype != dtype:
        raise TypeError(f"{name} must be {dtype}, got {t.dtype}")
    if tuple(t.shape) != tuple(shape):
        raise ValueError(f"{name} must have shape {tuple(shape)}, got {tuple(t.shape)}")
    return t.to(dev).contiguous()


def grow_view(pts, colors, R, T, K, mask2, valid_idx, pixel_coord, round_coord, image, depth,
              return_details: bool = False):
    """The dreaming stage's growth of the cloud from the inpainted view (`generate_pcd` after
    `depth_curr = self.d(image_curr)`): border points of `mask2`, their depth corrections, linear (then nearest)
    interpolation of the correction over the pixels where `mask2 != 1`, and their back-projection and colours.

    `pts` [3, N] float32 (the first view's cloud) or float64, `colors` [N, 3] float32; `K` float32, as
    `CameraParams` makes it; `mask2`, `valid_idx`, `pixel_coord`, `round_coord` as `warp_view` returns them; `image`
    uint8 [H, W, 3] (numpy, PIL image or CUDA tensor), `depth` float32 [H, W] (numpy or CUDA tensor). Returns the
    grown cloud as numpy, float64 [3, N + M] and float32 [N + M, 3], the old points copied exactly; with
    `return_details` also `border_valid_idx` (int64) and the interpolated correction `new_depth` [M] float64.

    The reference's scale fit is not run: `torch.tensor([[sc, ...]])` copies `sc`, so no gradient reaches it and
    `trans3d` stays the identity."""
    dev = _device()
    if getattr(K, "dtype", None) != np.float32:
        raise TypeError(f"K must be float32 as CameraParams makes it, got {getattr(K, 'dtype', type(K))}")
    K = np.asarray(K)
    if K.shape != (3, 3):
        raise ValueError(f"K must be 3x3, got {K.shape}")
    R = np.asarray(R, dtype=np.float64).reshape(3, 3)
    T = np.asarray(T, dtype=np.float64).reshape(3, 1)
    if isinstance(pts, torch.Tensor) and not pts.is_cuda or isinstance(colors, torch.Tensor) and not colors.is_cuda:
        raise TypeError("pts and colors must be numpy arrays or CUDA tensors")
    pts_h = pts.cpu().numpy() if isinstance(pts, torch.Tensor) else np.asarray(pts)
    cols_h = colors.cpu().numpy() if isinstance(colors, torch.Tensor) else np.asarray(colors)
    if pts_h.dtype not in (np.float32, np.float64) or pts_h.ndim != 2 or pts_h.shape[0] != 3:
        raise ValueError(f"pts must be [3, N] float32 or float64, got {pts_h.shape} {pts_h.dtype}")
    if cols_h.dtype != np.float32 or cols_h.shape != (pts_h.shape[1], 3):
        raise ValueError(f"colors must be [N, 3] float32 with N = {pts_h.shape[1]}, got {cols_h.shape} {cols_h.dtype}")
    mask_h = np.asarray(mask2)
    if mask_h.ndim != 2 or mask_h.dtype.kind not in "iub":
        raise ValueError(f"mask2 must be an integer [H, W] array, got {mask_h.shape} {mask_h.dtype}")
    H, W = mask_h.shape
    valid_h = np.asarray(valid_idx)
    nv = valid_h.shape[0] if valid_h.ndim == 1 else -1
    coords_h, rnd_h = np.asarray(pixel_coord), np.asarray(round_coord)
    if nv < 0 or coords_h.shape != (2, nv) or rnd_h.shape != (2, nv) or coords_h.dtype != np.float64 or \
            rnd_h.dtype != np.int32 or valid_h.dtype.kind not in "iu":
        raise ValueError("valid_idx [n], pixel_coord [2, n] float64 and round_coord [2, n] int32 as warp_view "
                         "returns them are required")
    n = pts_h.shape[1]
    if nv and (valid_h.min() < 0 or valid_h.max() >= n or rnd_h[0].min() < 0 or rnd_h[0].max() >= W or
               rnd_h[1].min() < 0 or rnd_h[1].max() >= H):
        raise ValueError("valid_idx or round_coord out of range")
    img = _as_cuda_exact(image, torch.uint8, dev, "image", (H, W, 3))
    dep = _as_cuda_exact(depth, torch.float32, dev, "depth", (H, W))
    M = int((mask_h != 1).sum())
    f32 = pts_h.dtype == np.float32
    p = torch.from_numpy(np.ascontiguousarray(pts_h)).to(dev)
    m2 = torch.from_numpy(np.ascontiguousarray(mask_h.astype(np.int32))).to(dev)
    vi = torch.from_numpy(valid_h.astype(np.int32)).to(dev)
    co = torch.from_numpy(np.ascontiguousarray(coords_h)).to(dev)
    rc = torch.from_numpy(np.ascontiguousarray(rnd_h)).to(dev)
    mats = grow_matrices(R, T, K)
    b = C.c_uint64()
    _check(lib().gspcd_grow_scratch_bytes(nv, H, W, C.byref(b)), "gspcd_grow_scratch_bytes")
    scratch = torch.empty(b.value, dtype=torch.uint8, device=dev)
    new_pts = torch.empty((3, max(M, 1)), dtype=torch.float64, device=dev)
    new_cols = torch.empty((max(M, 1), 3), dtype=torch.float32, device=dev)
    new_depth = torch.empty(max(M, 1), dtype=torch.float64, device=dev)
    border = torch.empty(max(nv, 1), dtype=torch.int32, device=dev)
    small = torch.zeros(2, dtype=torch.int32, device=dev)           # n_border, status
    _check(lib().gspcd_grow_view(p.data_ptr(), n, int(f32), vi.data_ptr(), co.data_ptr(), rc.data_ptr(), nv,
                                 m2.data_ptr(), dep.data_ptr(), img.data_ptr(), H, W, mats.ctypes.data, M,
                                 new_pts.data_ptr(), new_cols.data_ptr(), new_depth.data_ptr(), border.data_ptr(),
                                 small.data_ptr(), small.data_ptr() + 4, scratch.data_ptr(), scratch.numel(),
                                 _stream(dev)), "gspcd_grow_view")
    n_border, status = small.cpu().tolist()
    if status:
        raise RuntimeError(f"gspcd_grow_view: status {status} (exact predicate precision or walk cap exceeded)")
    out_pts = np.concatenate((pts_h, new_pts[:, :M].cpu().numpy()), axis=-1)
    out_cols = np.concatenate((cols_h, new_cols[:M].cpu().numpy()), axis=0)
    if not return_details:
        return out_pts, out_cols
    return out_pts, out_cols, border[:n_border].cpu().numpy().astype(np.int64), new_depth[:M].cpu().numpy()
