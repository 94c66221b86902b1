"""Build LucidDreamer's training scene with its camera images made on the device (include/gsscene.h).

`build_scene(traindata, gaussians, opt, presetdata, frames=None)` does what the reference's
`Scene(traindata, gaussians, opt)` does and returns an object with its interface (`train_cameras`,
`preset_cameras`, `cameras_extent`, `gaussians`, `getTrainCameras()`, `getPresetCameras(preset)`):

- every training frame becomes a camera with the attributes, values, dtypes and devices `Camera.__init__` gives it.
  The composited `original_image` and the `canny_mask` of all frames come from one device call, where the reference
  composites each frame in numpy and runs `cv2.Canny` on the host;
- every frame of every preset path becomes a `MiniCam`-like camera, as `loadCameraPreset` makes it;
- `random.shuffle` runs once on the training cameras, `cameras_extent` follows `getNerfppNorm`, and the Gaussians
  are created from the point cloud and set up for training in the reference's order.

The rotations, translations and view matrices come from the reference's numpy expressions on the host. The matrices
of all cameras go to the device in one copy; `full_proj_transform` is one batched `bmm` and `camera_center` one
batched `torch.inverse`, each bit-identical on the GPU to the per-camera call the reference makes (the GPU tests
check both). Every per-camera tensor is a view into a buffer shared by the scene's cameras.

`presetdata` is `utils.trajectory.get_camerapaths()`'s output. `frames`, when given, is the uint8 CUDA tensor
[F, H, W, 3 or 4] of the training frames, such as `pcd.align_frames(..., on_device=True)` returns; otherwise the
PIL images in `traindata["frames"]` are converted to RGBA, stacked and uploaded in one copy.
"""
from __future__ import annotations

import ctypes as C
import math
import os
import random
from typing import NamedTuple

import numpy as np
import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "scene_csrc", "libgsscene.so")

GSSCENE_OK = 0
_P = C.c_void_p
SYMBOLS = [
    ("gsscene_abi_version", C.c_int, []),
    ("gsscene_scratch_bytes", C.c_int, [C.c_int32, C.c_int32, C.c_int32, C.POINTER(C.c_uint64)]),
    ("gsscene_camera_images", C.c_int, [_P, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, _P, _P, _P,
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
    if rc != GSSCENE_OK:
        raise RuntimeError(f"{what} failed with code {rc}")


def camera_images(frames: torch.Tensor, white_background: bool):
    """(original_image [F, 3, H, W], canny_mask [F, H, W]) float32 of uint8 CUDA frames [F, H, W, 3 or 4]."""
    if not isinstance(frames, torch.Tensor) or not frames.is_cuda or frames.dtype != torch.uint8:
        raise TypeError("frames must be a uint8 CUDA tensor")
    if frames.dim() != 4 or frames.shape[-1] not in (3, 4):
        raise ValueError(f"frames must be [F, H, W, 3 or 4], got {tuple(frames.shape)}")
    F, H, W, Ch = frames.shape
    dev = frames.device
    with torch.cuda.device(dev):
        frames = frames.contiguous()
        b = C.c_uint64()
        _check(lib().gsscene_scratch_bytes(F, H, W, C.byref(b)), "gsscene_scratch_bytes")
        scratch = torch.empty(b.value, dtype=torch.uint8, device=dev)
        image = torch.empty((F, 3, H, W), dtype=torch.float32, device=dev)
        canny = torch.empty((F, H, W), dtype=torch.float32, device=dev)
        _check(lib().gsscene_camera_images(frames.data_ptr(), F, H, W, Ch, int(bool(white_background)),
                                           image.data_ptr(), canny.data_ptr(), scratch.data_ptr(), scratch.numel(),
                                           C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)),
               "gsscene_camera_images")
    return image, canny


# ---- host matrices: the reference's numpy / torch expressions (utils/graphics.py, scene/dataset_readers.py)

def rotation_translation(transform_matrix):
    """R (stored transposed) and T of a NeRF camera-to-world matrix, as loadCamerasFromData forms them."""
    c2w = np.array(transform_matrix)
    c2w[:3, 1:3] *= -1                                   # OpenGL / Blender axes -> COLMAP
    w2c = np.linalg.inv(c2w)
    return np.transpose(w2c[:3, :3]), w2c[:3, 3]


def world_to_view(R, t, translate=np.array([.0, .0, .0]), scale=1.0) -> np.ndarray:
    """getWorld2View2: the float32 world-to-view matrix, through the camera-to-world inverse and back."""
    Rt = np.zeros((4, 4))
    Rt[:3, :3] = R.transpose()
    Rt[:3, 3] = t
    Rt[3, 3] = 1.0
    C2W = np.linalg.inv(Rt)
    C2W[:3, 3] = (C2W[:3, 3] + translate) * scale
    return np.float32(np.linalg.inv(C2W))


def projection(znear, zfar, fovX, fovY) -> np.ndarray:
    """getProjectionMatrix as float32 (its entries are rounded from Python floats on assignment)."""
    top = math.tan(fovY / 2) * znear
    right = math.tan(fovX / 2) * znear
    bottom, left = -top, -right
    P = np.zeros((4, 4), np.float32)
    P[0, 0] = 2.0 * znear / (right - left)
    P[1, 1] = 2.0 * znear / (top - bottom)
    P[0, 2] = (right + left) / (right - left)
    P[1, 2] = (top + bottom) / (top - bottom)
    P[3, 2] = 1.0
    P[2, 2] = 1.0 * zfar / (zfar - znear)
    P[2, 3] = -(zfar * znear) / (zfar - znear)
    return P


def fov2focal(fov, pixels):
    return pixels / (2 * math.tan(fov / 2))


def focal2fov(focal, pixels):
    return 2 * math.atan(pixels / (2 * focal))


def nerfpp_radius(cameras):
    """getNerfppNorm's radius over the cameras' (R, T), in their order."""
    centers = np.hstack([np.linalg.inv(world_to_view(c.R, c.T))[:3, 3:4] for c in cameras])
    center = np.mean(centers, axis=1, keepdims=True)
    dist = np.linalg.norm(centers - center, axis=0, keepdims=True)
    return np.max(dist) * 1.1


# ---- cameras

_TRANS = np.array([0.0, 0.0, 0.0])                       # Camera's default `trans`, one object shared by all


class TrainCamera:
    """The attributes the reference's `Camera.__init__` sets, its tensors views into the scene's buffers."""

    def __init__(self, idx, R, T, FoVx, FoVy, original_image, canny_mask, world_view_transform, projection_matrix,
                 full_proj_transform, camera_center):
        self.uid = idx
        self.colmap_id = idx
        self.R = R
        self.T = T
        self.FoVx = FoVx
        self.FoVy = FoVy
        self.image_name = ''
        self.data_device = torch.device("cuda")
        self.original_image = original_image
        self.canny_mask = canny_mask
        self.image_width = original_image.shape[2]
        self.image_height = original_image.shape[1]
        self.zfar = 100.0
        self.znear = 0.01
        self.trans = _TRANS
        self.scale = 1.0
        self.world_view_transform = world_view_transform
        self.projection_matrix = projection_matrix
        self.full_proj_transform = full_proj_transform
        self.camera_center = camera_center


class PresetCamera:
    """The attributes of the reference's `MiniCam`."""

    def __init__(self, width, height, fovy, fovx, znear, zfar, world_view_transform, full_proj_transform,
                 camera_center):
        self.image_width = width
        self.image_height = height
        self.FoVy = fovy
        self.FoVx = fovx
        self.znear = znear
        self.zfar = zfar
        self.world_view_transform = world_view_transform
        self.full_proj_transform = full_proj_transform
        self.camera_center = camera_center


class PointCloud(NamedTuple):
    """What `create_from_pcd` reads of the reference's BasicPointCloud."""
    points: np.ndarray
    colors: np.ndarray
    normals: np.ndarray


class Scene:
    """The reference Scene's interface over cameras built by `build_scene`."""

    def __init__(self, gaussians, train_cameras, preset_cameras, cameras_extent):
        self.gaussians = gaussians
        self.train_cameras = train_cameras
        self.preset_cameras = preset_cameras
        self.cameras_extent = cameras_extent

    def getTrainCameras(self):
        return self.train_cameras

    def getPresetCameras(self, preset):
        assert preset in self.preset_cameras
        return self.preset_cameras[preset]


def _pil_frames(traindata) -> np.ndarray:
    images = [np.array(f["image"].convert("RGBA")) for f in traindata["frames"]]
    if not images:
        raise ValueError("traindata has no frames")
    shapes = {im.shape for im in images}
    if len(shapes) != 1:
        raise ValueError(f"training frames differ in size: {sorted(shapes)}")
    return np.stack(images)


def build_scene(traindata, gaussians, opt, presetdata, frames=None) -> Scene:
    """The reference's `Scene(traindata, gaussians, opt)` with `readDataInfo`'s preset paths `presetdata`
    (`get_camerapaths()`), the camera images made on the device. See the module docstring."""
    n_frames = len(traindata["frames"])
    if frames is None:
        host = _pil_frames(traindata)
        frames = torch.from_numpy(host).cuda()
    elif not isinstance(frames, torch.Tensor) or not frames.is_cuda or frames.dtype != torch.uint8 or \
            frames.dim() != 4 or frames.shape[0] != n_frames:
        raise ValueError(f"frames must be a uint8 CUDA tensor [{n_frames}, H, W, 3 or 4]")
    F, H, W = frames.shape[:3]
    dev = frames.device
    images, canny = camera_images(frames, opt.white_background)

    fovx = traindata["camera_angle_x"]
    fovy = focal2fov(fov2focal(fovx, H), W)              # loadCamerasFromData's order: H for the focal, W for the fov
    pose = [rotation_translation(f["transform_matrix"]) for f in traindata["frames"]]
    wv = [world_to_view(R, T, _TRANS, 1.0) for R, T in pose]
    pr = [projection(0.01, 100.0, fovx, fovy)] * F

    pfovx = fovx * 1.2
    pfovy = focal2fov(fov2focal(pfovx, W), H)
    keys = list(presetdata)
    for k in keys:
        for f in presetdata[k]["frames"]:
            R, T = rotation_translation(f["transform_matrix"])
            wv.append(world_to_view(R, T, np.array([0.0, 0.0, 0.0]), 1.0))
    pr += [projection(0.01, 100, pfovx, pfovy)] * (len(wv) - F)

    # one copy each; the per-camera matrices are the transposed views the reference's .transpose(0, 1) makes
    wv_dev = torch.from_numpy(np.stack(wv)).to(dev).transpose(1, 2)
    pr_dev = torch.from_numpy(np.stack(pr)).to(dev).transpose(1, 2)
    full = torch.bmm(wv_dev, pr_dev)
    center = torch.inverse(wv_dev)[:, 3, :3]

    train = [TrainCamera(i, R, T, fovx, fovy, images[i], canny[i], wv_dev[i], pr_dev[i], full[i], center[i])
             for i, (R, T) in enumerate(pose)]
    presets, at = {}, F
    for k in keys:
        n = len(presetdata[k]["frames"])
        presets[k] = [PresetCamera(W, H, pfovy, pfovx, 0.01, 100, wv_dev[j], full[j], center[j])
                      for j in range(at, at + n)]
        at += n

    extent = nerfpp_radius(train)
    random.shuffle(train)
    pcd = PointCloud(points=traindata["pcd_points"].T, colors=traindata["pcd_colors"], normals=None)
    gaussians.create_from_pcd(pcd, extent)
    gaussians.training_setup(opt)
    return Scene(gaussians, train, presets, extent)
