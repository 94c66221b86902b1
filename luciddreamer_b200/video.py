"""Batched video-render path (SURVEY.md 8f-4): the forward-only consumer of the rasterizer.

`render_video_frames` does what the loop of LucidDreamer.render_video does per view (luciddreamer.py:250-262) --
render, colour -> uint8 HWC, depth -> -(depth * (depth > 0)), running dmin/dmax -- but keeps every frame on the
device (gs_pack_frame writes into slot k of a batch buffer on the render stream) and copies the whole clip to pinned
host memory ONCE.  The reference pays two blocking float D2H copies (16 B/pixel) and a stream sync per frame.

`load_json` restates utils/camera.py:24-52 (the preset camera files under cameras/*.json), including its
MiniCam(W, H, FoVx, FoVy, ...) argument-order quirk (see synthetic.make_camera).
`colorize` restates utils/depth.py:7-62 for the host side of the depth video; `colorize_frames` does the same for a whole
clip on the device (gs_colorize_depth), and `render_video_frames(..., depth_rgba=True)` returns the coloured clip."""
from __future__ import annotations

import inspect
import json
from typing import Optional, Sequence

import numpy as np
import torch

from . import _native as N
from . import rasterizer as R
from . import synthetic as syn


def load_json(path: str, H: int, W: int):
    """[CameraView] for every frame of a preset file (utils/camera.py:24-52): NeRF c2w -> COLMAP axes -> w2c."""
    with open(path) as fh:
        contents = json.load(fh)
    fovx = contents["camera_angle_x"]
    return [syn.make_camera(W, H, c2w=syn.nerf_c2w_to_colmap(np.array(fr["transform_matrix"])), fovx=fovx,
                            swap_fov_like_load_json=True) for fr in contents["frames"]]


def pack_frame(color: torch.Tensor, depth: Optional[torch.Tensor], rgb8: torch.Tensor, neg_depth: Optional[torch.Tensor],
               minmax_state: Optional[torch.Tensor]) -> None:
    """One frame through gs_pack_frame on the current stream (outputs are views into batch buffers)."""
    if not color.is_cuda:
        raise RuntimeError("pack_frame: CUDA tensors only (no CPU fallback)")
    _, H, W = color.shape
    idx = color.device.index
    with R._guard(idx):
        N.check(N.lib().gs_pack_frame(R._ctx(idx), H, W, color.data_ptr(), depth.data_ptr() if depth is not None else None,
                                      rgb8.data_ptr(), neg_depth.data_ptr() if neg_depth is not None else None,
                                      minmax_state.data_ptr() if minmax_state is not None else None,
                                      R._raw_stream(idx)))


def colorize_frames(neg_depth: torch.Tensor):
    """`colorize` for every frame of a clip, on the device (gs_colorize_depth), on the current stream without a host sync.

    neg_depth: [F,H,W] float32 CUDA tensor (e.g. the depths render_video_frames packs).  Returns (rgba uint8 [F,H,W,4],
    vminmax float32 [F,2]) on the same device: frame k of `rgba` is bit-identical to `colorize(neg_depth[k])`, and
    vminmax[k] holds its (2nd, 98th) percentiles.  A frame without a valid pixel (where `colorize` raises) comes out as
    background with NaN percentiles.  invalid_val and the background colour are `colorize`'s defaults."""
    if not isinstance(neg_depth, torch.Tensor) or neg_depth.dtype != torch.float32 or neg_depth.dim() != 3:
        raise ValueError("colorize_frames: expected a float32 [F,H,W] tensor, got "
                         f"{getattr(neg_depth, 'dtype', type(neg_depth))} {tuple(getattr(neg_depth, 'shape', ()))}")
    if not neg_depth.is_cuda:
        raise RuntimeError("colorize_frames: CUDA tensors only (no CPU fallback)")
    value = neg_depth.contiguous()
    F, H, W = value.shape
    dev = value.device
    rgba = torch.empty((F, H, W, 4), dtype=torch.uint8, device=dev)
    vminmax = torch.empty((F, 2), dtype=torch.float32, device=dev)
    if value.numel() == 0:
        return rgba, vminmax.fill_(float("nan"))
    idx = dev.index
    lut = _device_lut(dev)
    L = N.lib()
    scratch = torch.empty(L.gs_colorize_scratch_bytes(F), dtype=torch.uint8, device=dev)
    with R._guard(idx):
        N.check(L.gs_colorize_depth(R._ctx(idx), F, H, W, value.data_ptr(), float(_INVALID_VAL), lut.data_ptr(),
                                    _BACKGROUND_RGBA, scratch.data_ptr(), scratch.numel(), rgba.data_ptr(),
                                    vminmax.data_ptr(), R._raw_stream(idx)))
    return rgba, vminmax


def render_video_frames(params: dict, settings_list: Sequence, rank: int = 0, world: int = 1, with_depth: bool = True,
                        depth_rgba: bool = False):
    """Renders this rank's share (views rank, rank+world, ...) of `settings_list`.

    params: dict(means3D, shs, opacities, scales, rotations) of CUDA tensors (activated values, as render() passes them).
    Returns (frames uint8 [F,H,W,3] numpy, depths float32 [F,H,W] numpy or None, dmin, dmax, view_indices) with the
    semantics of framelist / depthlist / dmin / dmax in luciddreamer.py:241-262.  One host copy for the whole clip.
    depth_rgba=True: the depths are colour-mapped on the device before that copy (`colorize_frames`, one call for the
    clip), and the second element is the coloured depth clip, uint8 [F,H,W,4] -- what luciddreamer.py:267 makes of
    depthlist."""
    if depth_rgba and not with_depth:
        raise ValueError("render_video_frames: depth_rgba=True needs with_depth=True")
    from .multiview import shard_views
    views = shard_views(len(settings_list), rank, world)
    dev = params["means3D"].device
    if not views:
        return np.zeros((0, 0, 0, 3), np.uint8), None, 1e8, -1e8, views
    H, W = settings_list[views[0]].image_height, settings_list[views[0]].image_width
    F = len(views)
    rgb8 = torch.empty((F, H, W, 3), dtype=torch.uint8, device=dev)
    negd = torch.empty((F, H, W), dtype=torch.float32, device=dev) if with_depth else None
    state = torch.tensor([-1, 0], dtype=torch.int32, device=dev)   # bits {0xffffffff, 0} if with_depth else None
    e = torch.empty(0)
    with torch.no_grad():
        for k, v in enumerate(views):
            rs = settings_list[v]
            if (rs.image_height, rs.image_width) != (H, W):
                raise RuntimeError("render_video_frames: all views of a clip must share one resolution")
            color, _radii, depth = R.GaussianRasterizer(rs)(params["means3D"], e, params["opacities"], shs=params["shs"],
                                                            scales=params["scales"], rotations=params["rotations"])
            pack_frame(color, depth if with_depth else None, rgb8[k], negd[k] if with_depth else None, state)
    h_rgb = torch.empty((F, H, W, 3), dtype=torch.uint8, pin_memory=True)
    h_rgb.copy_(rgb8, non_blocking=True)
    dmin, dmax, h_d = 1e8, -1e8, None
    if with_depth:
        mm = torch.empty(2, dtype=torch.float32, device=dev)
        idx = dev.index
        with R._guard(idx):
            N.check(N.lib().gs_minmax_read(R._ctx(idx), state.data_ptr(), mm.data_ptr(), R._raw_stream(idx)))
        if depth_rgba:
            d_rgba, _ = colorize_frames(negd)
            h_d = torch.empty((F, H, W, 4), dtype=torch.uint8, pin_memory=True)
            h_d.copy_(d_rgba, non_blocking=True)
        else:
            h_d = torch.empty((F, H, W), dtype=torch.float32, pin_memory=True)
            h_d.copy_(negd, non_blocking=True)
        h_mm = torch.empty(2, dtype=torch.float32, pin_memory=True)
        h_mm.copy_(mm, non_blocking=True)
    torch.cuda.current_stream(dev).synchronize()
    if with_depth:
        dmin, dmax = min(dmin, float(h_mm[0])), max(dmax, float(h_mm[1]))
    return h_rgb.numpy(), (h_d.numpy() if with_depth else None), dmin, dmax, views


# ------------------------------------------------------------------------------------------------ host side: colorize

_JET = {  # matplotlib's `jet` segment data (x, y0, y1) -- published colormap definition (matplotlib/_cm.py: _jet_data)
    "red": ((0.00, 0, 0), (0.35, 0, 0), (0.66, 1, 1), (0.89, 1, 1), (1.00, 0.5, 0.5)),
    "green": ((0.000, 0, 0), (0.125, 0, 0), (0.375, 1, 1), (0.640, 1, 1), (0.910, 0, 0), (1.000, 0, 0)),
    "blue": ((0.00, 0.5, 0.5), (0.11, 1, 1), (0.34, 1, 1), (0.65, 0, 0), (1.00, 0, 0)),
}


def _segment_lut(data, n=256):
    """matplotlib.colors._create_lookup_table for segment data: piecewise-linear interpolation sampled at n points."""
    a = np.array(data, dtype=float)
    x, y0, y1 = a[:, 0] * (n - 1), a[:, 1], a[:, 2]
    xi = np.linspace(0, n - 1, n)
    ind = np.searchsorted(x, xi)[1:-1]
    dist = (xi[1:-1] - x[ind - 1]) / (x[ind] - x[ind - 1])
    return np.clip(np.concatenate([[y1[0]], dist * (y0[ind] - y1[ind - 1]) + y1[ind - 1], [y0[-1]]]), 0.0, 1.0)


_JET_LUT = None


def jet_lut() -> np.ndarray:
    global _JET_LUT
    if _JET_LUT is None:
        rgb = np.stack([_segment_lut(_JET[c]) for c in ("red", "green", "blue")], 1)
        _JET_LUT = (np.concatenate([rgb, np.ones((256, 1))], 1) * 255).astype(np.uint8)      # bytes=True: truncation
    return _JET_LUT


def colorize(value, vmin=None, vmax=None, invalid_val=-99, invalid_mask=None, background_color=(128, 128, 128, 255)):
    """utils/depth.py:7-62 with cmap='jet': percentile-normalised depth -> uint8 RGBA [H,W,4].

    PARITY UNPINNED: matplotlib is not available in the build image, so the colormap table is restated from its
    published segment data and could not be checked against `matplotlib.cm.get_cmap('jet')(x, bytes=True)`."""
    value = np.asarray(value.detach().cpu().numpy() if isinstance(value, torch.Tensor) else value).squeeze()
    if invalid_mask is None:
        invalid_mask = value == invalid_val
    mask = np.logical_not(invalid_mask)
    vmin = np.percentile(value[mask], 2) if vmin is None else vmin
    vmax = np.percentile(value[mask], 98) if vmax is None else vmax
    value = (value - vmin) / (vmax - vmin) if vmin != vmax else value * 0.0
    x = np.array(value, dtype=float)
    idx = (x * 256).astype(np.int64, copy=False)
    idx[x * 256 == 256] = 255                       # matplotlib maps exactly 1.0 into the last bin
    idx = np.clip(idx, 0, 255)
    idx[x < 0] = 0                                  # under -> first colour, over -> last colour (no set_under/over)
    idx[x > 1] = 255
    img = jet_lut()[idx]
    img[invalid_mask] = background_color
    return img


# ------------------------------------------------------------------------------------------------ device side: colorize
_COLORIZE_DEFAULTS = inspect.signature(colorize).parameters
_INVALID_VAL = _COLORIZE_DEFAULTS["invalid_val"].default
_BACKGROUND_RGBA = int.from_bytes(bytes(_COLORIZE_DEFAULTS["background_color"].default), "little")   # R | G<<8 | B<<16 | A<<24
_LUT_ON_DEVICE = {}


def _device_lut(dev: torch.device) -> torch.Tensor:
    """jet_lut() as a [256,4] uint8 tensor on `dev`, copied once per device."""
    t = _LUT_ON_DEVICE.get(dev.index)
    if t is None:
        if torch.cuda.is_current_stream_capturing():
            raise RuntimeError("colorize_frames: call it once on this device before capturing a CUDA graph "
                               "(the colour table is copied to the device on first use)")
        t = _LUT_ON_DEVICE[dev.index] = torch.from_numpy(jet_lut().copy()).to(dev)
    return t
