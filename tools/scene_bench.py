"""Times the training scene's construction (LucidDreamer.create's `Scene(traindata, gaussians, opt)`) on the current GPU.

LucidDreamer's shape: 512 x 512 frames, 50 of them from the aligning stage (ten generation poses 2 degrees apart times
the five hemisphere views, through pcd.align_frames), the three preset camera paths and a 1.77 M-point cloud. Alternating
the arms in every round:
  reference   the reference's own Scene, executed from the bytecode oracle/build_pyref_scene.py compiles
              (needs oracle/_ref/pyref_scene and cv2; reported as not measured without them);
  pil         scene.build_scene from the PIL frames in traindata;
  device      scene.build_scene from the uint8 CUDA frames of align_frames(..., on_device=True).
Every arm creates the reference's GaussianModel from the same cloud (create_from_pcd, training_setup), so the
difference between arms is the camera side. Each time ends in a device synchronise; the best and the median of the
rounds are printed as one JSON line, with the card's name and power limit.
"""
import json
import os
import random
import subprocess
import sys
import time
import types

import numpy as np
import torch
from PIL import Image

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import pcd_cases  # noqa: E402
from luciddreamer_b200 import pcd, scene  # noqa: E402

PYREF = os.path.join(ROOT, "oracle", "_ref", "pyref_scene")


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    except (OSError, subprocess.CalledProcessError):
        q = torch.cuda.get_device_name(0) + ", power limit unknown"
    return q


def reference():
    """(Scene, GaussianModel, GSParams, get_camerapaths) of the reference, or None with the reason."""
    if not os.path.exists(os.path.join(PYREF, "scene", "__init__.pyc")):
        return None, "oracle/_ref/pyref_scene not built"
    try:
        import cv2  # noqa: F401
    except ImportError:
        return None, "cv2 not installed"
    sys.path.insert(0, PYREF)
    ply = types.ModuleType("plyfile")
    ply.PlyData = ply.PlyElement = object
    sys.modules["plyfile"] = ply
    sys.modules["imageio"] = types.ModuleType("imageio")
    import arguments
    import scene as ref_scene
    from utils.trajectory import get_camerapaths
    # loadCamerasFromData makes `Image.fromarray(<int8 array>, "RGB")` only for its size; Pillow 12 refuses int8
    sys.modules["scene.dataset_readers"].Image = types.SimpleNamespace(
        fromarray=lambda a, mode=None: Image.fromarray(np.ascontiguousarray(a).view(np.uint8)))
    return (ref_scene.Scene, ref_scene.GaussianModel, arguments.GSParams, get_camerapaths), None


def main(rounds=5, n_points=1_770_000):
    if not torch.cuda.is_available():
        raise SystemExit("scene_bench needs a GPU")
    dev_name = card()
    ref, why = reference()
    if ref is None:
        raise SystemExit(f"scene_bench needs the reference's GaussianModel: {why}")
    Scene, GaussianModel, GSParams, get_camerapaths = ref
    H = W = 512
    K = pcd_cases.intrinsics(H, W)
    pts, cols = pcd_cases.depth_cloud(0, H, W, extra=n_points - H * W)
    pts = pts.astype(np.float64)
    rp, hemi = pcd_cases.rotate360(10, step_deg=2.0), pcd_cases.hemisphere(2.0)
    frames_t, mats = pcd.align_frames(pts, cols, rp, hemi, K, H, W, on_device=True)
    assert len(mats) == 50, len(mats)
    frames_h = frames_t.cpu().numpy()
    traindata = {"camera_angle_x": 2 * np.arctan(W / (2 * K[0, 0])), "W": W, "H": H, "pcd_points": pts,
                 "pcd_colors": cols,
                 "frames": [{"image": Image.fromarray(f), "transform_matrix": m.tolist()} for f, m in zip(frames_h, mats)]}
    opt = GSParams()
    presets = get_camerapaths()
    arms = {
        "reference": lambda: Scene(traindata, GaussianModel(opt.sh_degree), opt),
        "pil": lambda: scene.build_scene(traindata, GaussianModel(opt.sh_degree), opt, presets),
        "device": lambda: scene.build_scene(traindata, GaussianModel(opt.sh_degree), opt, presets, frames=frames_t),
    }
    times = {k: [] for k in arms}
    for r in range(rounds + 1):                                       # round 0 warms every arm up
        for name, make in arms.items():
            random.seed(r)
            torch.cuda.synchronize()
            t = time.perf_counter()
            sc = make()
            torch.cuda.synchronize()
            if r:
                times[name].append(time.perf_counter() - t)
            del sc
    out = {"what": "Scene construction", "H": H, "W": W, "frames": len(mats), "points": int(pts.shape[1]),
           "preset_cameras": sum(len(v["frames"]) for v in presets.values()), "rounds": rounds, "card": dev_name}
    for name, ts in times.items():
        out[f"{name}_best_s"] = min(ts)
        out[f"{name}_median_s"] = float(np.median(ts))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
