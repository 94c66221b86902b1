"""Writes pcd_golden.json: digests of the reference's own warp loops (LucidDreamer.generate_pcd) on seeded clouds.

Run from the repository root with the reference checkout at REF (default /root/reference). The loop bodies are
taken from luciddreamer.py with `ast` and executed as they are; the poses come from the reference's
utils/trajectory.py and are stored in the JSON, so the tests that read it need no reference checkout.
Cases: a 128x96 depth-map cloud plus random extra points, the first three `rotate360` generation poses times the
five hemisphere views (aligning stage), and the dreaming stage's warp into two seeded random poses.
"""
import ast
import hashlib
import json
import os
import sys

import numpy as np
from PIL import Image
from scipy.interpolate import griddata as interp_grid
from scipy.ndimage import maximum_filter, minimum_filter

REF = os.environ.get("REF", "/root/reference")
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, REF)
import pcd_cases  # noqa: E402
from utils.trajectory import get_pcdGenPoses  # noqa: E402


def sha(a):
    a = np.ascontiguousarray(a)
    return {"shape": list(a.shape), "dtype": str(a.dtype), "sha256": hashlib.sha256(a.tobytes()).hexdigest()}


def loops():
    tree = ast.parse(open(os.path.join(REF, "luciddreamer.py")).read())
    fn = next(n for n in ast.walk(tree) if isinstance(n, ast.FunctionDef) and n.name == "generate_pcd")
    fors = [n for n in ast.walk(fn) if isinstance(n, ast.For)]
    dream = next(f for f in fors if ast.unparse(f.iter) == "iterable_dream")
    align = next(f for f in fors if ast.unparse(f.iter) == "iterable_align")
    # dreaming: the body up to and including the final masking of image2 (the warp; the diffusion follows)
    body = []
    for st in dream.body:
        if isinstance(st, ast.Assign) and ast.unparse(st.targets[0]) == "mask_hf":
            break
        body.append(st)
    dream_code = compile(ast.Module(body=body, type_ignores=[]), "luciddreamer.py:dream", "exec")
    inner = align.body[0]
    assert isinstance(inner, ast.For)
    align_code = compile(ast.Module(body=[inner], type_ignores=[]), "luciddreamer.py:align", "exec")
    return dream_code, align_code


def main():
    dream_code, align_code = loops()
    H, W = 96, 128
    pts, cols = pcd_cases.depth_cloud(7, H, W, extra=3000)
    K = pcd_cases.intrinsics(H, W)
    render_poses = get_pcdGenPoses("rotate360")[:3]
    internel_render_poses = get_pcdGenPoses("hemisphere", {"center_depth": 2.0})
    edgeN = 2
    edgemask = np.pad(np.ones((H - 2 * edgeN, W - 2 * edgeN)), ((edgeN, edgeN), (edgeN, edgeN)))
    base = dict(np=np, interp_grid=interp_grid, maximum_filter=maximum_filter, minimum_filter=minimum_filter,
                Image=Image, H=H, W=W, K=K, edgemask=edgemask, print=lambda *a, **k: None,
                yz_reverse=np.array([[1, 0, 0], [0, -1, 0], [0, 0, -1]]))
    out = {"H": H, "W": W, "cloud": {"seed": 7, "extra": 3000}, "K": K.tolist(),
           "render_poses": render_poses.tolist(), "internal_poses": internel_render_poses.tolist()}

    frames = []
    for i in range(len(render_poses)):
        ns = dict(base, i=i, render_poses=render_poses, internel_render_poses=internel_render_poses,
                  pts_coord_world=pts, pts_colors=cols, traindata={"frames": []})
        exec(align_code, ns)
        for fr in ns["traindata"]["frames"]:
            frames.append({"image": sha(np.array(fr["image"])), "transform_matrix": fr["transform_matrix"]})
    out["align_frames"] = frames

    dream = []
    dream_poses = np.zeros((3, 3, 4))
    dream_poses[0, :, :3] = np.eye(3)
    for i in (1, 2):
        R, T = pcd_cases.random_pose(i)
        dream_poses[i, :, :3], dream_poses[i, :, 3:] = R, T
    out["dream_poses"] = dream_poses.tolist()
    for i in (1, 2):
        ns = dict(base, i=i, render_poses=dream_poses, pts_coord_world=pts, pts_colors=cols)
        exec(dream_code, ns)
        dream.append({"pose": i, "image2": sha(ns["image2"]), "mask2": sha(ns["mask2"]),
                      "valid_idx": sha(ns["valid_idx"]), "coords": sha(ns["pixel_coord_cam2"]),
                      "round": sha(ns["round_coord_cam2"])})
    out["dream"] = dream
    with open(os.path.join(HERE, "pcd_golden.json"), "w") as f:
        json.dump(out, f, indent=1)
    print(f"{len(frames)} frames, {len(dream)} dreaming views")


if __name__ == "__main__":
    main()
