"""Writes grow_golden.json: digests of the reference's own dreaming-loop body (LucidDreamer.generate_pcd), which grows
the point cloud from each inpainted view, on seeded clouds with seeded stand-ins for the two models.

Run from the repository root with the reference checkout at REF (default /root/reference). The loop body is taken
from luciddreamer.py with `ast` and executed as it is, the 100-step scale fit included, so that the recorded `sc`
and `trans3d` show what the fit leaves. `self.rgb` and `self.d` are `grow_host.stub_image` / `stub_depth`. The
poses are stored in the JSON, so the tests that read it need no reference checkout.

Cases at 128x96 (W x H), float32 K: view 1 on the float32 depth-map cloud; view 2 on the cloud view 1 grew; a view
whose depth is 0 on rows holding border points (a zero-length ray: NaN corrections, then the nearest fallback); a
sparse cloud with no border point; the identity view of the depth-map cloud, with no inpainted pixel; and a view
with no valid point. In the last one the reference's warp raises QhullError (griddata with no points), so that
case takes the warp's outputs as luciddreamer_b200.pcd.warp_view returns them there (an empty cloud in view, image
and mask all zero) and executes the reference from `mask_hf` on.
"""
import ast
import hashlib
import json
import os
import sys
import warnings

import numpy as np
import torch
from PIL import Image
from scipy.interpolate import griddata as interp_grid
from scipy.ndimage import maximum_filter, minimum_filter

REF = os.environ.get("REF", "/root/reference")
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
import grow_host  # noqa: E402
import pcd_cases  # noqa: E402
import pcd_host  # noqa: E402


def sha(a):
    a = np.ascontiguousarray(a)
    return {"shape": list(a.shape), "dtype": str(a.dtype), "sha256": hashlib.sha256(a.tobytes()).hexdigest()}


def dream_body():
    tree = ast.parse(open(os.path.join(REF, "luciddreamer.py")).read())
    fn = next(n for n in ast.walk(tree) if isinstance(n, ast.FunctionDef) and n.name == "generate_pcd")
    dream = next(f for f in ast.walk(fn) if isinstance(f, ast.For) and ast.unparse(f.iter) == "iterable_dream")
    cut = next(k for k, st in enumerate(dream.body)
               if isinstance(st, ast.Assign) and ast.unparse(st.targets[0]) == "mask_hf")
    mk = lambda sts, name: compile(ast.Module(body=sts, type_ignores=[]), f"luciddreamer.py:{name}", "exec")
    return mk(dream.body[:cut], "warp"), mk(dream.body[cut:], "grow")


class Models:
    def __init__(self, H, W, image_seed, depth_seed, zero_rows):
        self.H, self.W, self.image_seed, self.depth_seed, self.zero_rows = H, W, image_seed, depth_seed, zero_rows

    def rgb(self, **kw):
        return Image.fromarray(grow_host.stub_image(self.image_seed, self.H, self.W))

    def d(self, image):
        return grow_host.stub_depth(self.depth_seed, self.H, self.W, self.zero_rows)


def pose(R, T):
    P = np.zeros((2, 3, 4))
    P[0, :, :3] = np.eye(3)
    P[1, :, :3], P[1, :, 3:] = R, np.asarray(T).reshape(3, 1)
    return P


def main():
    warp_code, grow_code = dream_body()
    H, W = 96, 128
    K = pcd_cases.intrinsics(H, W).astype(np.float32)
    edgeN = 2
    edgemask = np.pad(np.ones((H - 2 * edgeN, W - 2 * edgeN)), ((edgeN, edgeN), (edgeN, edgeN)))
    yaw = np.deg2rad(180.0)
    back = np.array([[np.cos(yaw), 0, np.sin(yaw)], [0, 1, 0], [-np.sin(yaw), 0, np.cos(yaw)]])
    cases = [
        dict(name="view1", cloud="depth", pose=pose(*pcd_cases.random_pose(1))[1], image_seed=11, depth_seed=12),
        dict(name="view2", cloud="grown:view1", pose=pose(*pcd_cases.random_pose(2))[1], image_seed=21,
             depth_seed=22),
        dict(name="zero_depth", cloud="depth", pose=pose(pcd_cases.random_pose(3)[0], np.zeros(3))[1], image_seed=31,
             depth_seed=32, zero_rows=list(range(2, 94, 4))),
        dict(name="no_border", cloud="sparse", pose=pose(np.eye(3), np.zeros(3))[1], image_seed=41, depth_seed=42),
        dict(name="no_inpainted", cloud="depth", pose=pose(np.eye(3), np.zeros(3))[1], image_seed=51, depth_seed=52),
        dict(name="no_valid", cloud="depth", pose=pose(back, np.zeros(3))[1], image_seed=61, depth_seed=62),
    ]
    grown = {}
    out = {"H": H, "W": W, "K": K.tolist(), "depth_cloud_seed": 7, "sparse_cloud_seed": 8, "cases": []}
    for c in cases:
        if c["cloud"] == "depth":
            pts, cols = pcd_cases.depth_cloud(7, H, W)
        elif c["cloud"] == "sparse":
            pts, cols = grow_host.sparse_cloud(8, H, W)
        else:
            pts, cols = grown[c["cloud"].split(":")[1]]
        P = np.zeros((2, 3, 4))
        P[0, :, :3] = np.eye(3)
        P[1] = c["pose"]
        ns = dict(np=np, torch=torch, interp_grid=interp_grid, maximum_filter=maximum_filter,
                  minimum_filter=minimum_filter, self=Models(H, W, c["image_seed"], c["depth_seed"],
                                                             c.get("zero_rows", [])),
                  i=1, render_poses=P, pts_coord_world=pts, pts_colors=cols, H=H, W=W, K=K, edgemask=edgemask,
                  prompt="", negative_prompt="", generator=None, diff_steps=1)
        warp_from_reference = True
        try:
            exec(warp_code, ns)
        except Exception as e:                     # scipy's QhullError: fewer than three valid points
            assert c["name"] == "no_valid", e
            warp_from_reference = False
            assert pcd_host._project(pts, P[1, :, :3], P[1, :, 3:], K, H, W)[0].size == 0
            img, mask = np.zeros((H, W, 3)), np.zeros((H, W), np.int64)
            valid, coords, rnd = np.zeros(0, np.int64), np.zeros((2, 0)), np.zeros((2, 0), np.int32)
            x, y = np.meshgrid(np.arange(W, dtype=np.float32), np.arange(H, dtype=np.float32), indexing='xy')
            ns.update(image2=img, mask2=mask, valid_idx=valid, pixel_coord_cam2=coords, round_coord_cam2=rnd, x=x, y=y)
        mask2, valid = ns["mask2"], ns["valid_idx"]
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            exec(grow_code, ns)
        new_depth_linear = ns.get("new_depth_linear", np.zeros(0))
        rec = {"name": c["name"], "cloud": c["cloud"], "pose": np.asarray(c["pose"]).tolist(),
               "image_seed": c["image_seed"], "depth_seed": c["depth_seed"], "zero_rows": c.get("zero_rows", []),
               "warp_from_reference": warp_from_reference,
               "n_valid": int(len(valid)), "n_border": int(len(ns["border_valid_idx"])),
               "n_inpainted": int((mask2 != 1).sum()), "n_linear_nan": int(np.isnan(new_depth_linear).sum()),
               "sc": float(ns["sc"].item()), "sc_grad_is_none": ns["sc"].grad is None,
               "trans3d": np.asarray(ns["trans3d"]).tolist(), "trans3d_dtype": str(np.asarray(ns["trans3d"]).dtype),
               "mask2": sha(mask2), "valid_idx": sha(valid), "border_valid_idx": sha(ns["border_valid_idx"]),
               "new_depth": sha(ns["new_depth"]), "pts_coord_world": sha(ns["pts_coord_world"]),
               "pts_colors": sha(ns["pts_colors"])}
        out["cases"].append(rec)
        grown[c["name"]] = (ns["pts_coord_world"], ns["pts_colors"])
        print({k: rec[k] for k in ("name", "n_valid", "n_border", "n_inpainted", "n_linear_nan", "sc")})
    with open(os.path.join(HERE, "grow_golden.json"), "w") as f:
        json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
