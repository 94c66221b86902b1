"""Inputs of the cases in tests/golden/grow_golden.json, rebuilt without the reference: the seeded cloud, the warp's
outputs from the warp's host restatement (tests/pcd_host.py) and the seeded model stand-ins of tests/grow_host.py."""
from __future__ import annotations

import json
import os

import numpy as np

import grow_host
import pcd_cases
import pcd_host

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = json.load(open(os.path.join(ROOT, "tests", "golden", "grow_golden.json")))


def warp(pts, cols, R, T, K, H, W):
    """warp_view_host, or warp_view's outputs for a view with no valid point (where griddata raises)."""
    if pcd_host._project(pts, R, T, K, H, W)[0].size == 0:
        return (np.zeros((H, W, 3)), np.zeros((H, W), np.int64), np.zeros(0, np.int64), np.zeros((2, 0)),
                np.zeros((2, 0), np.int32))
    return pcd_host.warp_view_host(pts, cols, R, T, K, H, W)


def golden_cases():
    """Yields (case record, inputs dict for grow_view_host / pcd.grow_view) in the golden's order; a grown cloud is
    the host restatement's result for the case it names."""
    H, W, K = GOLDEN["H"], GOLDEN["W"], np.array(GOLDEN["K"], np.float32)
    grown = {}
    for c in GOLDEN["cases"]:
        if c["cloud"] == "depth":
            pts, cols = pcd_cases.depth_cloud(GOLDEN["depth_cloud_seed"], H, W)
        elif c["cloud"] == "sparse":
            pts, cols = grow_host.sparse_cloud(GOLDEN["sparse_cloud_seed"], H, W)
        else:
            pts, cols = grown[c["cloud"].split(":")[1]]
        P = np.array(c["pose"])
        R, T = P[:, :3], P[:, 3:]
        _, mask2, valid, coords, rnd = warp(pts, cols, R, T, K, H, W)
        inp = dict(pts=pts, colors=cols, R=R, T=T, K=K, mask2=mask2, valid_idx=valid, coords=coords, rnd=rnd,
                   image=grow_host.stub_image(c["image_seed"], H, W),
                   depth=grow_host.stub_depth(c["depth_seed"], H, W, c["zero_rows"]))
        out = grow_host.grow_view_host(**inp)
        grown[c["name"]] = out[:2]
        yield c, inp, out
