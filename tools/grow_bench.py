"""Times the dreaming stage's growth of the cloud (pcd.grow_view) on the current GPU.

Per view at 512x512, with depth-map clouds of 0.26 M, 1 M and 2 M points and seeded stand-ins for the two models,
alternating the arms: grow_view on the device (synchronised), and the host restatement without the scale fit
(tests/grow_host.py). The reference's own body with its 100-step fit needs the reference checkout and is reported as
not measured here. Then a stub-model dreaming stage over the rotate360 poses with warp_view + grow_view.
Prints one JSON line per number, with the card's name and power limit.
"""
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import grow_host  # noqa: E402
import pcd_cases  # noqa: E402
from luciddreamer_b200 import pcd  # noqa: E402


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    except (OSError, subprocess.CalledProcessError):
        q = torch.cuda.get_device_name(0) + ", power limit unknown"
    return q


def main(reps=3):
    if not torch.cuda.is_available():
        raise SystemExit("grow_bench needs a GPU")
    dev_name = card()
    H = W = 512
    K = pcd_cases.intrinsics(H, W).astype(np.float32)
    for n in (262_144, 1_000_000, 2_000_000):
        pts, cols = pcd_cases.depth_cloud(0, H, W, extra=n - H * W)
        pts = pts.astype(np.float64)
        R, T = pcd_cases.random_pose(1)
        _, mask2, valid, coords, rnd = pcd.warp_view(pts, cols, R, T, K, H, W)
        inp = dict(pts=pts, colors=cols, R=R, T=T, K=K, mask2=mask2, valid_idx=valid, coords=coords, rnd=rnd,
                   image=grow_host.stub_image(2, H, W), depth=grow_host.stub_depth(3, H, W))
        args = [inp[k] for k in ("pts", "colors", "R", "T", "K", "mask2", "valid_idx", "coords", "rnd", "image",
                                 "depth")]
        pcd.grow_view(*args)                                           # warm-up
        dev_t, host_t = [], []
        for _ in range(reps):
            torch.cuda.synchronize()
            t = time.perf_counter()
            pcd.grow_view(*args)
            torch.cuda.synchronize()
            dev_t.append(time.perf_counter() - t)
            t = time.perf_counter()
            grow_host.grow_view_host(**inp)
            host_t.append(time.perf_counter() - t)
        print(json.dumps({"what": "grow_view per view", "H": H, "W": W, "points": n, "valid": int(len(valid)),
                          "inpainted": int((mask2 != 1).sum()), "device_s": min(dev_t), "host_restatement_s":
                          min(host_t), "reference_with_fit_s": "not measured", "card": dev_name}))
    # a stub-model dreaming stage over the rotate360 poses
    poses = pcd_cases.rotate360()
    pts, cols = pcd_cases.depth_cloud(0, H, W)
    torch.cuda.synchronize()
    t = time.perf_counter()
    for i in range(1, len(poses)):
        R, T = poses[i, :, :3], poses[i, :, 3:]
        _, mask2, valid, coords, rnd = pcd.warp_view(pts, cols, R, T, K, H, W)
        pts, cols = pcd.grow_view(pts, cols, R, T, K, mask2, valid, coords, rnd, grow_host.stub_image(i, H, W),
                                  grow_host.stub_depth(100 + i, H, W))
    torch.cuda.synchronize()
    print(json.dumps({"what": "dreaming stage, rotate360, warp_view + grow_view, stub models", "H": H, "W": W,
                      "views": len(poses) - 1, "final_points": int(pts.shape[1]), "total_s": time.perf_counter() - t,
                      "card": dev_name}))


if __name__ == "__main__":
    main()
