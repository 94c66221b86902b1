"""Times generate_pcd's aligning stage: the numpy/scipy restatement against luciddreamer_b200.pcd.align_frames,
alternating them, at LucidDreamer's shape (512x512, 10 rotate360 poses x 5 hemisphere views). Prints one JSON line
per cloud size with the card name and power limit.

    python tools/pcd_bench.py [--sizes 262144,1000000,2000000] [--host-views 2]

align_frames always runs the whole stage. The host restatement is timed on the first --host-views views that have
valid points (it takes seconds per view); its stage estimate is that per-view time times the number of views with
points, since the reference skips the other views at once."""
import argparse
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
import pcd_cases  # noqa: E402
import pcd_host  # noqa: E402
from luciddreamer_b200 import pcd  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    return q[0] if q else torch.cuda.get_device_name(0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="262144,1000000,2000000")
    ap.add_argument("--host-views", type=int, default=2)
    ap.add_argument("--reps", type=int, default=2)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "pcd_bench needs a GPU"
    H = W = 512
    K = pcd_cases.intrinsics(H, W)
    rp, hemi = pcd_cases.rotate360(10), pcd_cases.hemisphere(2.0)
    n_views = len(rp) * len(hemi)
    for n in (int(s) for s in a.sizes.split(",")):
        extra = max(n - H * W, 0)
        pts, cols = pcd_cases.depth_cloud(1, H, W, extra=extra)
        pts, cols = pts[:, :n], cols[:n]
        pcd.align_frames(pts, cols, rp[:1], hemi[:1], K, H, W)                  # warm-up
        views = pcd.compose_poses(rp, hemi)
        dev_ms, host_ms = [], []
        for _ in range(a.reps):
            torch.cuda.synchronize()
            t = time.perf_counter()
            frames, mats = pcd.align_frames(pts, cols, rp, hemi, K, H, W)
            torch.cuda.synchronize()
            dev_ms.append((time.perf_counter() - t) * 1e3)
            # the host on views that have points: the reference leaves the others at once
            kept = [k for k, v in enumerate(views) if any(np.array_equal(v[2], m) for m in mats)][:a.host_views]
            t = time.perf_counter()
            for k in kept:
                pcd_host.align_frames_host(pts, cols, rp[k // len(hemi):k // len(hemi) + 1],
                                           hemi[k % len(hemi):k % len(hemi) + 1], K, H, W)
            host_ms.append((time.perf_counter() - t) * 1e3 / max(len(kept), 1))
        d, h = min(dev_ms), min(host_ms)
        nk = len(frames)
        print(json.dumps({"points": n, "H": H, "W": W, "views": n_views, "views_with_points": nk,
                          "device_stage_ms": round(d, 1), "device_ms_per_view_with_points": round(d / max(nk, 1), 1),
                          "host_ms_per_view_with_points": round(h, 1),
                          "host_stage_ms_estimate": round(h * nk), "host_views_timed": len(kept),
                          "card": card()}), flush=True)


if __name__ == "__main__":
    main()
