"""Times the video-render path (BASELINE config 4 shape: forward-only view batch at 1080p, 1 M Gaussians):
  ours      = luciddreamer_b200.video.render_video_frames (device-side packing, one host copy per clip)
  reference = the reference rasterizer (oracle/_ref) driven by the per-frame loop of luciddreamer.py:250-262
              (two blocking float D2H copies + numpy per frame).
and, under "colour", the depth video's colour mapping (colour_rows): device vs host, on the same clip.
Usage (GPU box): python tools/video_bench.py [frames]"""
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from luciddreamer_b200 import GaussianRasterizationSettings, synthetic as syn, video


def run(F=48, impls=("ours", "reference")):
    ref_cuda = None
    if "reference" in impls:
        from oracle import ref_cuda          # the reference rasterizer (oracle/_ref), only when asked for
    d = torch.device("cuda:0")
    c = syn.CONFIGS[3]
    P, W, H = c["P"], c["W"], c["H"]
    sc = {k: v.to(d) for k, v in syn.make_scene(P, 1003).items()}
    poses = syn.rotate360_poses(F)
    cams = [syn.make_camera(W, H, c2w=poses[k]) for k in range(F)]
    settings = [GaussianRasterizationSettings(H, W, cm.tanfovx, cm.tanfovy, torch.zeros(3, device=d), 1.0, cm.viewmatrix.to(d),
                                              cm.projmatrix.to(d), 3, cm.campos.to(d), False, False) for cm in cams]


    def ours():
        return video.render_video_frames(sc, settings)


    def reference():
        rc = ref_cuda.RefContext()
        framelist, depthlist, dmin, dmax = [], [], 1e8, -1e8
        for cm, rs in zip(cams, settings):
            _R, color, depth, _rad = ref_cuda.rasterize_gaussians(rc, rs.bg, sc["means3D"], None, sc["opacities"], sc["scales"],
                                                                  sc["rotations"], 1.0, None, rs.viewmatrix, rs.projmatrix,
                                                                  cm.tanfovx, cm.tanfovy, H, W, sc["shs"], 3, rs.campos)
            framelist.append(np.round(color.permute(1, 2, 0).detach().cpu().numpy().clip(0, 1) * 255.).astype(np.uint8))
            dd = -(depth * (depth > 0)).detach().cpu().numpy()
            dmin, dmax = min(dmin, dd.min().item()), max(dmax, dd.max().item())
            depthlist.append(dd)
        return framelist, depthlist, dmin, dmax


    out = {"frames": F, "H": H, "W": W, "P": P}
    res = {}
    for name, fn in (("ours", ours if "ours" in impls else None),
                     ("reference", reference if ref_cuda is not None and ref_cuda.available() else None)):
        if fn is None:
            continue
        fn(); torch.cuda.synchronize()
        t0 = time.perf_counter()
        r = fn()
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        res[name] = r
        out[name + "_ms_per_frame"] = dt / F * 1e3
        out[name + "_fps"] = F / dt
    if "reference" in res and "ours" in res:
        a, b = res["ours"], res["reference"]
        diff = np.abs(a[0].astype(np.int16) - np.stack(b[0]).astype(np.int16))
        out["max_uint8_diff_vs_reference"] = int(diff.max())
        out["pixels_differing"] = float((diff.max(-1) > 0).mean())
        out["dmin_dmax"] = [a[2], a[3], b[2], b[3]]
    return out


def _median(xs):
    return float(np.median(np.asarray(xs)))


def colour_rows(F=48, rounds=5):
    """The depth video's colour mapping (luciddreamer.py:267) on the same clip:
      depth_rgba_ms_per_frame    render_video_frames(depth_rgba=True): clip + device colour mapping, one host copy
      no_colour_ms_per_frame     render_video_frames(): clip + float depths to the host (the two alternate, median)
      device_colorize_ms_per_frame  video.colorize_frames over the F depth frames alone (CUDA events)
      host_colorize_ms_per_frame    video.colorize per frame on this machine's CPU (what the depth video costs without it)
    Traffic model of the device pass: 20 B per pixel (three 4-byte histogram reads, a 4-byte read and a 4-byte RGBA
    write in the colour pass); the reported rate is that model over the measured time, not a counter."""
    d = torch.device("cuda:0")
    c = syn.CONFIGS[3]
    P, W, H = c["P"], c["W"], c["H"]
    sc = {k: v.to(d) for k, v in syn.make_scene(P, 1003).items()}
    poses = syn.rotate360_poses(F)
    cams = [syn.make_camera(W, H, c2w=poses[k]) for k in range(F)]
    settings = [GaussianRasterizationSettings(H, W, cm.tanfovx, cm.tanfovy, torch.zeros(3, device=d), 1.0, cm.viewmatrix.to(d),
                                              cm.projmatrix.to(d), 3, cm.campos.to(d), False, False) for cm in cams]
    fns = {"no_colour": lambda: video.render_video_frames(sc, settings),
           "depth_rgba": lambda: video.render_video_frames(sc, settings, depth_rgba=True)}
    res, times = {}, {k: [] for k in fns}
    for name, fn in fns.items():
        res[name] = fn()
    torch.cuda.synchronize()
    for _ in range(rounds):
        for name, fn in fns.items():                       # every call ends in a stream synchronise
            t0 = time.perf_counter()
            fn()
            times[name].append(time.perf_counter() - t0)
    out = {"frames": F, "H": H, "W": W, "P": P}
    for name in fns:
        out[name + "_ms_per_frame"] = _median(times[name]) / F * 1e3
    depths, rgba = res["no_colour"][1], res["depth_rgba"][1]
    negd = torch.from_numpy(depths).to(d)
    video.colorize_frames(negd)
    torch.cuda.synchronize()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    reps = 10
    ev[0].record()
    for _ in range(reps):
        video.colorize_frames(negd)
    ev[1].record()
    torch.cuda.synchronize()
    dev_ms = ev[0].elapsed_time(ev[1]) / reps
    out["device_colorize_ms_per_frame"] = dev_ms / F
    out["device_colorize_model_GBps"] = 20.0 * H * W * F / (dev_ms * 1e-3) / 1e9
    host_t = []
    for k in range(min(F, 8)):
        t0 = time.perf_counter()
        host = video.colorize(depths[k])
        host_t.append(time.perf_counter() - t0)
        out.setdefault("depth_rgba_equals_host_colorize", True)
        out["depth_rgba_equals_host_colorize"] &= bool(np.array_equal(host, rgba[k]))
    out["host_colorize_ms_per_frame"] = _median(host_t) * 1e3
    out["host_cpus"] = os.cpu_count()
    out["gpu"] = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        out["power_limit"] = q.stdout.strip() or None
    except (OSError, subprocess.SubprocessError):
        out["power_limit"] = None
    return out


if __name__ == "__main__":
    F = int(sys.argv[1]) if len(sys.argv) > 1 else 48
    print(json.dumps({**run(F), "colour": colour_rows(F)}))
