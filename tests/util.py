"""Shared helpers of the parity tests."""
import os

import numpy as np

import cases

GOLDEN_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")

# north_star tolerances: forward colour/depth within 1e-4 abs, gradients within 1e-3 rel of the reference
FWD_ABS_TOL = 1e-4
GRAD_REL_TOL = 1e-3


def load_golden(name):
    z = np.load(os.path.join(GOLDEN_DIR, name + ".npz"), allow_pickle=False)
    out = dict(num_rendered=int(z["num_rendered"]), color=z["color"], depth=z["depth"], radii=z["radii"])
    grads = {}
    for g in cases.GRAD_NAMES:
        shape = tuple(int(x) for x in z[g + "_shape"])
        grads[g] = cases.dense_rows(z[g + "_idx"], z[g + "_rows"], shape)
        out[g + "_jitter"] = float(z[g + "_jitter"])
    out["grads"] = grads
    return out


def rel_err(a, b):
    a = np.asarray(a, np.float64); b = np.asarray(b, np.float64)
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-30))


def assert_forward_close(color, depth, radii, gold, what="", audit=None, flip_div=20000):
    """Colour/depth within 1e-4 abs.  Discontinuities (SURVEY.md Appendix B.1/B.2: alpha<1/255, T<1e-4, the
    acc>0.5 depth gate) may flip for isolated pixels when two implementations differ in the last ulp; those
    are counted and bounded instead of hidden: at most 1 pixel in 20 000 may exceed the tolerance, and -- when the
    oracle's forward state is passed as `audit` -- every one of them must be ATTRIBUTED to a branch operand sitting on
    its threshold (tests/flip_audit.py); an unexplained outlier fails."""
    color = np.asarray(color); depth = np.asarray(depth)
    dc = np.abs(color - gold["color"]).max(axis=0)
    dd = np.abs(depth - gold["depth"]).reshape(dc.shape)
    n = dc.size
    bad_c, bad_d = int((dc > FWD_ABS_TOL).sum()), int((dd > FWD_ABS_TOL).sum())
    assert bad_c <= n // flip_div, f"{what}: {bad_c}/{n} pixels off by > {FWD_ABS_TOL} in colour (max {dc.max():.3e})"
    assert bad_d <= n // flip_div, f"{what}: {bad_d}/{n} pixels off by > {FWD_ABS_TOL} in depth (max {dd.max():.3e})"
    if audit is not None and (bad_c or bad_d):
        import flip_audit
        explained, unexplained = flip_audit.explain_outliers(audit, color, depth, gold["color"], gold["depth"], FWD_ABS_TOL)
        print(f"[flip audit] {what}: {len(explained)} outlier pixel(s) attributed to branch flips: {explained}")
        assert not unexplained, f"{what}: outliers with no branch operand near a threshold: {unexplained}"
    mism = int((np.asarray(radii) != gold["radii"]).sum())
    assert mism <= max(0, len(gold["radii"]) // 50000), f"{what}: {mism} radii differ"
    return dict(max_color=float(dc.max()), max_depth=float(dd.max()), flips_color=bad_c, flips_depth=bad_d,
                radii_mismatch=mism)


def blend_rows_per_warp(W, H, device_index=0):
    """Image rows per warp of the tile passes for a W x H frame on this device, as the library's launch code decides it:
    4 (16x4 strips) or 8 (16x8 blocks)."""
    from luciddreamer_b200 import _native as N
    from luciddreamer_b200 import rasterizer as R
    rows = N.lib().gs_debug_blend_rows_per_warp(R._ctx(device_index), W, H)
    assert rows in (4, 8), N.last_error()
    print(f"[geometry] {W}x{H}: {rows} rows per warp")
    return rows


def assert_binning_matches_oracle(f, W, H, binning, img, num_pairs=None):
    """Integer pipeline of one `_C` forward (its opaque `binning` / `img` buffers), bit-exact against the oracle's forward
    state `f`: the tile offsets are monotone and end at the device's pair count (when given), and every tile's list is
    the oracle's list minus pairs that cannot contribute (exact tile culling), in the same (depth, index) order.
    Returns the device's per-tile list lengths."""
    import ctypes as C

    import torch
    from luciddreamer_b200 import _native as N
    cap = binning.numel() // 12
    G = ((W + 15) // 16) * ((H + 15) // 16)
    off = torch.empty(G + 1, dtype=torch.int32, device=binning.device)
    lst = torch.empty(cap, dtype=torch.int32, device=binning.device)
    frame = N.GsFrame()
    frame.W, frame.H = W, H
    N.check(N.lib().gs_debug_export_binning(C.byref(frame), binning.data_ptr(), cap, img.data_ptr(), off.data_ptr(),
                                            lst.data_ptr(), cap, torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    off = off.cpu().numpy().astype(np.int64); lst = lst.cpu().numpy().astype(np.int64)
    assert off[0] == 0 and np.all(np.diff(off) >= 0), "tile offsets are not monotone"
    assert off[-1] <= f.num_rendered
    if num_pairs is not None:
        assert off[-1] == num_pairs, f"off[G] = {off[-1]}, the device counted {num_pairs} pairs"
    opl, orng = f.point_list.astype(np.int64), f.ranges.astype(np.int64)
    depths = f.geom("depths", 1)[:, 0]
    for t in range(G):
        mine = lst[off[t]:off[t + 1]]
        ref = opl[orng[t, 0]:orng[t, 1]]
        if len(mine) == 0:
            continue
        assert set(mine) <= set(ref), f"tile {t}: a Gaussian the oracle does not bin there"
        # same relative order as the reference list
        pos = {g: i for i, g in enumerate(ref)}
        idx = [pos[g] for g in mine]
        assert idx == sorted(idx), f"tile {t}: order differs from the oracle's list"
        key = [(depths[g], g) for g in mine]
        assert key == sorted(key), f"tile {t}: not in (depth, index) order"
    return np.diff(off)


def assert_grads_close(grads, gold_grads, names=None, tol=GRAD_REL_TOL, what=""):
    out = {}
    for k, g in grads.items():
        if names is not None and k not in names:
            continue
        ref = gold_grads[k]
        if ref.size == 0:
            continue
        e = rel_err(np.asarray(g).reshape(ref.shape), ref)
        out[k] = e
        assert e <= tol, f"{what}: {k} rel err {e:.3e} > {tol}"
    return out
