"""Attribution of forward outliers to branch flips (SURVEY.md Appendix B.1/B.2).

The rasterizer's forward has four discontinuities per (pixel, splat): `power > 0` and `alpha < 1/255` skip the splat
(forward.cu:336-346), `T * (1 - alpha) < 1e-4` ends the pixel (forward.cu:348-352), and the depth output is gated by
`acc > 0.5` (forward.cu:384-388).  Two correct implementations that differ in the last ulp of one operand can take
different sides of such a test on an isolated pixel and then differ by up to alpha * T * colour there.  The parity
tests therefore do not merely bound the NUMBER of pixels beyond the 1e-4 tolerance: every such pixel is replayed here
(float64, from the oracle's per-Gaussian state and depth-sorted tile list) and must sit within `rel_margin` of one of
the four thresholds.  A pixel beyond tolerance with no operand near a threshold is a real error and fails the test.
"""
from __future__ import annotations

import numpy as np


def pixel_margins(fwd, x: int, y: int):
    """Replays forward.cu:330-388 for pixel (x, y) with the oracle's state; returns the smallest relative distance of a
    branch operand to its threshold, per kind of branch."""
    H, W = fwd.depth.shape[-2:]
    gx = (W + 15) // 16
    tile = (y // 16) * gx + (x // 16)
    beg, end = (int(v) for v in fwd.ranges[tile])
    ids = fwd.point_list[beg:end].astype(np.int64)
    xy = fwd.geom("means2D", 2)[ids].astype(np.float64)
    co = fwd.geom("conic_opacity", 4)[ids].astype(np.float64)
    dx, dy = xy[:, 0] - x, xy[:, 1] - y
    power = -0.5 * (co[:, 0] * dx * dx + co[:, 2] * dy * dy) - co[:, 1] * dx * dy
    alpha = np.minimum(0.99, co[:, 3] * np.exp(np.minimum(power, 50.0)))
    m = dict(alpha=np.inf, power=np.inf, T=np.inf, acc=np.inf)
    T, acc = 1.0, 1e-6
    for j in range(len(ids)):
        scale = max(abs(co[j, 0] * dx[j] * dx[j]) + abs(co[j, 2] * dy[j] * dy[j]) + abs(co[j, 1] * dx[j] * dy[j]), 1e-30)
        m["power"] = min(m["power"], abs(power[j]) / scale if power[j] > -1e-3 * scale else np.inf)
        if power[j] > 0.0:
            continue
        m["alpha"] = min(m["alpha"], abs(alpha[j] - 1.0 / 255.0) * 255.0)
        if alpha[j] < 1.0 / 255.0:
            continue
        test_T = T * (1.0 - alpha[j])
        m["T"] = min(m["T"], abs(test_T - 1e-4) / 1e-4)
        if test_T < 1e-4:
            break
        acc += alpha[j] * T
        T = test_T
    m["acc"] = abs(acc - 0.5) / 0.5
    m["final_T"] = T                  # replay outputs, for the self-check in tests/test_oracle_properties.py
    m["n_visited"] = j + 1 if len(ids) else 0
    return m


def near_thresholds(m, rel_margin=2e-5):
    """The kinds of branch whose operand, in the margins `m` of pixel_margins, sits within `rel_margin` of its threshold."""
    # T accumulates one rounding per contributing splat, hence the wider margin on the termination test
    return [k for k, lim in (("alpha", rel_margin), ("power", rel_margin), ("T", 50 * rel_margin), ("acc", rel_margin))
            if m[k] < lim]


def explain_outliers(fwd, color, depth, ref_color, ref_depth, tol=1e-4, rel_margin=2e-5, max_pixels=64):
    """Returns (explained, unexplained): lists of (x, y, err_colour, err_depth, kind / margins) for every pixel whose
    colour or depth differs from the reference by more than `tol`."""
    color, depth = np.asarray(color, np.float64), np.asarray(depth, np.float64)
    dc = np.abs(color - ref_color).max(axis=0)
    dd = np.abs(depth - ref_depth).reshape(dc.shape)
    ys, xs = np.nonzero((dc > tol) | (dd > tol))
    explained, unexplained = [], []
    for y, x in list(zip(ys.tolist(), xs.tolist()))[:max_pixels]:
        m = pixel_margins(fwd, x, y)
        near = near_thresholds(m, rel_margin)
        rec = (x, y, float(dc[y, x]), float(dd[y, x]), near or {k: float(v) for k, v in m.items() if k in ("alpha", "power", "T", "acc")})
        (explained if near else unexplained).append(rec)
    return explained, unexplained
