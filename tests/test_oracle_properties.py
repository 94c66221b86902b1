"""Oracle self-checks that need no reference: float64 finite differences, independent SH / covariance
restatements, integer binning invariants, edge cases (P = 0, ragged images, ties)."""
import math

import numpy as np
import pytest
import torch

import cases
from luciddreamer_b200 import synthetic as syn
from oracle import oracle


def _fwd(inp, mode="f64", **over):
    a = list(cases.binding_args(inp))
    keys = ["bg", "means3D", "colors", "opacity", "scales", "rotations", "scale_modifier", "cov3D", "vm", "pm", "tfx",
            "tfy", "H", "W", "sh", "D", "campos"]
    for k, v in over.items():
        a[keys.index(k)] = v
    return oracle.rasterize_gaussians(*a[:17], mode=mode)


def test_f32_and_f64_agree():
    inp = cases.build_inputs(cases.BY_NAME["micro_1k_64"])
    a, b = _fwd(inp, "f32"), _fwd(inp, "f64")
    assert a.num_rendered == b.num_rendered
    assert np.abs(a.color - b.color).max() < 1e-4


def test_sh_colour_matches_independent_eval():
    """SH->RGB of the oracle vs a plain numpy restatement of the published real-SH basis (utils/sh.py:57-112)."""
    inp = cases.build_inputs(cases.BY_NAME["micro_1k_64"])
    f = _fwd(inp, "f64")
    vis = f.radii > 0
    p = inp["means3D"].double().numpy()
    d = p - inp["cam"].campos.double().numpy()[None]
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    x, y, z = d[:, 0], d[:, 1], d[:, 2]
    C0, C1 = 0.28209479177387814, 0.4886025119029199
    C2 = [1.0925484305920792, -1.0925484305920792, 0.31539156525252005, -1.0925484305920792, 0.5462742152960396]
    C3 = [-0.5900435899266435, 2.890611442640554, -0.4570457994644658, 0.3731763325901154, -0.4570457994644658,
          1.445305721320277, -0.5900435899266435]
    xx, yy, zz, xy, yz, xz = x * x, y * y, z * z, x * y, y * z, x * z
    B = np.stack([np.full_like(x, C0), -C1 * y, C1 * z, -C1 * x, C2[0] * xy, C2[1] * yz, C2[2] * (2 * zz - xx - yy),
                  C2[3] * xz, C2[4] * (xx - yy), C3[0] * y * (3 * xx - yy), C3[1] * xy * z,
                  C3[2] * y * (4 * zz - xx - yy), C3[3] * z * (2 * zz - 3 * xx - 3 * yy), C3[4] * x * (4 * zz - xx - yy),
                  C3[5] * z * (xx - yy), C3[6] * x * (xx - 3 * yy)], 1)
    rgb = np.maximum(np.einsum("pk,pkc->pc", B, inp["shs"].double().numpy()) + 0.5, 0.0)
    assert np.abs(f.geom("rgb", 3)[vis] - rgb[vis]).max() < 1e-12


def test_cov3d_matches_R_S_S_Rt():
    inp = cases.build_inputs(cases.BY_NAME["micro_1k_64"])
    f = _fwd(inp, "f64")
    vis = np.nonzero(f.radii > 0)[0]
    q = inp["rotations"].double().numpy(); s = inp["scales"].double().numpy()
    for i in vis[:50]:
        r, x, y, z = q[i]
        R = np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - r * z), 2 * (x * z + r * y)],
                      [2 * (x * y + r * z), 1 - 2 * (x * x + z * z), 2 * (y * z - r * x)],
                      [2 * (x * z - r * y), 2 * (y * z + r * x), 1 - 2 * (x * x + y * y)]])
        S = R @ np.diag(s[i] ** 2) @ R.T
        c6 = f.geom("cov3D", 6)[i]
        assert np.allclose(c6, [S[0, 0], S[0, 1], S[0, 2], S[1, 1], S[1, 2], S[2, 2]], rtol=1e-12, atol=1e-15)


def test_binning_invariants():
    """keys sorted; per-tile ranges partition the list; list order = (depth, index) inside every tile."""
    inp = cases.build_inputs(cases.BY_NAME["stress_4k_96_x6"])
    f = _fwd(inp, "f32")
    keys, pl, rng = f.keys, f.point_list, f.ranges
    assert np.all(keys[1:] >= keys[:-1])
    assert int(f.tiles_touched.sum()) == f.num_rendered == len(pl)
    depths = f.geom("depths", 1)[:, 0]
    covered = 0
    for t, (a, b) in enumerate(rng):
        if b > a:
            assert np.all((keys[a:b] >> np.uint64(32)) == t)
            d = depths[pl[a:b]]
            assert np.all(np.diff(d) >= 0)
            same = np.diff(d) == 0
            assert np.all(np.diff(pl[a:b].astype(np.int64))[same] > 0)     # ties: ascending Gaussian index
            covered += b - a
    assert covered == f.num_rendered


def test_depth_ties_resolve_by_index():
    """Two Gaussians with bit-identical depth in one tile: the lower index is composited first (stable sort)."""
    cam = syn.make_camera(32, 32)
    means = torch.tensor([[0.02, 0.0, 2.0], [-0.02, 0.0, 2.0]])
    sc = torch.full((2, 3), 0.05); rot = torch.tensor([[1.0, 0, 0, 0]] * 2); op = torch.tensor([[0.9], [0.9]])
    col = torch.tensor([[1.0, 0, 0], [0, 1.0, 0]])
    for order in ([0, 1], [1, 0]):
        f = oracle.rasterize_gaussians(torch.zeros(3), means[order], col[order], op, sc, rot, 1.0, None, cam.viewmatrix,
                                       cam.projmatrix, cam.tanfovx, cam.tanfovy, 32, 32, None, 0, cam.campos)
        pl, rng = f.point_list, f.ranges
        for a, b in rng:
            if b - a == 2:
                assert list(pl[a:b]) == [0, 1]


def test_zero_gaussians_gives_zero_image_not_background():
    cam = syn.make_camera(16, 16)
    f = oracle.rasterize_gaussians(torch.ones(3), torch.zeros(0, 3), None, torch.zeros(0, 1), torch.zeros(0, 3),
                                   torch.zeros(0, 4), 1.0, None, cam.viewmatrix, cam.projmatrix, cam.tanfovx,
                                   cam.tanfovy, 16, 16, torch.zeros(0, 16, 3), 3, cam.campos)
    assert f.num_rendered == 0 and not f.color.any() and not f.depth.any()   # rasterize_points.cu:68,82


def test_background_shows_where_nothing_is_rendered():
    inp = cases.build_inputs(cases.BY_NAME["odd_3k_100x70_bg"])
    f = _fwd(inp, "f32")
    empty = f.n_contrib == 0
    assert empty.any()
    for ch in range(3):
        assert np.allclose(f.color[ch][empty], inp["case"].bg[ch])
    assert not f.depth[0][empty].any()


def test_mark_visible_is_near_plane_only():
    inp = cases.build_inputs(cases.BY_NAME["micro_1k_64"])
    vis = oracle.mark_visible(inp["means3D"], inp["cam"].viewmatrix)
    assert np.array_equal(vis, (inp["means3D"][:, 2] > 0.2).numpy())        # identity camera: z_view = z


def _loss(inp, cot, **over):
    f = _fwd(inp, "f64", **over)
    return float((f.color * cot).sum()), f


@pytest.mark.parametrize("param,col", [("opacity", 2), ("sh", 5), ("scales", 6), ("rotations", 7), ("means3D", 3)])
def test_backward_matches_finite_differences_f64(param, col):
    """Central differences of the float64 forward against the explicit backward, on the entries where the forward
    is an exact derivative (SURVEY.md A.7b): away from the 0.99 clamp and the tan-fov guard band."""
    case = cases.Case("fd", 300, 48, 48, 3, 21, scale_mult=3.0, golden=False)
    inp = cases.build_inputs(case)
    cot = inp["cot"].double().numpy()
    base, f = _loss(inp, cot)
    g = oracle.rasterize_gaussians_backward(f, cot)
    grad = g[col]
    key = {"opacity": "opacities", "sh": "shs", "scales": "scales", "rotations": "rotations", "means3D": "means3D"}[param]
    x0 = inp[key].double()
    vis = np.nonzero(f.radii > 0)[0]
    rng = np.random.default_rng(0)
    checked = 0
    for i in rng.permutation(vis)[:12]:
        flat = x0[i].reshape(-1)
        j = int(rng.integers(flat.numel()))
        if param == "sh" and j // 3 >= 16:
            continue
        h = 1e-6 * max(1.0, abs(float(flat[j])))
        vals = []
        for sgn in (+1, -1):
            x = x0.clone()
            x[i].reshape(-1)[j] += sgn * h
            vals.append(_loss(inp, cot, **{param: x})[0])
        fd = (vals[0] - vals[1]) / (2 * h)
        an = float(np.asarray(grad[i]).reshape(-1)[j])
        # discontinuities (alpha/T thresholds, ceil radius) make a few FD probes meaningless: require agreement
        # for the smooth majority
        if abs(fd - an) <= 2e-4 * max(1.0, abs(an), abs(fd)):
            checked += 1
    assert checked >= 9, f"only {checked}/12 finite-difference probes of {param} agree"


def test_flip_audit_replay_is_faithful():
    """tests/flip_audit.py replays single pixels from the oracle's state; its final T must be the oracle's, and a
    synthetic "flip" (a pixel perturbed by more than the tolerance) with no operand near a threshold must be
    reported as unexplained."""
    import flip_audit
    case = cases.BY_NAME["opaque_40k_64_x8"]
    inp = cases.build_inputs(case)
    f = _fwd(inp, "f32")
    fT = f.final_T
    rng = np.random.RandomState(0)
    for _ in range(40):
        x, y = int(rng.randint(case.W)), int(rng.randint(case.H))
        m = flip_audit.pixel_margins(f, x, y)
        assert abs(m["final_T"] - float(fT[y, x])) <= 1e-5 * max(float(fT[y, x]), 1e-4) + 1e-9
    bad = f.color.copy()
    # pick a pixel whose margins are all wide, perturb it: the audit must refuse to explain it
    for y in range(case.H):
        for x in range(case.W):
            m = flip_audit.pixel_margins(f, x, y)
            if min(m["alpha"], m["T"], m["acc"], m["power"]) > 1e-2:
                bad[0, y, x] += 1e-2
                ex, un = flip_audit.explain_outliers(f, bad, f.depth, f.color, f.depth)
                assert len(un) == 1 and not ex and un[0][:2] == (x, y)
                return
    raise AssertionError("no wide-margin pixel found")


@pytest.mark.parametrize("name", [c.name for c in cases.EXTRA_CASES + cases.BLOCK_CASES])
def test_extra_cases_reach_their_branches(name):
    """The oracle-only cases exist to reach early termination, the 0.99 clamp, ill-conditioned conics and long
    tile lists, the block cases to reach them on a grid of 1 500 tiles or more with ragged sides; make sure the scenes
    really do (otherwise the GPU parity tests on them prove nothing)."""
    case = cases.BY_NAME[name]
    inp = cases.build_inputs(case)
    f = _fwd(inp, "f32")
    rg = f.ranges.astype(np.int64)
    lens = rg[:, 1] - rg[:, 0]
    longest = int(lens.max())
    terminated = float((f.final_T < 1e-3).mean())
    clamped = float((inp["opacities"] > 0.99).float().mean())
    visible = float((f.radii > 0).mean())
    rect = int(f.tiles_touched.max())
    co = f.geom("conic_opacity", 4)[f.radii > 0].astype(np.float64)
    det, tr = co[:, 0] * co[:, 2] - co[:, 1] ** 2, co[:, 0] + co[:, 2]
    ill = float((det < 1e-5 * tr * tr).mean())                 # the blend kernels' conditioning test routes these
    print(f"{name}: {len(lens)} tiles, terminated {terminated:.3f}, above the clamp {clamped:.3f}, ill-conditioned {ill:.3f}, "
          f"longest list {longest}, largest rect {rect} tiles, visible {visible:.3f}")
    if case in cases.BLOCK_CASES:
        assert len(lens) >= 1500 and case.W % 16 and case.H % 8
        assert (f.tiles_touched > 32).sum() > 100              # rects beyond the 32-bit hit mask: decisions recomputed
        full = f.n_contrib[:case.H // 16 * 16, :case.W // 16 * 16] > 0
        assert (f.n_contrib[case.H // 16 * 16:] > 0).any() and (f.n_contrib[:, case.W // 16 * 16:] > 0).any() and full.any()
    if name.startswith("blk_shell") or name.startswith("blk_precomp"):
        assert terminated < 0.01 and visible < 0.1 and (f.radii > 0).sum() > 1000     # the plain, sparse path
        assert any(case.bg) and (f.final_T > 0.1).mean() > 0.05                         # background shows through
    elif name.startswith("blk_opaque"):
        assert terminated > 0.9 and clamped > 0.3 and longest > 256
    elif name.startswith("blk_needles"):
        assert ill > 0.05 and rect > 1000 and longest > 256
    elif name.startswith("blk_frustum"):
        # dense regime (more than half of the Gaussians visible), lists on both sides of the 2 048-entry sort size with
        # room for the exact tile culling of the CUDA path, termination
        assert visible > 0.5 and terminated > 0.9 and lens.min() > 256
        assert (lens > 3000).sum() >= 10 and (lens < 1800).sum() >= 10
    elif name.startswith("opaque"):
        assert terminated > 0.5 and clamped > 0.2
    elif name.startswith("needles"):
        assert ill > 0.02
    else:
        assert terminated > 0.5 and longest > 1500
