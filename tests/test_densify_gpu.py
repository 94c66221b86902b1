"""Densification on the device (luciddreamer_b200.densify, include/gsdensify.h) against the reference's own
GaussianModel.densify_and_prune and reset_opacity (its bytecode from oracle/_ref/pyref): the same parameters, moments,
statistics, step counters, group layout and random-generator state, bit for bit; and a short LucidDreamer training
loop with TrainStep whose densifications run through densify.attach."""
import math
import os
import random
import sys
import types

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PYREF = os.path.join(ROOT, "oracle", "_ref", "pyref")
needs_pyref = pytest.mark.skipif(not os.path.exists(os.path.join(PYREF, "gaussian_renderer", "__init__.pyc")),
                                 reason="oracle/_ref/pyref not built (make -C oracle pyref needs /root/reference)")
NAMES = ("xyz", "f_dc", "f_rest", "opacity", "scaling", "rotation")


def dev():
    return torch.device("cuda:0")


@pytest.fixture(scope="module")
def refmods():
    """The reference's bytecode with this repository's rasterizer underneath."""
    saved_path, saved_mods = list(sys.path), dict(sys.modules)
    sys.path.insert(0, PYREF)
    if ROOT not in sys.path:
        sys.path.insert(1, ROOT)
    ply = types.ModuleType("plyfile")
    ply.PlyData = ply.PlyElement = object
    sys.modules["plyfile"] = ply
    for name in [m for m in sys.modules if m.split(".")[0] in ("utils", "scene", "gaussian_renderer", "arguments", "refrast")]:
        del sys.modules[name]
    import depth_diff_gaussian_rasterization_min as ours_rast
    shim = types.ModuleType("refrast._C")
    for n in ("rasterize_gaussians", "rasterize_gaussians_backward", "mark_visible"):
        setattr(shim, n, getattr(ours_rast._C, n))
    sys.modules["refrast._C"] = shim
    import arguments
    import gaussian_renderer
    from scene.gaussian_model import GaussianModel
    from utils.graphics import BasicPointCloud
    assert sys.modules["scene.gaussian_model"].__file__.startswith(PYREF)
    yield types.SimpleNamespace(render=gaussian_renderer.render, GaussianModel=GaussianModel, GSParams=arguments.GSParams,
                                BasicPointCloud=BasicPointCloud)
    sys.path[:] = saved_path
    ours = ("utils", "scene", "gaussian_renderer", "arguments", "refrast", "plyfile")
    for name in [m for m in sys.modules if m not in saved_mods and m.split(".")[0] in ours]:
        del sys.modules[name]


# ---- models ------------------------------------------------------------------------------------------------------------

def _model(refmods, P, sh, state, seed):
    """A GaussianModel with seeded parameters and statistics; state: "none" (torch Adam before its first step),
    "adam" (torch Adam after three steps) or "fused" (optim.FusedAdam after three steps)."""
    from luciddreamer_b200 import optim
    g = torch.Generator().manual_seed(seed)
    M = (sh + 1) ** 2
    gm = refmods.GaussianModel(sh)
    raw = dict(xyz=torch.randn(P, 3, generator=g), f_dc=torch.randn(P, 1, 3, generator=g),
               f_rest=torch.randn(P, M - 1, 3, generator=g) * 0.1, opacity=torch.randn(P, 1, generator=g) * 3,
               scaling=torch.randn(P, 3, generator=g) * 0.7 - 4, rotation=torch.randn(P, 4, generator=g))
    for n in NAMES:
        setattr(gm, "_" + {"f_dc": "features_dc", "f_rest": "features_rest"}.get(n, n),
                torch.nn.Parameter(raw[n].to(dev()).contiguous().requires_grad_(True)))
    gm.spatial_lr_scale = 1.0
    gm.max_radii2D = torch.zeros(P, device=dev())
    gm.training_setup(refmods.GSParams())
    denom = torch.randint(0, 6, (P, 1), generator=g).float()
    accum = torch.rand(P, 1, generator=g) * 4e-4 * denom
    if P >= 4:
        accum[0], denom[0] = 0.0, 0.0          # 0 / 0: NaN -> 0
        accum[1], denom[1] = 1e-4, 0.0         # x / 0: inf
    gm.xyz_gradient_accum, gm.denom = accum.to(dev()), denom.to(dev())
    gm.max_radii2D = torch.randint(0, 40, (P,), generator=g).float().to(dev())
    if state == "fused":
        optim.attach(gm)
    if state != "none":
        for _ in range(3):
            for grp in gm.optimizer.param_groups:
                p = grp["params"][0]
                p.grad = (torch.randn(p.shape, generator=g) * 1e-3).to(dev())
            gm.optimizer.step()
            gm.optimizer.zero_grad(set_to_none=True)
    torch.cuda.synchronize()
    return gm


def _snapshot(gm):
    out = {"xyz": gm._xyz, "f_dc": gm._features_dc, "f_rest": gm._features_rest, "opacity": gm._opacity,
           "scaling": gm._scaling, "rotation": gm._rotation, "xyz_gradient_accum": gm.xyz_gradient_accum,
           "denom": gm.denom, "max_radii2D": gm.max_radii2D}
    for grp in gm.optimizer.param_groups:
        assert grp["params"][0] is out[grp["name"]], grp["name"]
        st = gm.optimizer.state.get(grp["params"][0])
        if st is not None:
            for k, v in st.items():
                out[grp["name"] + "." + k] = v
    return out


def _layout(gm):
    return [(grp["name"], len(grp["params"]), grp["params"][0].requires_grad, grp["params"][0].dtype,
             type(grp["params"][0]), grp["params"][0] in gm.optimizer.state) for grp in gm.optimizer.param_groups]


def _ulps(a, b):
    ia = a.contiguous().view(torch.int32).long()
    ib = b.contiguous().view(torch.int32).long()
    ia = torch.where(ia < 0, -(ia & 0x7fffffff), ia)
    ib = torch.where(ib < 0, -(ib & 0x7fffffff), ib)
    return int((ia - ib).abs().max()) if a.numel() else 0


def _assert_same(ref, ours, before_ids, what, same_optimiser=True):
    """Every parameter, moment, statistic and step counter equal bit for bit, the same group layout, new Parameters."""
    a, b = _snapshot(ref), _snapshot(ours)
    assert a.keys() == b.keys(), (what, a.keys() ^ b.keys())
    for k in a:
        x, y = a[k], b[k]
        if k.endswith(".step"):
            assert float(x) == float(y), (what, k)
            assert not same_optimiser or (x.dtype == y.dtype and x.device == y.device), (what, k)
            continue
        assert x.shape == y.shape and x.dtype == y.dtype and x.device == y.device, (what, k, x.shape, y.shape)
        assert torch.equal(x, y), (what, k, "max ulps", _ulps(x, y), "rows differing",
                                   int((x != y).reshape(x.shape[0], -1).any(1).sum()),
                                   (x != y).reshape(x.shape[0], -1).any(1).nonzero()[:8].flatten().tolist())
    assert _layout(ref) == _layout(ours), what
    for grp in ours.optimizer.param_groups:           # every Parameter is a new object
        assert not any(grp["params"][0] is p for p in before_ids), (what, grp["name"])


# ---- thresholds --------------------------------------------------------------------------------------------------------

def _grads(gm):
    g = gm.xyz_gradient_accum / gm.denom
    g[g.isnan()] = 0.0
    return g.squeeze(-1)


def _args(gm, case):
    """(max_grad, min_opacity, extent, max_screen_size) of a named case, from the model's own values."""
    g = _grads(gm)
    smax = gm.get_scaling.max(dim=1).values
    op = gm.get_opacity.squeeze(-1)
    fin = g[torch.isfinite(g)]
    q = lambda t, p: float(torch.quantile(t.detach().double().cpu(), p)) if t.numel() else 0.0
    mid_grad, mid_scale = q(fin, 0.5), q(smax, 0.5) / gm.percent_dense
    if case == "mixed":                  # clone, split and the opacity prune fire
        return mid_grad, q(op, 0.2), mid_scale, None
    if case == "world":                  # and the world-size prune (max(exp(s)) > 0.1 * extent)
        return mid_grad, q(op, 0.1), q(smax, 0.3) * 10, 20
    if case == "screen0":
        return mid_grad, q(op, 0.2), mid_scale, 0
    if case == "screen_below_radii":     # 0 > 0.5 never holds: the zeroed max_radii2D prune nothing
        return mid_grad, q(op, 0.2), mid_scale, 0.5
    if case == "screen_negative":        # 0 > -1 prunes everything
        return mid_grad, q(op, 0.2), mid_scale, -1
    if case == "nothing":                # nothing selected, nothing pruned: every tensor still replaced
        return 1e9, 0.0, 1e9, None
    if case == "exact":                  # thresholds equal to values of the model (>=, <=, >, < as the reference)
        k = len(fin) // 3
        smid = float(smax.detach().sort().values[len(smax) // 2])
        return float(fin.sort().values[k]), float(op.detach().sort().values[len(op) // 4]), smid / gm.percent_dense, None
    if case == "between":                # thresholds that are not float32 values: a quarter ulp beside a model value,
        # on the side where comparing in double decides that row the other way than torch's float32 comparison
        # (gv >= gv + q, sv <= sv - q and ov < ov + q flip once the threshold is rounded to float32)
        gv = float(fin.sort().values[len(fin) // 3])
        sel = smax[g >= np.float32(gv)].detach()
        sv = float(sel.sort().values[len(sel) // 2])
        ov = float(op.detach().sort().values[len(op) // 4])
        return _quarter_ulp(gv, 1), _quarter_ulp(ov, 1), _quarter_ulp(sv, -1) / gm.percent_dense, None
    if case == "split_all":              # every row splits, none is pruned
        return 0.0, 0.0, 1e-30, None
    raise ValueError(case)


def _quarter_ulp(v, direction):
    """v moved a quarter of the float32 spacing towards +inf (direction 1) or -inf (-1): rounds back to v in float32."""
    f = np.float32(v)
    nxt = np.nextafter(f, np.float32(np.inf if direction > 0 else -np.inf))
    return float(f) + 0.25 * (float(nxt) - float(f))


def _run(refmods, P, sh, state, case, seed):
    from luciddreamer_b200 import densify
    ref, ours = _model(refmods, P, sh, state, seed), _model(refmods, P, sh, state, seed)
    if case in ("exact", "between"):
        ref.percent_dense = ours.percent_dense = 1.0      # so that percent_dense * extent is exactly the chosen value
    args = _args(ref, case)
    before = [g["params"][0] for g in ours.optimizer.param_groups]
    torch.manual_seed(seed)
    ref.densify_and_prune(*args)
    rng_ref = torch.cuda.get_rng_state()
    torch.manual_seed(seed)
    counts = densify.densify_and_prune(ours, *args)
    rng_ours = torch.cuda.get_rng_state()
    torch.cuda.synchronize()
    assert torch.equal(rng_ref, rng_ours)
    assert counts["P"] == ref._xyz.shape[0] == ours._xyz.shape[0]
    _assert_same(ref, ours, before, (P, sh, state, case))
    return counts


CASES = [
    (1, 3, "adam", "nothing"), (1, 0, "none", "mixed"),
    (7, 0, "fused", "mixed"), (7, 3, "adam", "screen_negative"),
    (1000, 3, "none", "mixed"), (1000, 3, "fused", "world"), (1000, 0, "adam", "exact"), (1000, 3, "fused", "screen0"),
    (1000, 3, "adam", "screen_below_radii"), (1000, 3, "fused", "nothing"),
    (100_000, 3, "fused", "mixed"), (100_000, 3, "adam", "world"), (100_000, 0, "none", "exact"),
    (100_000, 3, "fused", "screen_negative"), (1000, 3, "adam", "between"), (100_000, 3, "fused", "between"),
]


@needs_pyref
@pytest.mark.parametrize("P,sh,state,case", CASES)
def test_densify_and_prune_equals_the_reference(refmods, P, sh, state, case):
    counts = _run(refmods, P, sh, state, case, seed=P + sh + len(case))
    if case == "nothing":                    # only the x / 0 = inf row reaches max_grad = 1e9, and it is cloned
        assert counts == {"clones": int(P >= 4), "splits": 0, "survivors": P, "P": P + int(P >= 4)}
    if case == "screen_negative":
        assert counts["P"] == 0
    if P >= 1000 and case in ("mixed", "exact", "between"):
        assert counts["clones"] > 0 and counts["splits"] > 0 and counts["survivors"] < P - counts["splits"], counts
    if P >= 1000 and case == "world":
        assert counts["splits"] > 0 and counts["survivors"] < P - counts["splits"], counts


@needs_pyref
def test_the_cases_reach_every_decision(refmods):
    """The thresholds of the parity cases make each criterion fire, and the exact case puts values on each threshold."""
    gm = _model(refmods, 1000, 3, "fused", 1000 + 3 + len("world"))
    max_grad, min_op, extent, screen = _args(gm, "world")
    smax = gm.get_scaling.max(dim=1).values
    assert bool((smax > torch.tensor(0.1 * extent, dtype=torch.float32)).any())
    assert bool((gm.get_opacity < torch.tensor(min_op, dtype=torch.float32)).any())
    gm = _model(refmods, 1000, 0, "adam", 1000 + len("exact"))
    gm.percent_dense = 1.0
    max_grad, min_op, extent, _ = _args(gm, "exact")
    assert bool((_grads(gm) == torch.tensor(max_grad, dtype=torch.float32)).any())
    assert bool((gm.get_scaling.max(dim=1).values == torch.tensor(extent, dtype=torch.float32)).any())
    assert bool((gm.get_opacity == torch.tensor(min_op, dtype=torch.float32)).any())
    assert bool((gm.denom == 0).any())
    # the "between" thresholds decide differently in double than after torch's cast to float32
    gm = _model(refmods, 1000, 3, "adam", 1000 + 3 + len("between"))
    gm.percent_dense = 1.0
    max_grad, min_op, extent, _ = _args(gm, "between")
    g, smax, op = _grads(gm), gm.get_scaling.max(dim=1).values.detach(), gm.get_opacity.detach()
    f32 = lambda x: torch.tensor(x, dtype=torch.float32).item()
    assert float(np.float32(max_grad)) != max_grad and f32(max_grad) == float(np.float32(max_grad))
    assert bool(((g.double() >= max_grad) != (g >= f32(max_grad))).any())
    sel = g >= f32(max_grad)
    assert bool(((smax.double() <= extent) != (smax <= f32(extent)))[sel].any())
    assert bool(((op.double() < min_op) != (op < f32(min_op))).any())


@needs_pyref
@pytest.mark.parametrize("P", [6498, 6499, 18646, 18647, 42768])
def test_split_xyz_follows_bmm_across_batch_counts(refmods, P):
    """Every row splits, so torch.bmm runs over 2P matrices: chunks of 12 998 to 37 292 matrices are rounded by the
    other cuBLAS kernel (2 * 6499, 2 * 18646, and the 20 001-matrix tail of 2 * 42768); the split rows' xyz must still
    be bit-identical."""
    counts = _run(refmods, P, 0, "adam", "split_all", seed=P)
    assert counts == {"clones": 0, "splits": P, "survivors": 0, "P": 2 * P}


@needs_pyref
@pytest.mark.parametrize("P,state", [(1, "adam"), (1000, "fused"), (100_000, "adam")])
def test_reset_opacity_equals_the_reference(refmods, P, state):
    from luciddreamer_b200 import densify
    ref, ours = _model(refmods, P, 3, state, 5 + P), _model(refmods, P, 3, state, 5 + P)
    with torch.no_grad():                    # values on both sides of the 0.01 cap, and on it
        for gm in (ref, ours):
            gm._opacity[: (P + 1) // 2] -= 3.0
            gm._opacity[0] = torch.logit(torch.tensor(0.01)).item()
    before = [g["params"][0] for g in ours.optimizer.param_groups]
    ref.reset_opacity()
    densify.reset_opacity(ours)
    torch.cuda.synchronize()
    a, b = _snapshot(ref), _snapshot(ours)
    for k in a:
        assert torch.equal(a[k].cpu(), b[k].cpu()) and a[k].dtype == b[k].dtype, k
    assert float(a["opacity.step"]) == 3.0
    assert _layout(ref) == _layout(ours)
    now = {g["name"]: g["params"][0] for g in ours.optimizer.param_groups}
    kept = [n for n in NAMES if any(now[n] is p for p in before)]
    assert kept == [n for n in NAMES if n != "opacity"]


@needs_pyref
def test_attach_binds_the_device_methods(refmods):
    from luciddreamer_b200 import densify
    ref, ours = _model(refmods, 1000, 3, "adam", 77), _model(refmods, 1000, 3, "adam", 77)
    densify.attach(ours)
    args = _args(ref, "mixed")
    torch.manual_seed(3)
    ref.densify_and_prune(*args)
    ref.reset_opacity()
    torch.manual_seed(3)
    ours.densify_and_prune(*args)
    ours.reset_opacity()
    torch.cuda.synchronize()
    _assert_same(ref, ours, [], "attach")


# ---- the training loop -------------------------------------------------------------------------------------------------

def _loop_setup(refmods, P, W, H, ncams, seed, iters):
    from luciddreamer_b200 import synthetic as syn
    sc = syn.make_frustum_scene(P, seed, W, H, raster=True)
    g = torch.Generator().manual_seed(seed)
    pcd = refmods.BasicPointCloud(points=sc["means3D"].numpy(), colors=torch.rand(P, 3, generator=g).numpy(),
                                  normals=np.zeros((P, 3)))
    opt = refmods.GSParams()
    opt.iterations = iters
    cams = []
    for pose in syn.jitter_poses(ncams, seed):
        c = syn.make_camera(W, H, c2w=pose)
        gt = F.interpolate(torch.rand(1, 3, H // 8, W // 8, generator=g), size=(H, W), mode="bilinear",
                           align_corners=False)[0]
        cams.append(types.SimpleNamespace(FoVx=2 * math.atan(c.tanfovx), FoVy=2 * math.atan(c.tanfovy), image_width=W,
                                          image_height=H, world_view_transform=c.viewmatrix.to(dev()),
                                          full_proj_transform=c.projmatrix.to(dev()), camera_center=c.campos.to(dev()),
                                          original_image=gt.contiguous().to(dev())))

    def model():
        gm = refmods.GaussianModel(3)
        gm.create_from_pcd(pcd, 1.0)
        gm.training_setup(opt)
        with torch.no_grad():
            gm._scaling.copy_(torch.log(sc["scales"]).to(dev()))
            gm._rotation.copy_(sc["rotations"].to(dev()))
            gm._opacity.copy_(torch.logit(sc["opacities"].clamp(1e-3, 1 - 1e-3)).to(dev()))
            gm._features_rest.copy_(sc["shs"][:, 1:].to(dev()))
        return gm
    return model, cams, opt


def _rel(a, b):
    a, b = a.double(), b.double()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


def _assert_close(ref, ours, skip, what, tol=1e-4):
    """Every tensor within tol (relative, outside the rows in skip), every step counter equal."""
    a, b = _snapshot(ref), _snapshot(ours)
    assert a.keys() == b.keys(), (what, a.keys() ^ b.keys())
    for k in a:
        if k.endswith(".step"):
            assert float(a[k]) == float(b[k]), (what, k)
            continue
        assert a[k].shape == b[k].shape, (what, k)
        x, y = b[k][~skip], a[k][~skip]
        assert _rel(x, y) <= tol, (what, k, _rel(x, y))


def _anchor(dst, src):
    """Copies every parameter, moment and statistic of src into dst in place (the captured graph stays valid)."""
    with torch.no_grad():
        for gd, gs in zip(dst.optimizer.param_groups, src.optimizer.param_groups):
            gd["params"][0].copy_(gs["params"][0])
            sd, ss = dst.optimizer.state.get(gd["params"][0]), src.optimizer.state.get(gs["params"][0])
            if sd and ss:
                sd["exp_avg"].copy_(ss["exp_avg"])
                sd["exp_avg_sq"].copy_(ss["exp_avg_sq"])
        for name in ("xyz_gradient_accum", "denom", "max_radii2D"):
            getattr(dst, name).copy_(getattr(src, name))


@needs_pyref
def test_train_step_with_device_densify_follows_the_reference_loop(refmods):
    """luciddreamer.py:283-327 for 30 iterations with densification at 10 and 20 and an opacity reset at 25: the
    reference's render() + GaussianModel + torch.optim.Adam against TrainStep + FusedAdam with densify.attach, both in
    deterministic mode. The segments between edits agree to 1e-4 outside the rows where the rasterizer's discrete
    decisions went the other way (at most P / 500, detected from the gradient w.r.t. the means); before every edit the
    reference's state is copied into ours, so the densify and the reset themselves must agree bit for bit."""
    from luciddreamer_b200 import densify, optim, train
    from luciddreamer_b200 import rasterizer as R
    from oracle import loss_oracle as LO
    iters, W, H = 30, 96, 96
    model, cams, opt = _loop_setup(refmods, 3000, W, H, 6, 31, iters)
    densify_at, reset_at = (10, 20), (25,)
    bg = torch.tensor([0.1, 0.2, 0.3], device=dev())
    rng = random.Random(7)
    order = [rng.randrange(len(cams)) for _ in range(iters + 1)]
    rounds = []
    flipped = None
    with R.deterministic():
        ref, ours = model(), model()
        optim.attach(ours)
        densify.attach(ours)
        ts = train.TrainStep(ours, cams, bg, opt)
        for it in range(1, iters + 1):
            cam = cams[order[it]]
            ref.update_learning_rate(it)
            pkg = refmods.render(cam, ref, opt, bg)
            image, vsp, vis, radii = pkg["render"], pkg["viewspace_points"], pkg["visibility_filter"], pkg["radii"]
            img, gt = image.cpu().double(), cam.original_image.cpu().double()      # float64: only our rounding
            loss = (1.0 - opt.lambda_dssim) * LO.l1_loss(img, gt) + opt.lambda_dssim * (1.0 - LO.ssim(img, gt))
            loss.backward()
            edit = it in densify_at or it in reset_at
            ts.run(it, order[it], stats=True, step=not edit and it < iters)
            with torch.no_grad():
                g_ref, g_our = ref._xyz.grad, ts.bucket.means3D
                if flipped is None or flipped.numel() != g_ref.shape[0]:
                    flipped = torch.zeros(g_ref.shape[0], dtype=torch.bool, device=dev())
                rn = g_ref.norm(dim=1)
                flipped |= ((g_our - g_ref).norm(dim=1) > 1e-2 * rn) & (rn > 1e-3 * rn.max())
                ref.max_radii2D[vis] = torch.max(ref.max_radii2D[vis], radii[vis])
                ref.add_densification_stats(vsp, vis)
                if edit:
                    torch.cuda.synchronize()
                    assert int(flipped.sum()) <= max(2, ref._xyz.shape[0] // 500), it
                    _assert_close(ref, ours, flipped, f"before the edit at {it}")
                    _anchor(ours, ref)             # the edit starts from the same state on both sides
                    flipped = None
                if it in densify_at:
                    before = [g["params"][0] for g in ours.optimizer.param_groups]
                    args = (0.0002, 0.005, 1.0, None) if it == 10 else (0.0002, 0.005, 1.0, 20)
                    torch.manual_seed(1000 + it)
                    ref.densify_and_prune(*args)
                    torch.manual_seed(1000 + it)
                    ours.densify_and_prune(*args)
                    torch.cuda.synchronize()
                    _assert_same(ref, ours, before, f"densify at {it}", same_optimiser=False)
                    rounds.append(ours._xyz.shape[0])
                if it in reset_at:
                    ref.reset_opacity()
                    ours.reset_opacity()
                    torch.cuda.synchronize()
                    assert torch.equal(ref._opacity, ours._opacity)
                if it < iters:
                    ref.optimizer.step()
                    ref.optimizer.zero_grad(set_to_none=True)
                    if edit:
                        ts.step_unchanged()
            torch.cuda.synchronize()
        ts.check()
        torch.cuda.synchronize()
    assert int(flipped.sum()) <= max(2, ref._xyz.shape[0] // 500)
    _assert_close(ref, ours, flipped, "final state")
    assert len(rounds) == 2 and rounds[0] != 3000
    assert ts.captures >= 3                  # initial, after each densify and after the opacity reset


def test_torch_rules_the_kernels_restate():
    """On the device, ATen divides by a CPU scalar through its float reciprocal, and torch.norm over a size-1 dim is
    |g|, also where g * g underflows or overflows: the split scaling and the clone test rely on both."""
    g = torch.Generator(device=dev()).manual_seed(9)
    s = torch.exp(torch.randn(1 << 20, device=dev(), generator=g) * 3)
    assert torch.equal(s / (0.8 * 2), s * (torch.tensor(1.0) / torch.tensor(1.6)).item())
    x = torch.cat([s * 1e-20, s * 1e18, torch.tensor([0.0, float("inf")], device=dev())])
    assert torch.equal(torch.norm(x[:, None], dim=-1), x.abs())
