"""The deterministic backward on the GPU (rasterizer.deterministic / gs_backward_deterministic): gradients of one forward
are bit-identical from run to run and across schedules, capacities, graph replays and entry points; they equal the
atomic default where its sums have at most two terms; they match the golden fixtures, the CPU oracle and the default
path; a whole training run is reproducible from its seed."""
import math
import types

import numpy as np
import pytest
import torch

import cases
import util

pytestmark = pytest.mark.gpu

GOLDEN = [c for c in cases.CASES if c.golden]


def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return torch.device("cuda:0")


@pytest.fixture(autouse=True)
def _default_mode_after_each_test():
    from luciddreamer_b200 import rasterizer as R
    yield
    R.set_deterministic(False, 0)


def c_backward(args, fwd, cot, det):
    """All eight gradients of `_C.rasterize_gaussians_backward` on the buffers of forward `fwd`."""
    from luciddreamer_b200 import rasterizer as R
    (bg, means3D, colors, opacity, scales, rotations, mod, cov, vm, pm, tfx, tfy, H, W, sh, D, campos, _p, dbg) = args
    nr, color, depth, radii, geom, binning, img = fwd
    with R.deterministic(det):
        g = R._C.rasterize_gaussians_backward(bg, means3D, radii, colors, scales, rotations, mod, cov, vm, pm, tfx, tfy,
                                              cot, torch.zeros(1, H, W, device=cot.device), sh, D, campos, geom, nr,
                                              binning, img, dbg)
    return [t.clone() for t in g]


def autograd_forward(args, det):
    """GaussianRasterizer forward with leaves; the switch is read here, at forward time."""
    from luciddreamer_b200 import GaussianRasterizationSettings, GaussianRasterizer
    from luciddreamer_b200 import rasterizer as R
    (bg, means3D, colors, opacity, scales, rotations, mod, cov, vm, pm, tfx, tfy, H, W, sh, D, campos, _p, dbg) = args
    rs = GaussianRasterizationSettings(H, W, tfx, tfy, bg, mod, vm, pm, D, campos, _p, dbg)
    src = dict(means3D=means3D, opacities=opacity, shs=sh, colors_precomp=colors, scales=scales, rotations=rotations,
               cov3D_precomp=cov)
    leaves = {k: t.detach().requires_grad_(True) for k, t in src.items() if t.numel()}
    leaves["means2D"] = torch.zeros(means3D.size(0), 3, device=means3D.device, requires_grad=True)
    with R.deterministic(det):
        color, radii, depth = GaussianRasterizer(rs)(
            leaves["means3D"], leaves["means2D"], leaves["opacities"], shs=leaves.get("shs"),
            colors_precomp=leaves.get("colors_precomp"), scales=leaves.get("scales"), rotations=leaves.get("rotations"),
            cov3D_precomp=leaves.get("cov3D_precomp"))
    return color, radii, depth, leaves


def autograd_grads(color, leaves, cot):
    ks = sorted(leaves)
    g = torch.autograd.grad(color, [leaves[k] for k in ks], grad_outputs=cot, retain_graph=True)
    return dict(zip(ks, [t.clone() for t in g]))


def assert_all_equal(runs, what):
    for r in runs[1:]:
        assert len(r) == len(runs[0])
        for k in (r.keys() if isinstance(r, dict) else range(len(r))):
            a, b = runs[0][k], r[k]
            if a is None or not a.numel():
                continue
            assert torch.equal(a, b), f"{what}: gradient {k} differs between runs (max {float((a - b).abs().max()):.3e})"


def rel(a, b):
    return float((a.double() - b.double()).norm() / max(float(b.double().norm()), 1e-30))


AG_NAMES = dict(means3D="dL_dmeans3D", means2D="dL_dmeans2D", opacities="dL_dopacity", shs="dL_dsh",
                colors_precomp="dL_dcolors", scales="dL_dscales", rotations="dL_drotations", cov3D_precomp="dL_dcov3D")


def grad_names(case):
    names = set(cases.GRAD_NAMES)
    if case.precomp:
        names -= {"dL_dsh", "dL_dscales", "dL_drotations"}
    return names


# ---- 1 + 4: bit-reproducible, and parity (golden fixtures, default path, forward unchanged) -----------------------------

@pytest.mark.parametrize("case", GOLDEN, ids=[c.name for c in GOLDEN])
def test_C_entry_is_bit_reproducible_and_matches_golden(case):
    from luciddreamer_b200 import rasterizer as R
    inp = cases.build_inputs(case)
    args = cases.binding_args(inp, dev())
    cot = inp["cot"].to(dev())
    fwd = R._C.rasterize_gaussians(*args)
    runs = [c_backward(args, fwd, cot, True) for _ in range(3)]
    default = c_backward(args, fwd, cot, False)
    runs.append(c_backward(args, fwd, cot, True))          # after a default backward of the same forward
    torch.cuda.synchronize()
    assert_all_equal(runs, case.name)
    gold = util.load_golden(case.name)
    got = dict(zip(cases.GRAD_NAMES, [t.cpu().numpy() for t in runs[0]]))
    util.assert_grads_close(got, gold["grads"], names=grad_names(case), what=case.name)
    for k, (a, b) in enumerate(zip(runs[0], default)):
        if a.numel():
            assert rel(a, b) <= 1e-5, (case.name, cases.GRAD_NAMES[k], rel(a, b))


@pytest.mark.parametrize("case", GOLDEN, ids=[c.name for c in GOLDEN])
def test_autograd_entry_is_bit_reproducible_and_forward_unchanged(case):
    inp = cases.build_inputs(case)
    args = cases.binding_args(inp, dev())
    cot = inp["cot"].to(dev())
    color0, radii0, depth0, leaves0 = autograd_forward(args, False)
    default = autograd_grads(color0, leaves0, cot)
    color, radii, depth, leaves = autograd_forward(args, True)
    torch.cuda.synchronize()
    assert torch.equal(color, color0) and torch.equal(depth, depth0) and torch.equal(radii, radii0)
    runs = [autograd_grads(color, leaves, cot) for _ in range(3)]
    torch.cuda.synchronize()
    assert_all_equal(runs, case.name)
    gold = util.load_golden(case.name)
    got = {AG_NAMES[k]: v.cpu().numpy() for k, v in runs[0].items()}
    util.assert_grads_close(got, gold["grads"], names=grad_names(case), what=case.name)
    for k in runs[0]:
        assert rel(runs[0][k], default[k]) <= 1e-5, (case.name, k)


@pytest.mark.parametrize("name", ["opaque_40k_64_x8", "frustum_20k_96", "frustum_60k_64_bg"] + [c.name for c in cases.BLOCK_CASES])
def test_matches_cpu_oracle(name):
    """Behind strip partials (k_tile_partials<1>) and, for cases.BLOCK_CASES, behind block partials (k_tile_partials<2>)."""
    from oracle import oracle
    case = cases.BY_NAME[name]
    if case in cases.BLOCK_CASES:
        assert util.blend_rows_per_warp(case.W, case.H) == 8
    inp = cases.build_inputs(case)
    f = oracle.rasterize_gaussians(*cases.binding_args(inp))
    og = dict(zip(cases.GRAD_NAMES, oracle.rasterize_gaussians_backward(f, inp["cot"].numpy())[:8]))
    color, radii, depth, leaves = autograd_forward(cases.binding_args(inp, dev()), True)
    g = {AG_NAMES[k]: v.cpu().numpy() for k, v in autograd_grads(color, leaves, inp["cot"].to(dev())).items()}
    if "needles" in name:
        # beyond fp32 conditioning (test_parity_gpu._check_ill_conditioned): the fp64 oracle is the bar and the fp32
        # oracle's own distance from it the yardstick
        t = oracle.rasterize_gaussians(*cases.binding_args(inp)[:17], mode="f64")
        og64 = dict(zip(cases.GRAD_NAMES, oracle.rasterize_gaussians_backward(t, inp["cot"].numpy())[:8]))
        for k in grad_names(case) & g.keys():
            e_ref, e_our = util.rel_err(og[k], og64[k]), util.rel_err(g[k].reshape(og64[k].shape), og64[k])
            assert e_our <= max(util.GRAD_REL_TOL, 10 * e_ref), f"{name}: {k} rel err {e_our:.3e} vs fp64 (fp32 oracle: {e_ref:.3e})"
        return
    util.assert_grads_close(g, og, names=grad_names(case), what=name)


def _full_size(kind):
    from luciddreamer_b200 import synthetic as syn
    d = dev()
    if kind == "frustum":
        P, W, H = 1_000_000, 512, 512
        sc = syn.make_frustum_scene(P, 2001, W, H, raster=True)
    else:
        P, W, H = 1_000_000, 1920, 1080
        sc = syn.make_scene(P, 1003, scale_mult=kind)
    sc = {k: v.to(d) for k, v in sc.items()}
    cam = syn.make_camera(W, H)
    e = torch.empty(0)
    args = (torch.zeros(3, device=d), sc["means3D"], e, sc["opacities"], sc["scales"], sc["rotations"], 1.0, e,
            cam.viewmatrix.to(d), cam.projmatrix.to(d), cam.tanfovx, cam.tanfovy, H, W, sc["shs"], 3, cam.campos.to(d),
            False, False)
    return args, syn.make_cotangent(H, W, 1003).to(d)


@pytest.mark.parametrize("kind", [1.0, 4.0, "frustum"], ids=["config3", "config3_x4", "frustum_1M_512"])
def test_full_size_bit_reproducible_both_entries(kind):
    """Config 3 (sparse regime; x4: rects of more than 32 tiles and long tile lists) and the 1 M LucidDreamer-shaped
    scene at 512x512 (dense regime, 16x4 strips)."""
    from luciddreamer_b200 import rasterizer as R
    args, cot = _full_size(kind)
    fwd = R._C.rasterize_gaussians(*args)
    runs = [c_backward(args, fwd, cot, True) for _ in range(3)]
    default = c_backward(args, fwd, cot, False)
    torch.cuda.synchronize()
    assert_all_equal(runs, f"C {kind}")
    for k, (a, b) in enumerate(zip(runs[0], default)):
        if a.numel():
            assert rel(a, b) <= 1e-5, (kind, cases.GRAD_NAMES[k], rel(a, b))
    del fwd, runs, default
    color, radii, depth, leaves = autograd_forward(args, True)
    runs = [autograd_grads(color, leaves, cot) for _ in range(3)]
    torch.cuda.synchronize()
    assert_all_equal(runs, f"autograd {kind}")


# ---- 2: independent of schedule and capacity ----------------------------------------------------------------------------

def test_independent_of_capacity_graph_bucket_and_concurrent_work():
    from luciddreamer_b200 import GaussianRasterizationSettings, GaussianRasterizer
    from luciddreamer_b200 import multiview as MV
    from luciddreamer_b200 import rasterizer as R
    from luciddreamer_b200.graphs import GraphedStep
    case = cases.BY_NAME["cfg2_100k_512"]
    inp = cases.build_inputs(case)
    d = dev()
    cam = inp["cam"]
    rs = GaussianRasterizationSettings(cam.image_height, cam.image_width, cam.tanfovx, cam.tanfovy, inp["bg"].to(d),
                                       case.scale_modifier, cam.viewmatrix.to(d), cam.projmatrix.to(d), case.D,
                                       cam.campos.to(d), False, False)
    names = ("means3D", "shs", "opacities", "scales", "rotations")
    leaves = {k: inp[k].to(d).requires_grad_(True) for k in names}
    m2 = torch.zeros(case.P, 3, device=d, requires_grad=True)
    cot = inp["cot"].to(d)
    rast = GaussianRasterizer(rs)

    def step():
        for t in list(leaves.values()) + [m2]:
            t.grad = None
        color, _r, _d = rast(leaves["means3D"], m2, leaves["opacities"], shs=leaves["shs"], scales=leaves["scales"],
                             rotations=leaves["rotations"])
        torch.autograd.backward(color, grad_tensors=cot)
        return color.detach()

    def grads():
        return [leaves[k].grad.clone() for k in names] + [m2.grad.clone()]

    R.set_deterministic(True, 0)
    step(); torch.cuda.synchronize()
    ref, pairs = grads(), R._last_pairs[0]
    variants = {}
    for cap in (pairs + 1000, 3 * pairs + 50_000):
        with R.static_capacity(cap):
            step()
        R.check_static()
        variants[f"static {cap}"] = grads()
    g = GraphedStep(step, warmup=2)
    g.replay(); g.check()
    variants["graph replay"] = grads()
    g.release()                       # check_static() of later tests must not re-read this graph's status slot
    params = {k: leaves[k].detach() for k in names}
    _c, _d, _r, bucket, dm2 = MV.view_step(params, rs, cot)
    torch.cuda.synchronize()
    variants["view_step"] = [bucket.means3D, bucket.shs, bucket.opacities, bucket.scales, bucket.rotations, dm2]
    # one run while a heavy torch workload occupies another stream
    side = torch.cuda.Stream()
    a = torch.randn(4096, 4096, device=d)
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(8):
            a = torch.tanh(a @ a * 1e-3)
    step()
    torch.cuda.synchronize()
    variants["concurrent stream"] = grads()
    for what, gs in variants.items():
        for k, (x, y) in enumerate(zip(gs, ref)):
            assert torch.equal(x, y), f"{what}: gradient {k} differs (max {float((x - y).abs().max()):.3e})"


# ---- 3: exact against the default path where the default path is exact ------------------------------------------------

def test_equals_default_when_every_gaussian_is_binned_in_at_most_two_tiles():
    """Splats of radius <= 7 px centred on tile columns (x = 16k + 8) cover one tile column and at most two tile rows:
    every accumulator sum has at most two terms, which float addition makes order-independent, so the atomic default is
    exact there and the stored partials must reproduce it bit for bit."""
    import ctypes as C
    from luciddreamer_b200 import _native as N
    from luciddreamer_b200 import rasterizer as R
    from luciddreamer_b200 import synthetic as syn
    d = dev()
    P, W, H = 40_000, 256, 256
    sc = syn.make_frustum_scene(P, 77, W, H, sigma_px=0.8)
    tx = math.tan(syn.REF_FOVX / 2)
    g = torch.Generator().manual_seed(78)
    k = torch.randint(0, W // 16, (P,), generator=g).double()
    u = (2.0 * (16.0 * k + 8.0) + 1.0) / W - 1.0                # ndc x of pixel column 16k + 8
    z = sc["means3D"][:, 2].double()
    sc["means3D"][:, 0] = (u * tx * z).float()
    focal_px = W / (2.0 * tx)
    sc["scales"] = torch.minimum(sc["scales"], (z * (1.5 / focal_px)).float()[:, None])   # sigma <= 1.5 px: radius <= 5
    sc = {k2: v.contiguous().to(d) for k2, v in sc.items()}
    cam = syn.make_camera(W, H)
    e = torch.empty(0)
    args = (torch.zeros(3, device=d), sc["means3D"], e, sc["opacities"], sc["scales"], sc["rotations"], 1.0, e,
            cam.viewmatrix.to(d), cam.projmatrix.to(d), cam.tanfovx, cam.tanfovy, H, W, sc["shs"], 3, cam.campos.to(d),
            False, False)
    fwd = R._C.rasterize_gaussians(*args)
    nr, color, depth, radii, geom, binning, img = fwd
    # the property itself, from the binned pair list
    cap = binning.numel() // 12
    G = (W // 16) * (H // 16)
    ranges = torch.zeros(G + 1, dtype=torch.int32, device=d)
    plist = torch.zeros(cap, dtype=torch.int32, device=d)
    f = N.GsFrame()
    f.W, f.H = W, H
    N.check(N.lib().gs_debug_export_binning(C.byref(f), binning.data_ptr(), cap, img.data_ptr(), ranges.data_ptr(),
                                            plist.data_ptr(), cap, R._raw_stream(0)))
    torch.cuda.synchronize()
    npairs = int(ranges[-1])
    per = torch.bincount(plist[:npairs].long(), minlength=P)
    assert int(per.max()) <= 2 and int((per == 2).sum()) > 1000, (int(per.max()), int((per == 2).sum()))
    cot = syn.make_cotangent(H, W, 5).to(d)
    det = c_backward(args, fwd, cot, True)
    default = c_backward(args, fwd, cot, False)
    torch.cuda.synchronize()
    for k2, (a, b) in enumerate(zip(det, default)):
        if a.numel():
            assert torch.equal(a, b), (cases.GRAD_NAMES[k2], float((a - b).abs().max()))


# ---- 5: a training run is reproducible ----------------------------------------------------------------------------------

def _train(seed, iters=10, P=200_000, W=256, H=256):
    from luciddreamer_b200 import GaussianRasterizationSettings, GaussianRasterizer
    from luciddreamer_b200 import losses, multiview as MV, optim
    from luciddreamer_b200 import synthetic as syn
    d = dev()
    sc = syn.make_frustum_scene(P, seed, W, H, raster=True)
    xyz = sc["means3D"].to(d).contiguous()
    f_dc = sc["shs"][:, :1].to(d).contiguous()
    f_rest = sc["shs"][:, 1:].to(d).contiguous()
    opacity = torch.logit(sc["opacities"].clamp(1e-4, 1 - 1e-4)).to(d).contiguous()
    scaling = torch.log(sc["scales"]).to(d).contiguous()
    rotation = sc["rotations"].to(d).contiguous()
    opt = optim.FusedGaussianAdam(xyz, f_dc, f_rest, opacity, scaling, rotation)
    stats = MV.DensifyStats(P, d)
    poses = syn.jitter_poses(8, seed)
    rng = np.random.RandomState(seed)
    gt = torch.rand(3, H, W, generator=torch.Generator().manual_seed(seed)).to(d)
    for it in range(iters):
        cam = syn.make_camera(W, H, c2w=poses[rng.randint(len(poses))])
        rs = GaussianRasterizationSettings(H, W, cam.tanfovx, cam.tanfovy, torch.zeros(3, device=d), 1.0,
                                           cam.viewmatrix.to(d), cam.projmatrix.to(d), 3, cam.campos.to(d), False, False)
        act = dict(means3D=xyz.detach().clone(), shs=torch.cat([f_dc, f_rest], 1).detach(),
                   opacities=torch.sigmoid(opacity).detach(), scales=torch.exp(scaling).detach(),
                   rotations=torch.nn.functional.normalize(rotation).detach())
        for t in act.values():
            t.requires_grad_(True)
        m2 = torch.zeros(P, 3, device=d, requires_grad=True)
        image, radii, _depth = GaussianRasterizer(rs)(act["means3D"], m2, act["opacities"], shs=act["shs"],
                                                      scales=act["scales"], rotations=act["rotations"])
        losses.photometric_loss(image, gt, 0.2).backward()
        stats.add_view(m2.grad, radii)
        opt.step(types.SimpleNamespace(**{k: t.grad.contiguous() for k, t in act.items()}))
    torch.cuda.synchronize()
    out = {f"param {k}": t.clone() for k, t in opt.params.items()}
    out.update({f"exp_avg {k}": t.clone() for k, t in opt.exp_avg.items()})
    out.update({f"exp_avg_sq {k}": t.clone() for k, t in opt.exp_avg_sq.items()})
    out.update(xyz_gradient_accum=stats.xyz_gradient_accum.clone(), denom=stats.denom.clone(),
               max_radii2D=stats.max_radii2D.clone())
    return out


def test_training_run_is_reproducible_from_its_seed():
    from luciddreamer_b200 import rasterizer as R
    with R.deterministic():
        a = _train(4242)
        b = _train(4242)
    assert float(a["denom"].sum()) > 0
    for k in a:
        assert torch.equal(a[k], b[k]), f"{k} differs between two runs from one seed"


# ---- 6: edge cases ------------------------------------------------------------------------------------------------------

def test_overflowed_static_capacity_gives_zero_gradients_and_the_deferred_error():
    from luciddreamer_b200 import GaussianRasterizationSettings, GaussianRasterizer
    from luciddreamer_b200 import rasterizer as R
    case = cases.BY_NAME["rot40_5k_128x72"]
    inp = cases.build_inputs(case)
    d = dev()
    cam = inp["cam"]
    rs = GaussianRasterizationSettings(cam.image_height, cam.image_width, cam.tanfovx, cam.tanfovy, inp["bg"].to(d), 1.0,
                                       cam.viewmatrix.to(d), cam.projmatrix.to(d), case.D, cam.campos.to(d), False, False)
    leaves = {k: inp[k].to(d).requires_grad_(True) for k in ("means3D", "shs", "opacities", "scales", "rotations")}
    m2 = torch.zeros(case.P, 3, device=d, requires_grad=True)

    def step():
        color, _r, _d = GaussianRasterizer(rs)(leaves["means3D"], m2, leaves["opacities"], shs=leaves["shs"],
                                               scales=leaves["scales"], rotations=leaves["rotations"])
        torch.autograd.backward(color, grad_tensors=inp["cot"].to(d))

    with R.deterministic():
        step(); torch.cuda.synchronize()
        pairs = R._last_pairs[0]
        for t in list(leaves.values()) + [m2]:
            t.grad = None
        with R.static_capacity(max(64, pairs // 3)):
            step()
        torch.cuda.synchronize()
        for t in list(leaves.values()) + [m2]:
            assert float(t.grad.abs().max()) == 0.0
        with pytest.raises(RuntimeError, match="static pair capacity"):
            R.check_static()


def test_zero_gaussians():
    from luciddreamer_b200 import rasterizer as R
    d = dev()
    cam = cases.build_inputs(cases.BY_NAME["micro_1k_64"])["cam"]
    e = torch.zeros(0, 3, device=d)
    args = (torch.ones(3, device=d), e, torch.empty(0), torch.zeros(0, 1, device=d), e, torch.zeros(0, 4, device=d), 1.0,
            torch.empty(0), cam.viewmatrix.to(d), cam.projmatrix.to(d), cam.tanfovx, cam.tanfovy, 64, 64,
            torch.zeros(0, 16, 3, device=d), 3, cam.campos.to(d), False, False)
    fwd = R._C.rasterize_gaussians(*args)
    g = c_backward(args, fwd, torch.ones(3, 64, 64, device=d), True)
    torch.cuda.synchronize()
    assert g[0].shape == (0, 3) and g[3].shape == (0, 3)


def test_peer_reduce_is_rejected():
    from luciddreamer_b200 import GaussianRasterizationSettings
    from luciddreamer_b200 import multiview as MV
    from luciddreamer_b200 import rasterizer as R
    case = cases.BY_NAME["micro_1k_64"]
    inp = cases.build_inputs(case)
    d = dev()
    args = cases.binding_args(inp, d)
    (bg, means3D, colors, opacity, scales, rotations, mod, cov, vm, pm, tfx, tfy, H, W, sh, D, campos, _p, dbg) = args
    rs = GaussianRasterizationSettings(H, W, tfx, tfy, bg, mod, vm, pm, D, campos, False, False)
    params = dict(means3D=means3D, shs=sh, opacities=opacity, scales=scales, rotations=rotations)
    fake = MV.SymmGradBucket.__new__(MV.SymmGradBucket)          # the check comes before the bucket is touched
    with R.deterministic():
        n0 = R._last_pairs.get(0)
        with pytest.raises(RuntimeError, match="SymmGradBucket"):
            MV.view_step(params, rs, inp["cot"].to(d), bucket=fake)
        assert R._last_pairs.get(0) == n0                        # nothing was launched
    # the binding / C ABI refuse a peer backward in deterministic mode
    nr, color, depth, radii, geom, binning, img, cap, nvis, _pairs, _t = R._forward(*args[:17], False, False)
    dummy = torch.zeros(1 << 16, device=d)
    with pytest.raises(RuntimeError, match="peer"):
        R._binding().backward(R._ctx(0).value, bg, means3D, colors, opacity, scales, rotations, mod, cov, vm, pm, tfx, tfy,
                              H, W, sh, D, campos, False, radii, geom, binning, img, cap, nvis, inp["cot"].to(d), False,
                              False, peer_buckets=[dummy.data_ptr()], peer_seg_off=[0, 0, 0, 0, 0], deterministic=True)
