"""The backward tile pass (gs_blend_bwd.cu) reproduces, bit for bit, the deterministic backward's gradients pinned in
tests/golden/blend_bwd_digests.json.  The deterministic gradients are fixed-order sums of the per-(tile, splat)
partials that k_tile_partials stores, so equal gradients mean the pass stored the same partials.  The digests were
generated with both the shuffle-butterfly pass this one replaced and this pass, which gave identical files.  Each scene
runs in a process of its own (tests/golden/make_blend_bwd_digests.py).

The scenes above go through the `_C` surface, which always takes k_grad_vis + k_grad_write.  ROUTES drive every other
single-GPU route of the per-Gaussian backward (gs_gauss_bwd.cu) in deterministic mode: the autograd node with the
reference's input mode (sparse, P % 4 != 0, dense, static capacity), with precomputed colours or covariances, and
multiview.view_step into a GradBucket.  Each route pins its gradients and the set of backward kernel slots that launched
(gs_profile_read), so a change to the host's choice of writers shows up even where the gradients would not."""
import json
import os
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
SCENES = ("golden", "config3", "config3_x4", "frustum_1m_512")
ROUTES = ("node_config3", "node_config3_p_odd", "node_frustum_200k_256", "node_colors_precomp", "node_cov3D_precomp",
          "node_config3_static", "view_step_bucket")
BWD_SLOTS = ("k_blend_bwd", "k_fill_zero", "k_grad_vis", "k_grad_write", "k_grad_dense")


def _scene_args(name, d):
    """(case name, binding args, cotangent) of every case the scene stands for."""
    import torch
    import cases
    from luciddreamer_b200 import synthetic as syn
    if name == "golden":
        for c in (c for c in cases.CASES if c.golden):
            inp = cases.build_inputs(c)
            yield c.name, cases.binding_args(inp, d), inp["cot"].to(d)
        return
    if name == "frustum_1m_512":                 # 16x4 strips (NH = 1): 1024 tiles
        W = H = 512
        sc = syn.make_frustum_scene(1_000_000, 1003, W, H)
    else:
        c = syn.CONFIGS[3]
        W, H = c["W"], c["H"]
        sc = syn.make_scene(c["P"], 1003, scale_mult=4.0 if name == "config3_x4" else 1.0)
    sc = {k: v.contiguous().to(d) for k, v in sc.items()}
    cam = syn.make_camera(W, H)
    e = torch.empty(0, device=d)
    args = (torch.zeros(3, device=d), sc["means3D"], e, sc["opacities"], sc["scales"], sc["rotations"], 1.0, e,
            cam.viewmatrix.to(d), cam.projmatrix.to(d), cam.tanfovx, cam.tanfovy, H, W, sc["shs"], 3, cam.campos.to(d),
            False, False)
    yield name, args, syn.make_cotangent(H, W, 5).to(d)


def _route(name, d, res):
    """Forward + deterministic backward of route `name`, its gradients added to `res`.  Returns the sorted names of the
    backward kernel slots that launched."""
    import ctypes as C
    import torch
    import cases
    from luciddreamer_b200 import _native as N, multiview as MV, rasterizer as R, synthetic as syn
    if name == "node_frustum_200k_256":          # dense regime: nearly every Gaussian visible
        W = H = 256
        sc = syn.make_frustum_scene(200_000, 1003, W, H)
    else:
        c = syn.CONFIGS[3]
        W, H = c["W"], c["H"]
        sc = syn.make_scene(c["P"], 1003)
    if name == "node_config3_p_odd":
        sc = {k: v[:-1] for k, v in sc.items()}
    if name == "node_colors_precomp":
        sc["colors_precomp"] = torch.rand(sc.pop("shs").shape[0], 3, generator=torch.Generator().manual_seed(1004))
    if name == "node_cov3D_precomp":
        sc["cov3D_precomp"] = cases.cov3D_of(sc.pop("scales"), sc.pop("rotations"))
    leaves = {k: v.contiguous().to(d).requires_grad_(True) for k, v in sc.items()}
    P = leaves["means3D"].shape[0]
    m2 = torch.zeros(P, 3, device=d, requires_grad=True)
    cam = syn.make_camera(W, H)
    rs = R.GaussianRasterizationSettings(H, W, cam.tanfovx, cam.tanfovy, torch.zeros(3, device=d), 1.0,
                                         cam.viewmatrix.to(d), cam.projmatrix.to(d), 3, cam.campos.to(d), False, False)
    cot = syn.make_cotangent(H, W, 5).to(d)

    def node():
        return R.rasterize_gaussians(leaves["means3D"], m2, leaves.get("shs"), leaves.get("colors_precomp"),
                                     leaves["opacities"], leaves.get("scales"), leaves.get("rotations"),
                                     leaves.get("cov3D_precomp"), rs)[0]

    L, ctx = N.lib(), R._ctx(d.index)
    names = [L.gs_profile_kernel_name(i).decode() for i in range(L.gs_profile_num_kernels())]
    with R.deterministic(True):
        if name == "node_config3_static":        # the host does not learn num_visible: the dense kernel is launched
            with torch.no_grad():
                node()
            cap = R._last_pairs[d.index]
            N.check(L.gs_profile_enable(ctx, 1))
            with R.static_capacity(cap):
                torch.autograd.backward(node(), grad_tensors=cot)
            R.check_static(d)
        elif name == "view_step_bucket":
            N.check(L.gs_profile_enable(ctx, 1))
            params = {k: v.detach() for k, v in leaves.items()}
            *_, bucket, dm2 = MV.view_step(params, rs, cot, bucket=MV.GradBucket(P, params["shs"].shape[1], d))
            grads = dict(means3D=bucket.means3D, shs=bucket.shs, opacities=bucket.opacities, scales=bucket.scales,
                         rotations=bucket.rotations, means2D=dm2)
        else:
            N.check(L.gs_profile_enable(ctx, 1))
            torch.autograd.backward(node(), grad_tensors=cot)
    if name != "view_step_bucket":
        grads = dict({k: v.grad for k, v in leaves.items()}, means2D=m2.grad)
    torch.cuda.synchronize()
    ms = (C.c_float * len(names))()
    N.check(L.gs_profile_read(ctx, ms))
    N.check(L.gs_profile_enable(ctx, 0))
    for k, t in grads.items():
        res[f"{name}/{k}"] = t.cpu().numpy()
    return sorted(n for n, t in zip(names, ms) if t >= 0 and n in BWD_SLOTS)


def _run(scene, out):
    """Child process: forward + deterministic backward of every case of `scene` (or of the route `scene`), gradients
    saved to `out`; a route's launched backward slots go to `out` with the suffix .json."""
    import torch
    from luciddreamer_b200 import rasterizer as R
    d = torch.device("cuda:0")
    res = {}
    if scene in ROUTES:
        launched = _route(scene, d, res)
        np.savez(out, **res)
        with open(out + ".json", "w") as f:
            json.dump(launched, f)
        return
    for name, args, cot in _scene_args(scene, d):
        (bg, means3D, colors, opacity, scales, rotations, mod, cov, vm, pm, tfx, tfy, H, W, sh, D, campos, _p, dbg) = args
        nr, color, depth, radii, geom, binning, img = R._C.rasterize_gaussians(*args)
        with R.deterministic(True):
            g = R._C.rasterize_gaussians_backward(bg, means3D, radii, colors, scales, rotations, mod, cov, vm, pm, tfx,
                                                  tfy, cot, torch.zeros(1, H, W, device=d), sh, D, campos, geom, nr,
                                                  binning, img, dbg)
        torch.cuda.synchronize()
        for k, t in enumerate(g):
            if t.numel():
                res[f"{name}/{k}"] = t.cpu().numpy()
    np.savez(out, **res)


@pytest.mark.parametrize("scene", SCENES)
def test_slab_pass_stores_the_partials_of_the_butterfly_pass(scene):
    sys.path.insert(0, GOLDEN)
    try:
        import make_blend_bwd_digests as D
    finally:
        sys.path.remove(GOLDEN)
    gold = json.load(open(os.path.join(GOLDEN, "blend_bwd_digests.json")))
    want, have = gold["scenes"][scene], D.digests(scene)
    assert want and sorted(have) == sorted(want)
    for k in want:
        assert have[k] == want[k], (k, have[k], want[k], gold["card"])


@pytest.mark.parametrize("route", ROUTES)
def test_every_route_launches_its_writers_and_reproduces_its_gradients(route):
    sys.path.insert(0, GOLDEN)
    try:
        import make_blend_bwd_digests as D
    finally:
        sys.path.remove(GOLDEN)
    gold = json.load(open(os.path.join(GOLDEN, "blend_bwd_digests.json")))
    want, have = gold["routes"][route], D.route_record(route)
    assert have["launched"] == want["launched"], (have["launched"], want["launched"])
    assert want["digests"] and sorted(have["digests"]) == sorted(want["digests"])
    for k in want["digests"]:
        assert have["digests"][k] == want["digests"][k], (k, have["digests"][k], want["digests"][k], gold["card"])


if __name__ == "__main__":
    _run(sys.argv[1], sys.argv[2])
