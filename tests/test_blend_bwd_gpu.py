"""The backward tile pass (gs_blend_bwd.cu) reproduces, bit for bit, the deterministic backward's gradients pinned in
tests/golden/blend_bwd_digests.json.  The deterministic gradients are fixed-order sums of the per-(tile, splat)
partials that k_tile_partials stores, so equal gradients mean the pass stored the same partials.  The digests were
generated with both the shuffle-butterfly pass this one replaced and this pass, which gave identical files.  Each scene
runs in a process of its own (tests/golden/make_blend_bwd_digests.py)."""
import json
import os
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
SCENES = ("golden", "config3", "config3_x4", "frustum_1m_512")


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


def _run(scene, out):
    """Child process: forward + deterministic backward of every case of `scene`, gradients saved to `out`."""
    import torch
    from luciddreamer_b200 import rasterizer as R
    d = torch.device("cuda:0")
    res = {}
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


if __name__ == "__main__":
    _run(sys.argv[1], sys.argv[2])
