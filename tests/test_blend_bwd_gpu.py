"""The slab-reduction backward tile pass (gs_blend_bwd.cu, the default) against the shuffle-butterfly pass of gs_blend.cu
(GS_BLEND_BWD=0): on the same forward, the deterministic backward's gradients are fixed-order sums of the per-(tile,
splat) partials that k_tile_partials stores, so equal gradients mean the two passes stored the same partials.  The
switch is read when the library creates its context, so each pass runs in a process of its own."""
import os
import subprocess
import sys
import tempfile

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
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


def _grads(scene, arm, tmp):
    out = os.path.join(tmp, f"{scene}_{arm}.npz")
    env = dict(os.environ, GS_BLEND_BWD=arm,
               PYTHONPATH=os.pathsep.join([ROOT, os.path.join(ROOT, "tests")]))
    subprocess.run([sys.executable, "-s", os.path.abspath(__file__), scene, out], env=env, check=True, timeout=900)
    return np.load(out)


@pytest.mark.parametrize("scene", SCENES)
def test_slab_pass_stores_the_partials_of_the_butterfly_pass(scene):
    with tempfile.TemporaryDirectory() as tmp:
        old, new = _grads(scene, "0", tmp), _grads(scene, "1", tmp)
        assert sorted(old.files) == sorted(new.files) and old.files
        for k in old.files:
            a, b = old[k], new[k]
            assert a.shape == b.shape and np.array_equal(a, b), \
                (k, float(np.abs(a.astype(np.float64) - b).max()), int((a != b).sum()))


if __name__ == "__main__":
    _run(sys.argv[1], sys.argv[2])
