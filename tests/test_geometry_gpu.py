"""Where the tile passes change shape (run with -m gpu on an H100), all against the CPU oracle on the same inputs:
  * ragged image borders in both geometries of the blend kernels (16x4 strips, 16x8 blocks; the library is asked which
    one a size runs in), down to images smaller than a tile, with a cotangent that lives on the border alone;
  * tile grids that need one, two or many rounds of the 4 096-tile scan, and long per-tile lists in a later round;
  * a block-geometry step under a static capacity and in a CUDA graph replayed with a second camera.
The block-geometry versions of the oracle-only scenes are cases.BLOCK_CASES, run by test_parity_gpu and
test_deterministic_gpu."""

import numpy as np
import pytest
import torch

import cases
import flip_audit
import util
from test_parity_gpu import _training_step_fixture, dev, grad_names, image_state, run

pytestmark = pytest.mark.gpu

BG = (0.3, 0.6, 0.9)
SCAN_ROUND = 4096                      # tiles per round of the scan (csrc/gs_preprocess.cu: cta_tile_scan<256, 16>)


def c_backward(args, r, cot, det=False):
    """All eight gradients for cotangent `cot` on the buffers of the `_C` forward `r`."""
    from luciddreamer_b200 import rasterizer as R
    (bg, means3D, colors, _op, scales, rotations, mod, cov, vm, pm, tfx, tfy, H, W, sh, D, campos, _p, dbg) = args
    geom, binning, img = r["bufs"]
    with R.deterministic(det):
        g = R._C.rasterize_gaussians_backward(bg, means3D, r["radii"], colors, scales, rotations, mod, cov, vm, pm, tfx, tfy,
                                              cot.to(dev()), torch.zeros(1, H, W, device=dev()), sh, D, campos, geom,
                                              r["num_rendered"], binning, img, dbg)
    torch.cuda.synchronize()
    return dict(zip(cases.GRAD_NAMES, [t.cpu().numpy() for t in g]))


def edge_mask(W, H):
    """The pixels of the last tile row and the last tile column."""
    m = np.zeros((H, W), bool)
    m[(H - 1) // 16 * 16:, :] = True
    m[:, (W - 1) // 16 * 16:] = True
    return m


def check_forward(case, f, r, edge=None):
    """The `_C` forward `r` against the oracle's forward state `f`: pair count and radii exact, colour / depth within
    tolerance with every outlier attributed to a branch flip, final_T as test_cuda_matches_cpu_oracle checks it.  Inside
    `edge` a pixel that differs in colour, depth OR final_T must have a branch operand on its threshold: the image-wide
    allowance does not cover a border defect.  Returns the mask of pixels that differ (branch flips)."""
    H, W = case.H, case.W
    color, depth, radii = (r[k].cpu().numpy() for k in ("color", "depth", "radii"))
    assert r["num_rendered"] == f.num_rendered
    assert np.array_equal(radii, f.radii)
    util.assert_forward_close(color, depth, radii, dict(color=f.color, depth=f.depth, radii=f.radii), what=case.name, audit=f)
    fT, _nc = image_state(r, H, W)
    bad_T = np.abs(fT - f.final_T) > 1e-5
    assert int(bad_T.sum()) <= H * W // 20000, f"{case.name}: final_T differs on {int(bad_T.sum())} pixels"
    flip = bad_T | (np.abs(color - f.color).max(axis=0) > util.FWD_ABS_TOL) | (np.abs(depth - f.depth)[0] > util.FWD_ABS_TOL)
    if edge is not None:
        for y, x in zip(*(a.tolist() for a in np.nonzero(flip & edge))):
            m = flip_audit.pixel_margins(f, x, y)
            assert flip_audit.near_thresholds(m), f"{case.name}: border pixel ({x}, {y}) differs, no branch operand near a threshold: {m}"
    return flip


# ---- a. ragged borders ---------------------------------------------------------------------------------------------------
# Blocks: a thread owns rows pyb, pyb+2, pyb+4, pyb+6 of its warp's 8; an odd H % 16 splits a thread's pair of rows
# between the image and the outside, H % 16 <= 8 leaves the lower warp of the last tile row without a live pixel.

RESIDUES = [(rw, rh) for rh in (1, 2, 3, 5, 7, 8, 9, 15) for rw in (0, 1, 8, 15)]
BORDER_SIZES = ([(704 + rw, 528 + rh, 8) for rw, rh in RESIDUES] + [(320 + rw, 240 + rh, 4) for rw, rh in RESIDUES]
                + [(1, 1, 4), (17, 5, 4), (5, 33, 4), (15, 31, 4), (16, 16, 4), (300, 1, 4)])      # below a tile / a strip


@pytest.mark.parametrize("W,H,rows", BORDER_SIZES, ids=[f"{w}x{h}" for w, h, _ in BORDER_SIZES])
def test_ragged_borders_in_both_geometries(W, H, rows):
    from oracle import oracle
    case = cases.Case(f"border_{W}x{H}", 40_000, W, H, 3, 41, scale_mult=2.0, bg=BG, golden=False)
    inp = cases.build_inputs(case)
    assert util.blend_rows_per_warp(W, H) == rows
    f = oracle.rasterize_gaussians(*cases.binding_args(inp))
    args = cases.binding_args(inp, dev())
    r = run("C", args)
    edge = edge_mask(W, H)
    flip = check_forward(case, f, r, edge)
    # backward on that forward: the full cotangent, and one that is zero off the last tile row and column -- a gradient
    # that leaks from a pixel outside the image, or is lost from one inside, is then not diluted by the rest of the image.
    # A pixel whose traversal flipped a branch legitimately has another gradient: it gets no cotangent on either side.
    keep = torch.from_numpy(~flip)
    for what, mask in (("full", keep), ("border", keep & torch.from_numpy(edge))):
        cot = (inp["cot"] * mask).contiguous()
        og = dict(zip(cases.GRAD_NAMES, oracle.rasterize_gaussians_backward(f, cot.numpy())[:8]))
        for det in ((False,) if what == "full" else (False, True)):
            util.assert_grads_close(c_backward(args, r, cot, det), og, names=grad_names(case),
                                    what=f"{case.name}, {what} cotangent, deterministic={det}")
    if W * H >= 20000:
        assert np.abs(og["dL_dmeans3D"]).max() > 0 and np.abs(og["dL_dsh"]).max() > 0      # the border sees Gaussians


# ---- b. rounds of the tile scan ---------------------------------------------------------------------------------------------
# One CTA scans the tile counts 4 096 at a time (256 threads x 16 tiles, 128-bit accesses when a thread's 16 tiles all
# exist, scalar ones for the thread that straddles the end) and carries the running total from round to round.

SCAN_GRIDS = [(1024, 1024),            # 64 x 64 = 4 096: exactly one round
              (1008, 1040),            # 63 x 65 = 4 095: the last thread of the round straddles the end
              (272, 3856),             # 17 x 241 = 4 097: a second round of one tile
              (1904, 1080),            # 119 x 68 = 8 092: two rounds, a straddling thread in the second
              (3840, 2160),            # 240 x 135 = 32 400: eight rounds
              (8192, 16)]              # one tile row


def grid_of(W, H):
    return (W + 15) // 16, (H + 15) // 16


@pytest.mark.parametrize("W,H", SCAN_GRIDS, ids=[f"{w}x{h}" for w, h in SCAN_GRIDS])
def test_tile_scan_rounds(W, H):
    from luciddreamer_b200 import rasterizer as R
    from oracle import oracle
    case = cases.Case(f"scan_{W}x{H}", 20_000, W, H, 1, 43, bg=BG, golden=False)
    inp = cases.build_inputs(case)
    f = oracle.rasterize_gaussians(*cases.binding_args(inp))
    r = run("C", cases.binding_args(inp, dev()))
    gx, gy = grid_of(W, H)
    print(f"{gx} x {gy} = {gx * gy} tiles, {util.blend_rows_per_warp(W, H)} rows per warp, {f.num_rendered} pairs")
    lens = util.assert_binning_matches_oracle(f, W, H, r["bufs"][1], r["bufs"][2], num_pairs=R._last_pairs[0])
    assert lens.sum() > 100
    if gx * gy > SCAN_ROUND + 1:                     # 4 097 tiles: the one tile of round two is an empty corner
        assert lens[SCAN_ROUND:].sum() > 0
    check_forward(case, f, r)


# ---- c. long lists beyond the first round ------------------------------------------------------------------------------------

def cluster(cam, n, cx, cy, seed, sigma_px=4.0):
    """n Gaussians of ~sigma_px pixels whose centres project within 3 px of the tile corner (cx, cy) of the identity
    camera `cam`: each lands in the four tiles around the corner.  Faint (alpha <= 0.04), depth ties included."""
    g = torch.Generator().manual_seed(seed)
    W, H = cam.image_width, cam.image_height
    z = torch.rand(n, generator=g) * 2 + 1
    z[1::7] = z[0::7][: z[1::7].shape[0]]                                   # bit-identical depths
    px = cx + (torch.rand(n, generator=g) - 0.5) * 6
    py = cy + (torch.rand(n, generator=g) - 0.5) * 6
    means = torch.stack([((2 * px + 1) / W - 1) * cam.tanfovx * z, ((2 * py + 1) / H - 1) * cam.tanfovy * z, z], 1)
    focal = W / (2 * cam.tanfovx)
    scales = (sigma_px * z / focal)[:, None] * (1 + 0.2 * torch.rand(n, 3, generator=g))
    rots = torch.randn(n, 4, generator=g)
    shs = torch.randn(n, 16, 3, generator=g) * 0.05
    shs[:, 0] = (torch.rand(n, 3, generator=g) - 0.5) / 0.28209479177387814
    return dict(means3D=means, scales=scales, rotations=rots / rots.norm(dim=1, keepdim=True), shs=shs,
                opacities=torch.rand(n, 1, generator=g) * 0.02 + 0.02)


def test_long_lists_in_a_later_scan_round():
    """The per-tile sorts are dispatched from counts the device derives from the tile histogram: here the only tiles
    beyond the 256- and the 2 048-entry sort sizes lie in the second round of the scan (69 x 65 = 4 485 tiles)."""
    from luciddreamer_b200 import rasterizer as R
    from oracle import oracle
    W, H = 1104, 1040
    case = cases.Case("late_lists_1104x1040", 20_000, W, H, 3, 44, bg=BG, golden=False)
    inp = cases.build_inputs(case)
    gx, gy = grid_of(W, H)
    # corners of tiles (51, 62) and (13, 62): tile indices 62 * 69 + 51 = 4 329 and 4 291, and their three neighbours
    parts = [cluster(inp["cam"], 2600, 816.0, 992.0, 45), cluster(inp["cam"], 500, 208.0, 992.0, 46)]
    for k in ("means3D", "scales", "rotations", "shs", "opacities"):
        inp[k] = torch.cat([inp[k]] + [p[k] for p in parts]).contiguous()
    f = oracle.rasterize_gaussians(*cases.binding_args(inp))
    og = dict(zip(cases.GRAD_NAMES, oracle.rasterize_gaussians_backward(f, inp["cot"].numpy())[:8]))
    rg = f.ranges.astype(np.int64)
    olens = rg[:, 1] - rg[:, 0]
    assert olens[:SCAN_ROUND].max() <= 256 and (olens[SCAN_ROUND:] > 2048).sum() >= 4
    assert ((olens[SCAN_ROUND:] > 256) & (olens[SCAN_ROUND:] <= 2048)).sum() >= 4
    d = f.geom("depths", 1)[case.P:, 0]
    assert len(np.unique(d)) < len(d) - 300                                 # ties survive the projection
    r = run("C", cases.binding_args(inp, dev()), inp["cot"])
    lens = util.assert_binning_matches_oracle(f, W, H, r["bufs"][1], r["bufs"][2], num_pairs=R._last_pairs[0])
    late = lens[SCAN_ROUND:]
    assert lens[:SCAN_ROUND].max() <= 256 and (late > 2048).any() and ((late > 256) & (late <= 2048)).any()
    check_forward(case, f, r)
    util.assert_grads_close(r["grads"], og, names=grad_names(case), what=case.name)


# ---- d. static capacity and graph replay in blocks -----------------------------------------------------------------------------

def test_block_geometry_step_under_static_capacity_and_graph_replay():
    """A 16x8-block step (forward + deterministic backward through the autograd node): the same bits with a static pair
    capacity and from a CUDA graph, also after the camera is rewritten in place."""
    from luciddreamer_b200 import rasterizer as R
    from luciddreamer_b200 import synthetic as syn
    from luciddreamer_b200.graphs import GraphedStep
    case, inp, d_cam, step, grads, out = _training_step_fixture("blk_shell_60k_721x531_bg")
    assert util.blend_rows_per_warp(case.W, case.H) == 8

    def assert_same(got, want, what):
        for k, (a, b) in enumerate(zip(got, want)):
            assert torch.equal(a, b), f"{what}: gradient {k} differs (max {float((a - b).abs().max()):.3e})"

    with R.deterministic():
        step(); torch.cuda.synchronize()
        ref_color, ref_grads, pairs = out["color"].clone(), grads(), R._last_pairs[0]
        with R.static_capacity(pairs + 1000):
            step()
        R.check_static()                                   # raises if the capacity was exceeded
        assert torch.equal(out["color"], ref_color)
        assert_same(grads(), ref_grads, "static capacity")
        g = GraphedStep(step, warmup=2)
        g.replay(); g.check()
        assert torch.equal(g.outputs, ref_color)
        assert_same(grads(), ref_grads, "graph replay")
        cam2 = syn.make_camera(case.W, case.H, c2w=syn.rotate360_poses(16)[1])
        d_cam.copy_(torch.cat([cam2.viewmatrix.reshape(-1), cam2.projmatrix.reshape(-1), cam2.campos.reshape(-1)]).to(d_cam.device))
        g.replay(); g.check()
        graphed_color, graphed_grads = g.outputs.clone(), grads()
        g.release()
        step(); torch.cuda.synchronize()
        assert torch.equal(graphed_color, out["color"]) and not torch.equal(graphed_color, ref_color)
        assert_same(graphed_grads, grads(), "graph replay with a new camera")
