"""Seeded parity cases shared by the golden-vector generator (tests/golden/make_golden.py, run once on the GPU
box against the reference CUDA rasterizer) and by the CPU / GPU parity tests.  Inputs are regenerated from the
seed on every machine (torch CPU generators are bit-reproducible), so the fixtures hold outputs only."""
from __future__ import annotations

import math
from typing import Dict, NamedTuple, Optional

import numpy as np
import torch

from luciddreamer_b200 import synthetic as syn


class Case(NamedTuple):
    name: str
    P: int
    W: int
    H: int
    D: int                      # active SH degree
    seed: int
    scale_mult: float = 1.0
    bg: tuple = (0.0, 0.0, 0.0)
    scale_modifier: float = 1.0
    precomp: bool = False       # feed colors_precomp + cov3D_precomp instead of shs + scales/rotations
    pose: Optional[str] = None  # None = identity; "rot:<deg>" = yaw about the vertical axis; "llff:<frame>"
    golden: bool = True         # has a fixture under tests/golden/
    opacity_shift: float = 0.0  # added to the opacity logits (same random draws)
    aniso_sigma: float = 0.3    # log-normal spread of the per-axis scale factors (same random draws)
    scene: str = "shell"        # "shell" (SURVEY 8d) or "frustum" (LucidDreamer-shaped, synthetic.make_frustum_scene)


CASES = [
    Case("micro_1k_64", 1000, 64, 64, 3, 11, scale_mult=2.0),
    Case("cfg1_10k_256_d0", 10_000, 256, 256, 0, 1001),
    Case("odd_3k_100x70_bg", 3000, 100, 70, 2, 12, scale_mult=2.0, bg=(0.3, 0.6, 0.9)),
    Case("stress_4k_96_x6", 4000, 96, 96, 3, 13, scale_mult=6.0),
    Case("precomp_2k_80", 2000, 80, 80, 0, 14, scale_mult=2.0, precomp=True, bg=(0.1, 0.0, 0.2)),
    Case("modifier_2k_80", 2000, 80, 80, 1, 15, scale_mult=2.0, scale_modifier=1.7),
    Case("rot40_5k_128x72", 5000, 128, 72, 3, 16, scale_mult=2.0, pose="rot:40"),
    Case("llff_5k_128x72", 5000, 128, 72, 3, 17, scale_mult=2.0, pose="llff:37"),
    Case("cfg2_100k_512", 100_000, 512, 512, 3, 1002),
]
# oracle-only cases (no reference fixture): the branches the shell scenes hardly reach
EXTRA_CASES = [
    # opacities pushed towards 1 (a third above the 0.99 clamp of forward.cu:343), thick stacks of large splats: early
    # termination at T < 1e-4 (forward.cu:348-352) on most pixels, generic (non fast-path) evaluation of the clamped ones
    Case("opaque_40k_64_x8", 40_000, 64, 64, 3, 21, scale_mult=8.0, opacity_shift=4.0, golden=False),
    # needle-shaped splats: ill-conditioned 2-D conics -> generic path via the conditioning test, huge tile rectangles
    Case("needles_2k_96", 2000, 96, 96, 2, 22, scale_mult=3.0, aniso_sigma=2.5, golden=False),
    # LucidDreamer-shaped: everything inside the frustum, ~1.5 px sigma, long tile lists, termination
    Case("frustum_20k_96", 20_000, 96, 96, 3, 23, golden=False, scene="frustum"),
    Case("frustum_60k_64_bg", 60_000, 64, 64, 1, 24, bg=(0.2, 0.5, 0.1), opacity_shift=1.0, golden=False, scene="frustum"),
]
# oracle-only cases in the 16x8-block geometry of the tile passes (csrc/gs_blend.cuh: chosen from the tile count and the
# SM count; 1 500 tiles and more are blocks on every H100 variant, and the GPU tests ask the library which one ran).
# Between them they reach, in blocks, what EXTRA_CASES reach in strips; both image sides are ragged (not multiples of
# 16, and H % 8 != 0: the bottom warp of the last tile row holds live and dead rows).
BLOCK_CASES = [
    # the plain path: W % 16 = 1, H % 16 = 3
    Case("blk_shell_60k_721x531_bg", 60_000, 721, 531, 3, 31, scale_mult=2.0, bg=(0.3, 0.6, 0.9), golden=False),
    # a third of the opacities above the 0.99 clamp, thick stacks: termination on most pixels, whole threads on the
    # generic path, warps and tiles that leave their lists early
    Case("blk_opaque_150k_650x615_x6", 150_000, 650, 615, 3, 32, scale_mult=6.0, opacity_shift=4.0, golden=False),
    # needles: ill-conditioned conics, tile rectangles of hundreds of tiles (hit decisions recomputed per tile)
    Case("blk_needles_3k_599x685", 3000, 599, 685, 2, 33, scale_mult=3.0, aniso_sigma=2.5, golden=False),
    # LucidDreamer-shaped and dense (every Gaussian visible); splats of ~12 px sigma, so that 80 000 Gaussians give
    # per-tile lists on both sides of the 2 048-entry sort size (the same density at 1.5 px sigma would take millions)
    Case("blk_frustum_80k_633x613_x8", 80_000, 633, 613, 3, 36, scale_mult=8.0, opacity_shift=1.0, golden=False,
         scene="frustum"),
    Case("blk_precomp_40k_811x470_bg", 40_000, 811, 470, 0, 35, scale_mult=2.0, bg=(0.1, 0.0, 0.2), scale_modifier=1.7,
         precomp=True, golden=False),
]
CASES_ALL = CASES + EXTRA_CASES + BLOCK_CASES
BY_NAME = {c.name: c for c in CASES_ALL}


def cov3D_of(scales: torch.Tensor, rotations: torch.Tensor) -> torch.Tensor:
    """[P, 6] upper triangle of R diag(s^2) R^T, computed in float64 and rounded to float32."""
    q = rotations.double(); s = scales.double()
    r, x, y, z = q[:, 0], q[:, 1], q[:, 2], q[:, 3]
    R = torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y - r * z), 2 * (x * z + r * y),
                     2 * (x * y + r * z), 1 - 2 * (x * x + z * z), 2 * (y * z - r * x),
                     2 * (x * z - r * y), 2 * (y * z + r * x), 1 - 2 * (x * x + y * y)], -1).reshape(-1, 3, 3)
    Sg = R @ torch.diag_embed(s * s) @ R.transpose(1, 2)
    return torch.stack([Sg[:, 0, 0], Sg[:, 0, 1], Sg[:, 0, 2], Sg[:, 1, 1], Sg[:, 1, 2], Sg[:, 2, 2]],
                       -1).float().contiguous()


def build_inputs(case: Case) -> Dict[str, object]:
    """CPU float32 tensors + camera in the reference binding's vocabulary."""
    if case.scene == "frustum":
        sc = syn.make_frustum_scene(case.P, case.seed, case.W, case.H, sigma_px=1.5 * case.scale_mult)
        if case.opacity_shift:
            sc["opacities"] = torch.sigmoid(torch.logit(sc["opacities"]) + case.opacity_shift).contiguous()
    else:
        sc = syn.make_scene(case.P, case.seed, scale_mult=case.scale_mult, opacity_shift=case.opacity_shift,
                            aniso_sigma=case.aniso_sigma)
    c2w = None
    swap = False
    if case.pose:
        kind, arg = case.pose.split(":")
        if kind == "rot":
            th = math.radians(float(arg))
            c, s = math.cos(th), math.sin(th)
            c2w = np.array([[c, 0, s, 0], [0, 1, 0, 0], [-s, 0, c, 0], [0, 0, 0, 1.0]])
        elif kind == "llff":
            c2w = syn.llff_poses(400)[int(arg)]
            swap = True          # exercise the load_json fov-swap quirk (utils/camera.py:48)
    cam = syn.make_camera(case.W, case.H, c2w=c2w, swap_fov_like_load_json=swap)
    out = dict(case=case, cam=cam, bg=torch.tensor(case.bg, dtype=torch.float32), means3D=sc["means3D"],
               opacities=sc["opacities"], cot=syn.make_cotangent(case.H, case.W, case.seed))
    if case.precomp:
        # colours and covariances computed here in plain torch (float64 -> float32): any valid input will do
        g = torch.Generator().manual_seed(case.seed + 99)
        out["colors_precomp"] = torch.rand(case.P, 3, generator=g).contiguous()
        out["cov3D_precomp"] = cov3D_of(sc["scales"], sc["rotations"])
        out["shs"] = None; out["scales"] = None; out["rotations"] = None
    else:
        out["shs"] = sc["shs"]; out["scales"] = sc["scales"]; out["rotations"] = sc["rotations"]
        out["colors_precomp"] = None; out["cov3D_precomp"] = None
    return out


def binding_args(inp, device=None):
    """Positional args of `_C.rasterize_gaussians` (rasterize_points.h:18-38) for a case's inputs."""
    case, cam = inp["case"], inp["cam"]

    def mv(t):
        if t is None:
            return torch.empty(0) if device is None else torch.empty(0, device=device)
        return t if device is None else t.to(device)

    return (mv(inp["bg"]), mv(inp["means3D"]), mv(inp["colors_precomp"]), mv(inp["opacities"]), mv(inp["scales"]),
            mv(inp["rotations"]), case.scale_modifier, mv(inp["cov3D_precomp"]), mv(cam.viewmatrix),
            mv(cam.projmatrix), cam.tanfovx, cam.tanfovy, cam.image_height, cam.image_width, mv(inp["shs"]), case.D,
            mv(cam.campos), False, False)


GRAD_NAMES = ("dL_dmeans2D", "dL_dcolors", "dL_dopacity", "dL_dmeans3D", "dL_dcov3D", "dL_dsh", "dL_dscales",
              "dL_drotations")


def sparse_rows(a: np.ndarray):
    """Row-sparse encoding of a [P, ...] gradient tensor (most rows are exactly zero: invisible Gaussians)."""
    a2 = a.reshape(a.shape[0], -1)
    idx = np.nonzero(np.any(a2 != 0, axis=1))[0].astype(np.int32)
    return idx, a2[idx].astype(np.float32)


def dense_rows(idx, rows, shape):
    out = np.zeros((shape[0], int(np.prod(shape[1:])) if len(shape) > 1 else 1), np.float32)
    out[idx] = rows
    return out.reshape(shape)
