"""The conservative screen test that k_project runs ahead of the exact per-Gaussian path (csrc/gs_preprocess.cu:
surely_offscreen) may only reject Gaussians whose exact path ends with an empty tile rect.  The device code needs a GPU;
its ARITHMETIC is restated here in numpy float32, operation for operation, and checked against the radii of the reference
fixtures and of the CPU oracle on every parity case plus adversarial inputs (un-normalised quaternions, huge and tiny
scales, scale modifiers, precomputed covariances, rotated / off-centre cameras): no Gaussian with radius > 0 may be
rejected.  The GPU parity tests then check the kernel itself (radii and pair counts are compared exactly there)."""
import numpy as np
import pytest
import torch

import cases
import util
from oracle import oracle

f32 = np.float32
NEAR = f32(0.2)


def view_norm2_np(vm):
    """Upper bound of ||V3||_2^2: (tr G^8)^(1/8) with G = V3^T V3 (1.147 for a rigid view matrix), tr G when G^8 leaves the
    float range."""
    V = np.array([[vm[4 * j + i] for j in range(3)] for i in range(3)], dtype=f32)     # V[i][j] = vm[i + 4 j]
    G = (V.T @ V).astype(f32)
    G2 = (G @ G).astype(f32)
    G4 = (G2 @ G2).astype(f32)
    t8 = f32((G4 * G4).sum())
    trG = f32(G[0, 0] + G[1, 1] + G[2, 2])
    if t8 > f32(1e-30) and t8 < f32(1e30):
        return min(trG, f32(np.sqrt(np.sqrt(np.sqrt(t8)))) * f32(1.001))
    return trG


def surely_offscreen_np(means, scales, rots, cov6, vm, pm, tanx, tany, W, H, mod):
    """-> (candidate_by_z, rejected) per Gaussian; float32 throughout like the kernel."""
    means = means.astype(f32)
    vm = vm.astype(f32).reshape(-1); pm = pm.astype(f32).reshape(-1)          # flat, element [k] as the kernel indexes it
    x, y, z = means[:, 0], means[:, 1], means[:, 2]
    tx = vm[0] * x + vm[4] * y + vm[8] * z + vm[12]
    ty = vm[1] * x + vm[5] * y + vm[9] * z + vm[13]
    tz = vm[2] * x + vm[6] * y + vm[10] * z + vm[14]
    zerr = f32(2e-6) * (np.abs(vm[2] * x) + np.abs(vm[6] * y) + np.abs(vm[10] * z) + np.abs(vm[14]))
    by_z = ~(tz <= NEAR - zerr)
    with np.errstate(all="ignore"):
        hx = pm[0] * x + pm[4] * y + pm[8] * z + pm[12]
        hy = pm[1] * x + pm[5] * y + pm[9] * z + pm[13]
        hw = pm[3] * x + pm[7] * y + pm[11] * z + pm[15]
        iw = f32(1.0) / (hw + f32(0.0000001))
        px = ((hx * iw + f32(1.0)) * f32(W) - f32(1.0)) * f32(0.5)
        py = ((hy * iw + f32(1.0)) * f32(H) - f32(1.0)) * f32(0.5)
        iz = f32(1.0) / tz
        limx, limy = f32(1.3) * f32(tanx), f32(1.3) * f32(tany)
        cx = np.minimum(limx, np.maximum(-limx, tx * iz)); cy = np.minimum(limy, np.maximum(-limy, ty * iz))
        fx, fy = f32(W / (2.0 * tanx)), f32(H / (2.0 * tany))
        J00 = fx * iz; J11 = fy * iz
        nJ = J00 * J00 * (f32(1.0) + cx * cx) + J11 * J11 * (f32(1.0) + cy * cy)
        vnorm2 = view_norm2_np(vm)
        if cov6 is not None:
            c = cov6.astype(f32)
            nS = np.sqrt(c[:, 0] ** 2 + c[:, 3] ** 2 + c[:, 5] ** 2 + f32(2) * (c[:, 1] ** 2 + c[:, 2] ** 2 + c[:, 4] ** 2))
        else:
            q = rots.astype(f32)
            n = q[:, 0] * q[:, 0] + q[:, 1] * q[:, 1] + q[:, 2] * q[:, 2] + q[:, 3] * q[:, 3]
            d = np.abs(f32(1.0) - n) + n
            sc = np.abs(scales.astype(f32))
            sm = f32(mod) * np.maximum(sc[:, 0], np.maximum(sc[:, 1], sc[:, 2])) * d
            nS = sm * sm
        nA = nJ * vnorm2
        L = f32(1.52) * nA * nS + f32(1.0)
        ok = L < f32(1e30)
        Rb = f32(3.0) * np.sqrt(L) + f32(2.0)
        sx = Rb + f32(1e-5) * np.abs(px); sy = Rb + f32(1e-5) * np.abs(py)
        gx, gy = (W + 15) // 16, (H + 15) // 16
        off = (px + sx + f32(15) < 0) | (px - sx >= f32(16 * gx)) | (py + sy + f32(15) < 0) | (py - sy >= f32(16 * gy))
    rejected = by_z & (tz > f32(0.5) * NEAR) & ok & off
    return by_z, rejected


def _check(inp, radii, what):
    case, cam = inp["case"], inp["cam"]
    npy = lambda t: None if t is None else t.numpy()
    by_z, rej = surely_offscreen_np(npy(inp["means3D"]), npy(inp["scales"]), npy(inp["rotations"]), npy(inp["cov3D_precomp"]),
                                    cam.viewmatrix.numpy(), cam.projmatrix.numpy(), cam.tanfovx, cam.tanfovy,
                                    cam.image_width, cam.image_height, case.scale_modifier)
    vis = np.asarray(radii) > 0
    assert not (vis & ~by_z).any(), f"{what}: near-plane pre-test dropped {int((vis & ~by_z).sum())} visible Gaussians"
    assert not (vis & rej).any(), f"{what}: screen pre-test rejected {int((vis & rej).sum())} visible Gaussians"
    inv = by_z & ~vis
    return int(rej.sum()), int(inv.sum())


@pytest.mark.parametrize("case", cases.CASES, ids=lambda c: c.name)
def test_precull_never_rejects_what_the_reference_keeps(case):
    inp = cases.build_inputs(case)
    rej, inv = _check(inp, util.load_golden(case.name)["radii"], case.name)
    print(f"{case.name}: off-screen {inv}, rejected early {rej}")
    if inv > 100 and case.scene == "shell" and not case.pose and case.scale_mult <= 2.0:
        assert rej > 0.7 * inv, f"{case.name}: only {rej} of {inv} off-screen Gaussians rejected -- the bound is too loose to pay"


@pytest.mark.parametrize("case", cases.EXTRA_CASES + cases.BLOCK_CASES, ids=lambda c: c.name)
def test_precull_never_rejects_what_the_oracle_keeps(case):
    inp = cases.build_inputs(case)
    f = oracle.rasterize_gaussians(*cases.binding_args(inp))
    _check(inp, f.radii, case.name)


@pytest.mark.parametrize("seed", range(6))
def test_precull_on_adversarial_inputs(seed):
    """Un-normalised quaternions (|q| from 1e-3 to 30), scales over 8 decades, means on and around the frustum border,
    a scale modifier, odd image sizes: the oracle's radii decide."""
    g = torch.Generator().manual_seed(900 + seed)
    P = 6000
    W, H = [(100, 70), (64, 64), (333, 17), (16, 16), (1920, 1080), (31, 250)][seed]
    case = cases.Case(f"adv{seed}", P, W, H, 0, 900 + seed, scale_modifier=[1.0, 0.01, 7.5, 1.0, 2.0, 1.0][seed], golden=False)
    inp = cases.build_inputs(case)
    cam = inp["cam"]
    # means: a fan that straddles the image border at every depth, some behind / on the near plane
    z = torch.exp(torch.empty(P).uniform_(-2.5, 4.0, generator=g))
    z[: P // 20] = 0.2 + torch.empty(P // 20).uniform_(-1e-6, 1e-6, generator=g)
    u = torch.empty(P).uniform_(-1.6, 1.6, generator=g) * cam.tanfovx
    v = torch.empty(P).uniform_(-1.6, 1.6, generator=g) * cam.tanfovy
    inp["means3D"] = torch.stack([u * z, v * z, z], 1).contiguous()
    inp["scales"] = (torch.exp(torch.empty(P, 3).uniform_(-12.0, 6.0, generator=g)) * z[:, None] * 0.01).contiguous()
    q = torch.randn(P, 4, generator=g)
    inp["rotations"] = (q * torch.exp(torch.empty(P, 1).uniform_(-7.0, 3.4, generator=g))).contiguous()
    f = oracle.rasterize_gaussians(*cases.binding_args(inp))
    rej, inv = _check(inp, f.radii, case.name)
    print(f"{case.name}: visible {int((np.asarray(f.radii) > 0).sum())}, off-screen {inv}, rejected early {rej}")
    assert int((np.asarray(f.radii) > 0).sum()) > 100 and (rej > 100 or W * H <= 256)      # the case exercises both outcomes


def test_view_norm_bound_holds_over_the_float_range():
    rng = np.random.default_rng(5)
    for k in range(200):
        V = rng.standard_normal((3, 3)) * 10.0 ** rng.uniform(-7, 5)
        if k % 4 == 0:                                                       # rigid rotations, scaled
            V = np.linalg.qr(rng.standard_normal((3, 3)))[0] * 10.0 ** rng.uniform(-7, 5)
        vm = np.zeros(16, f32)
        for i in range(3):
            for j in range(3):
                vm[i + 4 * j] = V[i, j]
        true = np.linalg.svd(vm.reshape(4, 4)[:3, :3].astype(np.float64), compute_uv=False)[0] ** 2
        got = float(view_norm2_np(vm))
        assert got >= true * (1 - 1e-5) or not np.isfinite(got), (k, got, true)
        if 1e-2 < true < 1e3:
            assert got <= 3.01 * true                                        # never looser than the Frobenius norm


@pytest.mark.parametrize("unit", [1e3, 1e-3, 3e4])
def test_precull_with_a_scaled_world(unit):
    """The same scene in other length units: world coordinates and scales multiplied by `unit`, the 3x3 block of the view
    matrix divided by it (view space, and so the image, unchanged).  At 1e3 and beyond G^8 underflows in float32."""
    case = cases.BY_NAME["rot40_5k_128x72"]
    inp = cases.build_inputs(case)
    cam = inp["cam"]
    vm = cam.viewmatrix.double().clone()
    proj_t = torch.linalg.solve(vm, cam.projmatrix.double())                 # projmatrix = viewmatrix @ Proj^T
    vm[:3, :3] /= unit
    inp["cam"] = cam._replace(viewmatrix=vm.float().contiguous(), projmatrix=(vm @ proj_t).float().contiguous(),
                              campos=(cam.campos.double() * unit).float().contiguous())
    inp["means3D"] = (inp["means3D"].double() * unit).float().contiguous()
    inp["scales"] = (inp["scales"].double() * unit).float().contiguous()
    f = oracle.rasterize_gaussians(*cases.binding_args(inp))
    base = util.load_golden(case.name)["radii"]
    assert (np.asarray(f.radii) > 0).sum() > 0.9 * (base > 0).sum()          # it IS the same picture
    rej, inv = _check(inp, f.radii, f"{case.name} x{unit}")
    assert rej > 0.5 * inv
