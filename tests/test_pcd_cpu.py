"""Point-cloud warp (include/gspcd.h), without a GPU: the host restatement reproduces the reference's own loops,
the host build of the exact predicates and locate step agrees with scipy's Delaunay, and the library's ABI."""
import ctypes as C
import hashlib
import json
import os
import re
import subprocess

import numpy as np
import pytest
from scipy.spatial import Delaunay

import pcd_cases
import pcd_host
from luciddreamer_b200 import pcd

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "luciddreamer_b200", "pcd_csrc")
GOLDEN = json.load(open(os.path.join(ROOT, "tests", "golden", "pcd_golden.json")))


@pytest.fixture(scope="module", autouse=True)
def built():
    subprocess.check_call(["make", "-C", CSRC, "-j4"], stdout=subprocess.DEVNULL)


def digest(a):
    a = np.ascontiguousarray(a)
    return {"shape": list(a.shape), "dtype": str(a.dtype), "sha256": hashlib.sha256(a.tobytes()).hexdigest()}


def golden_inputs():
    g = GOLDEN
    pts, cols = pcd_cases.depth_cloud(g["cloud"]["seed"], g["H"], g["W"], extra=g["cloud"]["extra"])
    return pts, cols, np.array(g["K"]), g["H"], g["W"]


def test_host_restatement_reproduces_the_reference_aligning_loop():
    pts, cols, K, H, W = golden_inputs()
    frames, mats = pcd_host.align_frames_host(pts, cols, np.array(GOLDEN["render_poses"]),
                                              np.array(GOLDEN["internal_poses"]), K, H, W)
    assert len(frames) == len(GOLDEN["align_frames"]) < 5 * len(GOLDEN["render_poses"])   # some views skipped
    for f, m, g in zip(frames, mats, GOLDEN["align_frames"]):
        assert digest(f) == g["image"]
        assert m.tolist() == g["transform_matrix"]


def test_host_restatement_reproduces_the_reference_dreaming_warp():
    pts, cols, K, H, W = golden_inputs()
    P = np.array(GOLDEN["dream_poses"])
    for g in GOLDEN["dream"]:
        img, mask, valid, coords, rnd = pcd_host.warp_view_host(pts, cols, P[g["pose"], :3, :3], P[g["pose"], :3, 3:4],
                                                                K, H, W)
        assert digest(img) == g["image2"] and digest(mask) == g["mask2"]
        assert digest(valid) == g["valid_idx"] and digest(coords) == g["coords"] and digest(rnd) == g["round"]


def host_lib():
    L = C.CDLL(os.path.join(CSRC, "libgspcd_host.so"))
    L.gspcd_host_locate.argtypes = [C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_double, C.c_int32, C.c_int32,
                                    C.c_void_p]
    return L


def host_locate(xy, q, W, H, cell):
    xy, q = np.ascontiguousarray(xy, np.float64), np.ascontiguousarray(q, np.float64)
    tri = np.empty((len(q), 3), np.int32)
    st = host_lib().gspcd_host_locate(xy.ctypes.data, len(xy), q.ctypes.data, len(q), cell, W, H, tri.ctypes.data)
    return st, tri


@pytest.mark.parametrize("seed,n,W,H", [(0, 40, 128, 96), (1, 10_000, 128, 96), (2, 100_000, 256, 192),
                                        (3, 1_000_000, 512, 512)])
def test_locate_finds_scipys_triangle_and_hull_membership(seed, n, W, H):
    rng = np.random.default_rng(seed)
    xy = np.stack([rng.uniform(0, W - 1, n), rng.uniform(0, H - 1, n)], 1)
    gx, gy = np.meshgrid(np.arange(W, dtype=np.float64), np.arange(H, dtype=np.float64))
    q = np.stack([gx.ravel(), gy.ravel()], 1)
    if n > 50_000:                                         # keep the CPU time down: a seeded subset of pixels
        q = q[rng.choice(len(q), 20_000, replace=False)]
        q = np.concatenate([q, [[0, 0], [W - 1, H - 1], [W // 2, 0], [0, H // 2]]])   # corners: outside the hull
    st, tri = host_locate(xy, q, W, H, np.sqrt(W * H * 2.0 / n))
    assert st == 0
    d = Delaunay(xy)
    s = d.find_simplex(q)
    ref = np.where(s[:, None] >= 0, np.sort(d.simplices[s], 1), -1)
    np.testing.assert_array_equal(np.sort(tri, 1), ref)
    assert (s < 0).any() and (s >= 0).any()


def test_locate_on_exact_lattice_duplicates_and_collinear_points():
    W, H = 16, 12
    gx, gy = np.meshgrid(np.arange(W, dtype=np.float64), np.arange(H, dtype=np.float64))
    lattice = np.stack([gx.ravel(), gy.ravel()], 1)
    q = lattice + 0.25
    # cocircular everywhere: any triangle of the lattice that contains q is a Delaunay triangle; it must contain q
    for pts in (lattice, np.concatenate([lattice, lattice])):
        st, tri = host_locate(pts, q, W, H, 1.0)
        assert st == 0
        inside = (q[:, 0] <= W - 1) & (q[:, 1] <= H - 1)
        assert (tri[inside] >= 0).all() and (tri[~inside] < 0).all()
        assert (tri[inside] < len(lattice)).all()          # of duplicates only the lowest index is a vertex
        for t, p in zip(tri[inside], q[inside]):
            a, b, c = pts[t]
            area = lambda u, v, w: (v[0] - u[0]) * (w[1] - u[1]) - (v[1] - u[1]) * (w[0] - u[0])
            s0, s1, s2 = area(a, b, p), area(b, c, p), area(c, a, p)
            assert min(s0, s1, s2) >= 0 or max(s0, s1, s2) <= 0
    line = np.stack([np.arange(10.0), np.arange(10.0) * 0.5], 1)
    st, tri = host_locate(line, np.array([[2.0, 1.0], [3.0, 3.0]]), W, H, 1.0)
    assert st == 0 and (tri < 0).all()                     # only collinear points: nothing to interpolate
    st, tri = host_locate(line[:2], np.array([[0.5, 0.25]]), W, H, 1.0)
    assert (tri < 0).all()


def test_exact_predicates_decide_near_degenerate_cases():
    L = host_lib()
    L.gspcd_host_orient.argtypes = [C.c_void_p] * 3
    L.gspcd_host_incircle.argtypes = [C.c_void_p] * 4
    arr = lambda *v: np.array(v, np.float64)
    keep = []

    def o(a, b, c):
        keep.extend([a, b, c])
        return L.gspcd_host_orient(a.ctypes.data, b.ctypes.data, c.ctypes.data)

    def ic(a, b, c, d):
        keep.extend([a, b, c, d])
        return L.gspcd_host_incircle(a.ctypes.data, b.ctypes.data, c.ctypes.data, d.ctypes.data)

    e = np.nextafter(0.5, 1.0)
    assert o(arr(0.5, 0.5), arr(12.0, 12.0), arr(24.0, 24.0)) == 0
    assert o(arr(e, 0.5), arr(12.0, 12.0), arr(24.0, 24.0)) == -1
    assert o(arr(0.5, e), arr(12.0, 12.0), arr(24.0, 24.0)) == 1
    a, b, c = arr(0.0, 0.0), arr(4.0, 0.0), arr(0.0, 4.0)
    assert ic(a, b, c, arr(4.0, 4.0)) == 0
    assert ic(a, b, c, arr(np.nextafter(4.0, 0.0), 4.0)) == 1
    assert ic(a, b, c, arr(np.nextafter(4.0, 9.0), 4.0)) == -1
    assert ic(arr(0.1, 0.3), arr(300.7, 0.3), arr(0.1, 200.9), arr(300.7, 200.9)) == 0
    # one ulp off cocircular, where the float64 determinant is all rounding: the sign must be the rational one
    rng = np.random.default_rng(9)
    for _ in range(200):
        a, b, c, d = (arr(*v) for v in rng.uniform(0, 511, (4, 2)))
        d = arr(np.nextafter(a[0], np.inf), a[1]) if rng.random() < 0.5 else d
        assert ic(a, b, c, d) == exact_incircle(a, b, c, d)
    for x in (np.nextafter(0.1, 1.0), np.nextafter(0.1, 0.0)):
        pts = [arr(x, 0.3), arr(300.7, 0.3), arr(0.1, 200.9), arr(300.7, 200.9)]
        s = exact_incircle(*pts)
        assert s != 0 and ic(*pts) == s


def exact_incircle(a, b, c, d):
    from fractions import Fraction as F
    m = [[F(p[0]) - F(d[0]), F(p[1]) - F(d[1])] for p in (a, b, c)]
    rows = [[u, v, u * u + v * v] for u, v in m]
    det = (rows[0][0] * (rows[1][1] * rows[2][2] - rows[2][1] * rows[1][2])
           - rows[0][1] * (rows[1][0] * rows[2][2] - rows[2][0] * rows[1][2])
           + rows[0][2] * (rows[1][0] * rows[2][1] - rows[2][0] * rows[1][1]))
    return (det > 0) - (det < 0)


def test_library_exports_and_argument_errors():
    L = pcd.lib()
    assert L.gspcd_abi_version() == 1
    b = C.c_uint64()
    assert L.gspcd_scratch_bytes(1000, 96, 128, C.byref(b)) == 0
    small = b.value
    assert small >= 1000 * 40 + 96 * 128 * 50 and small % 256 == 0
    assert L.gspcd_scratch_bytes(2000, 96, 128, C.byref(b)) == 0 and b.value > small
    assert L.gspcd_scratch_bytes(0, 96, 128, C.byref(b)) == 0
    for n, H, W in ((-1, 96, 128), (10, 2, 128), (10, 96, 2)):
        assert L.gspcd_scratch_bytes(n, H, W, C.byref(b)) == -22
    assert L.gspcd_scratch_bytes(10, 96, 128, None) == -22
    assert L.gspcd_scratch_bytes(10, 96, 128, C.byref(b)) == 0
    need = b.value
    # every call below has exactly one invalid argument, so none of them reaches a device
    K = np.eye(3)
    pose = np.zeros(12)
    A = 1 << 20                                            # fake, well-aligned device addresses: never dereferenced
    args = dict(pts=A, colors=A, n=10, pose=pose.ctypes.data, K=K.ctypes.data, H=96, W=128, image=A, mask=A,
                vidx=A, coords=A, rnd=A, count=A, status=A, scratch=A, bytes=need)

    def call(**kw):
        a = dict(args, **kw)
        return L.gspcd_warp_view(a["pts"], a["colors"], a["n"], a["pose"], a["K"], a["H"], a["W"], a["image"],
                                 a["mask"], a["vidx"], a["coords"], a["rnd"], a["count"], a["status"], a["scratch"],
                                 a["bytes"], None)
    assert call(pts=None) == -22
    assert call(pts=A + 4) == -22                          # misaligned float64
    assert call(scratch=A + 128) == -22                    # scratch must be 256-byte aligned
    assert call(bytes=need - 1) == -22                    # short scratch
    assert call(H=2) == -22 and call(W=2) == -22
    assert call(status=None) == -22 and call(K=None) == -22
    assert L.gspcd_align(A, A, 10, pose.ctypes.data, K.ctypes.data, 1, 96, 128, None, A, A, A, need, None) == -22
    assert L.gspcd_align(A, A, 10, pose.ctypes.data, K.ctypes.data, 1, 96, 128, A, A, A, A, need - 1, None) == -22
    assert L.gspcd_align(A, A, 10, None, K.ctypes.data, 1, 96, 128, A, A, A, A, need, None) == -22


def test_no_spills_and_no_float_atomics():
    log = open(os.path.join(CSRC, "gs_pcd.o.ptxas.log")).read()
    spills = re.findall(r"(\d+) bytes spill stores, (\d+) bytes spill loads", log)
    assert spills and all(s == ("0", "0") for s in spills)
    sass = subprocess.run(["cuobjdump", "-sass", os.path.join(CSRC, "gs_pcd.o")], capture_output=True, text=True,
                          check=True).stdout
    assert "k_interp" in sass
    assert not re.search(r"\b(RED|ATOM|ATOMS)\.[A-Z0-9.]*F(16|32|64)", sass)


def test_module_refuses_cpu_tensors():
    import torch
    with pytest.raises((TypeError, RuntimeError)):
        pcd.warp_view(torch.zeros(3, 4, dtype=torch.float64), np.zeros((4, 3), np.float32), np.eye(3),
                      np.zeros((3, 1)), np.eye(3), 8, 8)
