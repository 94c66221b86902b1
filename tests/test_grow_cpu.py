"""Growth of the dreamed point cloud (pcd.grow_view, gspcd_grow_view) without a GPU: the host restatement reproduces
the reference's own dreaming-loop body, the reference's scale fit is a no-op, the CPU BLAS rounds 3x3 products as
the device does, and the new symbols' ABI."""
import ctypes as C
import hashlib
import os
import re
import subprocess
from fractions import Fraction

import numpy as np
import pytest
import torch

import grow_inputs
from luciddreamer_b200 import pcd

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "luciddreamer_b200", "pcd_csrc")


@pytest.fixture(scope="module", autouse=True)
def built():
    subprocess.check_call(["make", "-C", CSRC, "-j4"], stdout=subprocess.DEVNULL)


def digest(a):
    a = np.ascontiguousarray(a)
    return {"shape": list(a.shape), "dtype": str(a.dtype), "sha256": hashlib.sha256(a.tobytes()).hexdigest()}


def test_host_restatement_reproduces_the_reference_growth():
    names = []
    for c, inp, (pts, cols, border, new_depth) in grow_inputs.golden_cases():
        assert digest(inp["mask2"]) == c["mask2"] and digest(inp["valid_idx"]) == c["valid_idx"]
        assert digest(border) == c["border_valid_idx"]
        assert digest(new_depth) == c["new_depth"]
        assert digest(pts) == c["pts_coord_world"] and digest(cols) == c["pts_colors"]
        assert pts.dtype == np.float64 and cols.dtype == np.float32
        names.append(c["name"])
    cases = {c["name"]: c for c in grow_inputs.GOLDEN["cases"]}
    assert cases["zero_depth"]["n_linear_nan"] > 0                 # the nearest fallback is exercised
    assert cases["no_border"]["n_border"] == 0 and cases["no_border"]["n_inpainted"] > 0
    assert cases["no_inpainted"]["n_inpainted"] == 0 and cases["no_valid"]["n_valid"] == 0
    assert names == ["view1", "view2", "zero_depth", "no_border", "no_inpainted", "no_valid"]


def test_the_reference_scale_fit_leaves_the_identity():
    for c in grow_inputs.GOLDEN["cases"]:
        assert c["sc"] == 1.0 and c["sc_grad_is_none"]
        assert c["trans3d"] == np.eye(4).tolist() and c["trans3d_dtype"] == "float32"


def _r32(q):
    r = np.float32(float(q))
    cands = [np.nextafter(r, np.float32(-np.inf)), r, np.nextafter(r, np.float32(np.inf))]
    return min(cands, key=lambda c: (abs(Fraction(float(c)) - q), int(np.array(c).view(np.int32)) & 1))


def _chain(A, B, f32):
    """fma(a2, b2, fma(a1, b1, a0 * b0)) per entry, each step rounded once (exactly, through Fraction)."""
    rnd = _r32 if f32 else float
    F = lambda v: Fraction(float(v))
    out = np.empty((3, B.shape[1]), A.dtype)
    for r in range(3):
        for c in range(B.shape[1]):
            p = rnd(F(A[r, 0]) * F(B[0, c]))
            p = rnd(F(A[r, 1]) * F(B[1, c]) + F(p))
            out[r, c] = rnd(F(A[r, 2]) * F(B[2, c]) + F(p))
    return out


def test_cpu_blas_rounds_3x3_products_as_an_fma_chain():
    """numpy (float32 and float64) and torch (float32) round [3x3] @ [3xn] as fma(a2,b2, fma(a1,b1, a0*b0)) for
    every n >= 2 tried here; the device uses that chain for every n. For n = 1 numpy's float32 product takes another
    path ((a0b0 + a1b1) + a2b2), so a single border point or inpainted pixel may differ from it in the last bit."""
    rng = np.random.default_rng(0)
    zeros = 0
    for n in list(range(2, 17)) + [31, 64, 257]:
        A = rng.standard_normal((3, 3)).astype(np.float32)
        A[0, 1] = A[1, 0] = 0.0                                      # zero entries, as in inv(K)
        B = (rng.standard_normal((3, n)) * rng.uniform(0.5, 3, n)).astype(np.float32)
        B[:, 0] = [-0.0, 0.0, -0.0]
        c = _chain(A, B, True)
        assert (A @ B).tobytes() == c.tobytes(), n
        assert (torch.from_numpy(A) @ torch.from_numpy(B)).numpy().tobytes() == c.tobytes(), n
        A64, B64 = rng.standard_normal((3, 3)), rng.standard_normal((3, n))
        assert (A64 @ B64).tobytes() == _chain(A64, B64, False).tobytes(), n
        zeros += int((c == 0).sum())
    assert zeros > 0
    A = rng.standard_normal((3, 3)).astype(np.float32)
    one = [int(((A @ b) != _chain(A, b, True)).any()) for b in rng.standard_normal((200, 3, 1)).astype(np.float32)]
    print(f"n = 1: numpy float32 differs from the chain in {sum(one)} of 200 products")


def test_grow_symbols_argument_errors_and_scratch():
    L = pcd.lib()
    assert L.gspcd_abi_version() == 1
    b = C.c_uint64()
    sizes = []
    for nv in (0, 1, 1000, 100_000, 1_000_000):
        assert L.gspcd_grow_scratch_bytes(nv, 96, 128, C.byref(b)) == 0
        assert b.value % 256 == 0
        sizes.append(b.value)
    assert sizes == sorted(sizes) and sizes[-1] > sizes[0]
    prev = 0
    for H in (3, 4, 17, 96, 512):
        assert L.gspcd_grow_scratch_bytes(1000, H, H, C.byref(b)) == 0 and b.value >= prev
        prev = b.value
    for nv, H, W in ((-1, 96, 128), (10, 2, 128), (10, 96, 2)):
        assert L.gspcd_grow_scratch_bytes(nv, H, W, C.byref(b)) == -22
    assert L.gspcd_grow_scratch_bytes(10, 96, 128, None) == -22
    assert L.gspcd_grow_scratch_bytes(10, 96, 128, C.byref(b)) == 0
    need = b.value
    mats = np.zeros(48)
    A = 1 << 20                                            # fake, well-aligned device addresses: never dereferenced
    args = dict(pts=A, n=20, f32=0, vidx=A, coords=A, rnd=A, nv=10, mask=A, depth=A, image=A, H=96, W=128,
                mats=mats.ctypes.data, m=5, new_pts=A, new_cols=A, new_depth=A, border=A, nb=A, status=A, scratch=A,
                bytes=need)

    def call(**kw):
        a = dict(args, **kw)
        return L.gspcd_grow_view(a["pts"], a["n"], a["f32"], a["vidx"], a["coords"], a["rnd"], a["nv"], a["mask"],
                                 a["depth"], a["image"], a["H"], a["W"], a["mats"], a["m"], a["new_pts"],
                                 a["new_cols"], a["new_depth"], a["border"], a["nb"], a["status"], a["scratch"],
                                 a["bytes"], None)
    # every call below has exactly one invalid argument, so none of them reaches a device
    bad = [dict(pts=None), dict(pts=A + 4), dict(f32=2), dict(n=5), dict(nv=-1), dict(vidx=None), dict(vidx=A + 2),
           dict(coords=None), dict(coords=A + 4), dict(rnd=None), dict(rnd=A + 2), dict(mask=None), dict(mask=A + 2),
           dict(depth=None), dict(depth=A + 2), dict(image=None), dict(H=2), dict(W=2), dict(mats=None), dict(m=-1),
           dict(m=96 * 128 + 1), dict(new_pts=None), dict(new_pts=A + 4), dict(new_cols=None), dict(new_cols=A + 2),
           dict(new_depth=A + 4), dict(border=A + 2), dict(nb=None), dict(nb=A + 2), dict(status=None),
           dict(status=A + 2), dict(scratch=None), dict(scratch=A + 128), dict(bytes=need - 1)]
    for kw in bad:
        assert call(**kw) == -22, kw
    assert call(f32=1, pts=A + 4, bytes=need - 1) == -22                 # float32 cloud: 4-byte alignment suffices


def test_grow_kernels_have_no_spills_and_no_float_atomics():
    log = open(os.path.join(CSRC, "gs_pcd.o.ptxas.log")).read()
    spills = re.findall(r"(\d+) bytes spill stores, (\d+) bytes spill loads", log)
    assert spills and all(s == ("0", "0") for s in spills)
    sass = subprocess.run(["cuobjdump", "-sass", os.path.join(CSRC, "gs_pcd.o")], capture_output=True, text=True,
                          check=True).stdout
    for k in ("k_grow", "k_border_values", "k_border_flags", "k_corners", "k_inpaint_flags"):
        assert k in sass
    assert not re.search(r"\b(RED|ATOM|ATOMS)\.[A-Z0-9.]*F(16|32|64)", sass)


def test_grow_view_checks_its_inputs():
    H, W = 8, 8
    K = np.eye(3, dtype=np.float32)
    z = dict(pts=np.zeros((3, 0)), colors=np.zeros((0, 3), np.float32), R=np.eye(3), T=np.zeros((3, 1)), K=K,
             mask2=np.zeros((H, W), np.int64), valid_idx=np.zeros(0, np.int64), pixel_coord=np.zeros((2, 0)),
             round_coord=np.zeros((2, 0), np.int32), image=np.zeros((H, W, 3), np.uint8),
             depth=np.ones((H, W), np.float32))
    bad = [dict(K=K.astype(np.float64)), dict(depth=np.ones((H, W))), dict(image=np.zeros((H, W, 3), np.float32)),
           dict(depth=torch.ones(H, W)), dict(pts=torch.zeros(3, 0, dtype=torch.float64)),
           dict(image=np.zeros((H, W + 1, 3), np.uint8)), dict(pixel_coord=np.zeros((2, 1)))]
    for kw in bad:
        with pytest.raises((TypeError, ValueError, RuntimeError)):
            pcd.grow_view(**dict(z, **kw))
