"""Training-scene images (luciddreamer_b200.scene, include/gsscene.h) without a GPU: the host restatement of the
compositing and of OpenCV's Canny equals the golden data byte for byte, the rules it relies on hold, and the new
library's ABI, argument checks and machine code."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest
import torch

import canny_host
from luciddreamer_b200 import scene

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "luciddreamer_b200", "scene_csrc")
GOLDEN = np.load(os.path.join(ROOT, "tests", "golden", "canny_golden.npz"))
NAMES = sorted({k.split("/")[0] for k in GOLDEN.files})


@pytest.fixture(scope="module", autouse=True)
def built():
    subprocess.check_call(["make", "-C", CSRC, "-j4"], stdout=subprocess.DEVNULL)


@pytest.mark.parametrize("name", NAMES)
def test_restatement_equals_the_golden(name):
    frame, white = GOLDEN[f"{name}/frame"], bool(GOLDEN[f"{name}/white"])
    image, mask = canny_host.scene_images(frame[None], white)
    assert canny_host.canny(canny_host.canny_input(image[0])).tobytes() == GOLDEN[f"{name}/canny"].tobytes()
    assert mask[0].tobytes() == (1. - GOLDEN[f"{name}/canny"] / 255.).astype(np.float32).tobytes()
    if f"{name}/image" in GOLDEN.files:
        assert image[0].tobytes() == GOLDEN[f"{name}/image"].tobytes()


def test_golden_covers_the_rules():
    edges = {n: int((GOLDEN[f"{n}/canny"] > 0).sum()) for n in NAMES}
    # threshold brackets: 50 and 150 are not exceeded, 52 and 152 are
    assert edges["bump_m150"] == 0 and edges["bump_m152"] > 0 and edges["step_m148"] == 0 and edges["step_m152"] > 0
    u8 = canny_host.canny_input(canny_host.composite(GOLDEN["bump_m52/frame"][None], False)[0])
    cand, strong = canny_host.classify(u8)
    assert cand.any() and not strong.any()
    # a vertical step marks the column left of it, a horizontal one the row above it
    c = GOLDEN["plateau_v/canny"]
    assert (c[:, 5] == 255).all() and (np.delete(c, 5, axis=1) == 0).all()
    c = GOLDEN["plateau_h/canny"]
    assert (c[5] == 255).all() and (np.delete(c, 5, axis=0) == 0).all()
    # outermost rows and columns can be edges
    assert (GOLDEN["border_col0/canny"][:, 0] == 255).all() and (GOLDEN["border_rowN/canny"][-2] == 255).all()
    # hysteresis follows a weak chain from its one strong end across the whole frame
    assert edges["chain_spiral_512"] > 60_000 and edges["chain_spiral"] > 1000
    shapes = {GOLDEN[f"{n}/frame"].shape[:2] for n in NAMES}
    assert {(3, 3), (5, 7), (512, 512)} <= shapes
    assert {GOLDEN[f"{n}/frame"].shape[2] for n in NAMES} == {3, 4}
    assert {int(GOLDEN[f"{n}/white"]) for n in NAMES} == {0, 1}


def test_sobel_magnitude_is_always_even():
    rng = np.random.default_rng(3)
    for _ in range(20):
        _, _, m = canny_host.gradient(rng.integers(0, 256, (9, 13, 3)).astype(np.uint8))
        assert (m % 2 == 0).all()


def test_canny_input_gives_back_the_frame_bytes():
    """With alpha 255, `(float32(u / 255.0) * 255.).astype(uint8)` is u for every byte value (numpy 2 keeps the
    product float32), so the Canny input of a frame from align_frames is the frame itself."""
    u = np.arange(256, dtype=np.uint8)
    frame = np.stack([u.reshape(16, 16)] * 3, -1)
    image = canny_host.composite(frame[None], False)[0]
    assert image.dtype == np.float32
    assert (canny_host.canny_input(image) == frame).all()
    arr = torch.Tensor(u[:, None] / 255.0 * (255 / 255.0) + np.array([0]) * (1 - 255 / 255.0)).numpy()
    assert ((arr * 255.).dtype == np.float32) and ((arr * 255.).astype(np.uint8)[:, 0] == u).all()


def test_restatement_matches_opencv_on_seeded_frames():
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(11)
    for k in range(60):
        H, W = (int(v) for v in rng.integers(3, 48, 2))
        u = rng.integers(0, 256, (H, W, 3)).astype(np.uint8)
        if k % 2:
            u = cv2.GaussianBlur(u, (0, 0), 1.0 + k % 3)
        assert (cv2.Canny(u, 50, 150) == canny_host.canny(u)).all(), (k, H, W)


def test_header_and_ctypes_symbol_tables_agree():
    header = open(os.path.join(ROOT, "include", "gsscene.h")).read()
    declared = re.findall(r"^int (gsscene_\w+)\(", header, re.M)
    assert declared == [s[0] for s in scene.SYMBOLS]
    exported = subprocess.run(["nm", "-D", "--defined-only", scene.LIB_PATH], capture_output=True, text=True,
                              check=True).stdout
    assert sorted(re.findall(r" T (gsscene_\w+)", exported)) == sorted(declared)
    for name, _, args in scene.SYMBOLS:
        decl = re.search(rf"int {name}\(([^)]*)\)", header).group(1)
        n = 0 if decl.strip() == "void" else decl.count(",") + 1
        assert n == len(args), name


def test_argument_errors_and_scratch():
    L = scene.lib()
    assert L.gsscene_abi_version() == 1
    b = C.c_uint64()
    sizes = []
    for F, H, W in ((0, 1, 1), (1, 3, 3), (1, 512, 512), (50, 512, 512)):
        assert L.gsscene_scratch_bytes(F, H, W, C.byref(b)) == 0
        assert b.value % 256 == 0
        sizes.append(b.value)
    assert sizes == sorted(sizes) and sizes[-1] >= 17 * 50 * 512 * 512
    for F, H, W in ((-1, 8, 8), (1, 0, 8), (1, 8, 0), (1 << 14, 512, 512)):
        assert L.gsscene_scratch_bytes(F, H, W, C.byref(b)) == -22
    assert L.gsscene_scratch_bytes(2, 8, 8, None) == -22
    assert L.gsscene_scratch_bytes(2, 8, 8, C.byref(b)) == 0
    need = b.value
    A = 1 << 20                                            # fake, well-aligned device addresses: never dereferenced
    args = dict(frames=A, F=2, H=8, W=8, C=3, white=0, image=A, canny=A, scratch=A, bytes=need)

    def call(**kw):
        a = dict(args, **kw)
        return L.gsscene_camera_images(a["frames"], a["F"], a["H"], a["W"], a["C"], a["white"], a["image"],
                                       a["canny"], a["scratch"], a["bytes"], None)
    # every call below has exactly one invalid argument, so none of them reaches a device
    bad = [dict(frames=None), dict(F=-1), dict(H=0), dict(W=0), dict(C=1), dict(C=5), dict(white=2), dict(white=-1),
           dict(image=None), dict(image=A + 2), dict(canny=None), dict(canny=A + 1), dict(scratch=None),
           dict(scratch=A + 128), dict(bytes=need - 1)]
    for kw in bad:
        assert call(**kw) == -22, kw
    assert call(F=0, bytes=0) == -22                       # even an empty scene needs its (minimal) scratch
    assert call(F=0) == 0                                  # nothing to enqueue


def test_kernels_have_no_spills_and_no_float_atomics():
    log = open(os.path.join(CSRC, "gs_scene.o.ptxas.log")).read()
    spills = re.findall(r"(\d+) bytes spill stores, (\d+) bytes spill loads", log)
    assert len(spills) == 6 and all(s == ("0", "0") for s in spills)
    sass = subprocess.run(["cuobjdump", "-sass", os.path.join(CSRC, "gs_scene.o")], capture_output=True, text=True,
                          check=True).stdout
    for k in ("k_composite", "k_gradient", "k_classify", "k_union", "k_resolve", "k_output"):
        assert k in sass
    assert "sm_90a" in subprocess.run(["cuobjdump", "-lelf", os.path.join(CSRC, "gs_scene.o")], capture_output=True,
                                      text=True, check=True).stdout
    assert not re.search(r"\b(RED|ATOM|ATOMS)\.[A-Z0-9.]*F(16|32|64)", sass)
    assert re.search(r"\b(ATOM|RED)G?\.[A-Z.]*MIN", sass)             # the union-find links by integer atomicMin


def test_camera_images_checks_its_inputs():
    for bad in (np.zeros((1, 4, 4, 3), np.uint8), torch.zeros(1, 4, 4, 3, dtype=torch.uint8)):
        with pytest.raises(TypeError):
            scene.camera_images(bad, False)


def test_host_matrices_follow_the_reference_expressions():
    """Spot checks of the numpy restatements: a pose round-trips through rotation_translation and world_to_view,
    and the projection has getProjectionMatrix's entries."""
    c2w = np.eye(4)
    c2w[:3, 3] = [0.5, -0.25, 2.0]
    R, T = scene.rotation_translation(c2w.tolist())
    assert R.dtype == np.float64 and T.shape == (3,)
    wv = scene.world_to_view(R, T)
    assert wv.dtype == np.float32
    assert np.allclose(np.linalg.inv(wv)[:3, 3], [0.5, -0.25, 2.0], atol=1e-6)      # the camera centre
    P = scene.projection(0.01, 100.0, 1.0, 0.8)
    assert P.dtype == np.float32 and P[3, 2] == 1.0 and P[0, 2] == 0.0
    assert P[0, 0] == np.float32(1 / np.tan(0.5)) and P[2, 3] == np.float32(-1.0 / (100.0 - 0.01))
