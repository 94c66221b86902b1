"""Training scene on the device (luciddreamer_b200.scene): camera images and Canny masks bit for bit against the
golden data and the host restatement, the device frames of pcd.align_frames against their PIL route, and
build_scene against the reference's own Scene, executed from bytecode (oracle/build_pyref_scene.py), camera by
camera, attribute by attribute, then one deterministic TrainStep iteration over each scene."""
import json
import os
import random
import sys
import types

import numpy as np
import pytest
import torch
from PIL import Image
from scipy import ndimage

import canny_host
import pcd_cases
from luciddreamer_b200 import pcd, scene

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = np.load(os.path.join(ROOT, "tests", "golden", "canny_golden.npz"))
NAMES = sorted({k.split("/")[0] for k in GOLDEN.files})
PRESETS = json.load(open(os.path.join(ROOT, "tests", "golden", "preset_cameras.json")))
PCD = json.load(open(os.path.join(ROOT, "tests", "golden", "pcd_golden.json")))
PYREF = os.path.join(ROOT, "oracle", "_ref", "pyref_scene")

TRAIN_ATTRS = ("uid", "colmap_id", "R", "T", "FoVx", "FoVy", "image_name", "data_device", "original_image",
               "canny_mask", "image_width", "image_height", "znear", "zfar", "trans", "scale", "world_view_transform",
               "projection_matrix", "full_proj_transform", "camera_center")
PRESET_ATTRS = ("image_width", "image_height", "FoVy", "FoVx", "znear", "zfar", "world_view_transform",
                "full_proj_transform", "camera_center")


def device_images(frames: np.ndarray, white: bool):
    img, mask = scene.camera_images(torch.from_numpy(np.ascontiguousarray(frames)).cuda(), white)
    return img.cpu().numpy(), mask.cpu().numpy()


def golden_mask(name):
    return (1. - GOLDEN[f"{name}/canny"] / 255.).astype(np.float32)


@pytest.mark.parametrize("name", NAMES)
def test_golden_frames_one_at_a_time(name):
    """F = 1: every golden frame, as given and, for three-channel frames, as RGBA and over the other background
    (alpha 255 leaves both unchanged)."""
    frame, white = GOLDEN[f"{name}/frame"], bool(GOLDEN[f"{name}/white"])
    variants = [(frame, white)]
    if frame.shape[-1] == 3:
        variants += [(canny_host.rgba(frame), white), (frame, not white)]
    for f, w in variants:
        img, mask = device_images(f[None], w)
        h_img, h_mask = canny_host.scene_images(f[None], w)
        assert mask.dtype == np.float32 and mask.shape == (1,) + frame.shape[:2]
        assert mask[0].tobytes() == golden_mask(name).tobytes() == h_mask[0].tobytes(), (name, f.shape, w)
        assert img.tobytes() == h_img.tobytes(), (name, f.shape, w)
        if f"{name}/image" in GOLDEN.files:
            assert img[0].tobytes() == GOLDEN[f"{name}/image"].tobytes()


def fifty_frames(C: int) -> np.ndarray:
    """50 frames at 512 x 512: the golden's seeded and spiral frames, then smoothed seeded noise; with C = 4 a
    seeded alpha channel, opaque at 30 % of the pixels."""
    rng = np.random.default_rng(50 + C)
    out = [GOLDEN["seeded_512/frame"], GOLDEN["chain_spiral_512/frame"]]
    for k in range(48):
        u = rng.integers(0, 256, (512, 512, 3)).astype(np.float64)
        out.append(np.clip(np.round(ndimage.gaussian_filter(u, (0.8 + k % 4, 0.8 + k % 3, 0))), 0, 255)
                   .astype(np.uint8))
    f = np.stack(out)
    if C == 4:
        a = rng.integers(0, 256, f.shape[:3] + (1,)).astype(np.uint8)
        a[rng.random(a.shape) < 0.3] = 255
        f = np.concatenate([f, a], -1)
    return np.ascontiguousarray(f)


@pytest.mark.parametrize("C,white", [(3, False), (3, True), (4, False), (4, True)])
def test_fifty_frames_in_one_call(C, white):
    frames = fifty_frames(C)
    img, mask = device_images(frames, white)
    h_img, h_mask = canny_host.scene_images(frames, white)
    for k in range(len(frames)):
        assert mask[k].tobytes() == h_mask[k].tobytes(), k
        assert img[k].tobytes() == h_img[k].tobytes(), k
    if C == 3:
        assert mask[0].tobytes() == golden_mask("seeded_512").tobytes()
        assert mask[1].tobytes() == golden_mask("chain_spiral_512").tobytes()
    one_img, one_mask = device_images(frames[7:8], white)           # a frame alone gives what it gave in the batch
    assert one_img.tobytes() == img[7:8].tobytes() and one_mask.tobytes() == mask[7:8].tobytes()


def test_camera_images_are_capturable_and_repeatable():
    frames = torch.from_numpy(fifty_frames(3)[:4]).cuda()
    img0, mask0 = scene.camera_images(frames, False)
    g = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        with torch.cuda.graph(g, stream=s):
            img, mask = scene.camera_images(frames, False)
    torch.cuda.current_stream().wait_stream(s)
    for _ in range(3):
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(img, img0) and torch.equal(mask, mask0)
    g.reset()


def aligned_traindata(on_device: bool):
    """traindata as LucidDreamer.generate_pcd returns it, over the point-cloud warp's golden cloud and poses; with
    on_device its frames carry only their matrices, the images staying in the returned CUDA tensor."""
    H, W = PCD["H"], PCD["W"]
    pts, cols = pcd_cases.depth_cloud(PCD["cloud"]["seed"], H, W, extra=PCD["cloud"]["extra"])
    rp, hemi = np.array(PCD["render_poses"]), np.array(PCD["internal_poses"])
    frames, mats = pcd.align_frames(pts, cols, rp, hemi, np.array(PCD["K"]), H, W, on_device=on_device)
    data = {"camera_angle_x": 2 * np.arctan(W / (2 * PCD["K"][0][0])), "W": W, "H": H,
            "pcd_points": pts.astype(np.float64), "pcd_colors": cols, "frames": []}
    for k, m in enumerate(mats):
        data["frames"].append({"transform_matrix": m.tolist()} if on_device else
                              {"image": Image.fromarray(frames[k]), "transform_matrix": m.tolist()})
    return data, frames


class GaussianStub:
    """Records what build_scene asks of the Gaussian model."""

    def __init__(self):
        self.calls = []

    def create_from_pcd(self, pcd_, extent):
        self.calls.append(("create_from_pcd", pcd_.points, pcd_.colors, pcd_.normals, extent))

    def training_setup(self, opt):
        self.calls.append(("training_setup", opt))


def same(a, b, what):
    assert type(a) is type(b), (what, type(a), type(b))
    if isinstance(a, torch.Tensor):
        assert a.dtype == b.dtype and a.device == b.device and a.shape == b.shape and torch.equal(a, b), what
    elif isinstance(a, np.ndarray):
        assert a.dtype == b.dtype and a.shape == b.shape and a.tobytes() == b.tobytes(), what
    elif isinstance(a, (np.generic, float)):
        assert np.asarray(a).tobytes() == np.asarray(b).tobytes(), what
    else:
        assert a == b, what


def same_cameras(a, b, attrs, what):
    assert len(a) == len(b), what
    for k, (ca, cb) in enumerate(zip(a, b)):
        for n in attrs:
            same(getattr(ca, n), getattr(cb, n), f"{what}[{k}].{n}")


def test_align_frames_on_device_and_pil_frames_build_the_same_scene():
    data, frames_np = aligned_traindata(False)
    data_t, frames_t = aligned_traindata(True)
    assert isinstance(frames_np, np.ndarray) and frames_np.dtype == np.uint8
    assert frames_t.is_cuda and frames_t.dtype == torch.uint8 and frames_t.shape == frames_np.shape
    assert np.array_equal(frames_t.cpu().numpy(), frames_np)
    assert [f["transform_matrix"] for f in data["frames"]] == [f["transform_matrix"] for f in data_t["frames"]]
    opt = types.SimpleNamespace(white_background=False)
    ga, gb = GaussianStub(), GaussianStub()
    random.seed(5)
    a = scene.build_scene(data, ga, opt, PRESETS)
    state = random.getstate()
    random.seed(5)
    b = scene.build_scene(data_t, gb, opt, PRESETS, frames=frames_t)
    assert random.getstate() == state
    same_cameras(a.getTrainCameras(), b.getTrainCameras(), TRAIN_ATTRS, "train")
    assert list(a.preset_cameras) == list(b.preset_cameras) == list(PRESETS)
    for k in PRESETS:
        same_cameras(a.getPresetCameras(k), b.getPresetCameras(k), PRESET_ATTRS, k)
    same(a.cameras_extent, b.cameras_extent, "cameras_extent")
    assert [c[0] for c in ga.calls] == ["create_from_pcd", "training_setup"] == [c[0] for c in gb.calls]
    assert ga.calls[0][1].tobytes() == data["pcd_points"].T.tobytes() and ga.calls[0][3] is None
    # the masks come from the frames: the Canny input of an align_frames frame is the frame itself
    for c in a.getTrainCameras():
        f = frames_np[c.uid]
        assert c.canny_mask.cpu().numpy().tobytes() == (1. - canny_host.canny(f) / 255.).astype(np.float32).tobytes()
    # the per-camera tensors are views into shared buffers
    cams = a.getTrainCameras()
    assert len({c.original_image.untyped_storage().data_ptr() for c in cams}) == 1
    assert len({c.camera_center.untyped_storage().data_ptr() for c in cams}) == 1


# ---- the reference's own Scene


@pytest.fixture(scope="module")
def ref():
    """Imports the reference's Scene from bytecode, with this repo's packages underneath."""
    if not os.path.exists(os.path.join(PYREF, "scene", "__init__.pyc")):
        pytest.skip("oracle/_ref/pyref_scene not built (oracle/build_pyref_scene.py needs the reference checkout)")
    pytest.importorskip("cv2", reason="the reference's image2canny needs cv2")
    saved_path, saved_mods = list(sys.path), dict(sys.modules)
    ours = ("utils", "scene", "arguments", "plyfile", "imageio")
    for name in [m for m in sys.modules if m.split(".")[0] in ours]:
        del sys.modules[name]
    sys.path.insert(0, PYREF)
    if ROOT not in sys.path:
        sys.path.insert(1, ROOT)
    ply = types.ModuleType("plyfile")                       # only save_ply / fetchPly use these
    ply.PlyData = ply.PlyElement = object
    sys.modules["plyfile"] = ply
    sys.modules["imageio"] = types.ModuleType("imageio")    # only the COLMAP / Blender readers use it
    import arguments
    import scene as ref_scene
    from utils.trajectory import get_camerapaths
    assert ref_scene.__file__.startswith(PYREF) and ref_scene.__file__.endswith(".pyc")
    pillow_int8_shim(sys.modules["scene.dataset_readers"])
    yield types.SimpleNamespace(Scene=ref_scene.Scene, GaussianModel=ref_scene.GaussianModel,
                                GSParams=arguments.GSParams, get_camerapaths=get_camerapaths)
    sys.path[:] = saved_path
    for name in [m for m in sys.modules if m not in saved_mods and m.split(".")[0] in ours]:
        del sys.modules[name]
    sys.modules.update({n: m for n, m in saved_mods.items() if n.split(".")[0] in ours})


def pillow_int8_shim(dataset_readers):
    """loadCamerasFromData builds `Image.fromarray(np.array(arr * 255.0, dtype=np.byte), "RGB")` only to read its
    size; Pillow 12 refuses int8 data, so that module gets a `fromarray` that reads the same bytes as uint8."""
    dataset_readers.Image = types.SimpleNamespace(fromarray=lambda a, mode=None: Image.fromarray(
        np.ascontiguousarray(a).view(np.uint8)))


def gaussian_state(gm):
    out = {}
    for k, v in vars(gm).items():
        if isinstance(v, torch.Tensor) or isinstance(v, (int, float, np.generic)):
            out[k] = v
    out["groups"] = [{k: v for k, v in g.items() if k != "params"} for g in gm.optimizer.param_groups]
    out["group_params"] = [g["params"][0] for g in gm.optimizer.param_groups]
    return out


def same_gaussians(a, b):
    sa, sb = gaussian_state(a), gaussian_state(b)
    assert sa.keys() == sb.keys()
    for k in sa:
        if k in ("groups",):
            assert sa[k] == sb[k]
        elif k == "group_params":
            for x, y in zip(sa[k], sb[k]):
                same(x.detach(), y.detach(), "optimizer param")
        elif isinstance(sa[k], torch.Tensor):
            same(sa[k].detach(), sb[k].detach(), k)
        else:
            same(sa[k], sb[k], k)


@pytest.mark.parametrize("white", [False, True])
def test_build_scene_equals_the_reference_scene(ref, white):
    data, _ = aligned_traindata(False)
    opt = ref.GSParams()
    opt.white_background = white
    presets = ref.get_camerapaths()
    assert json.loads(json.dumps(presets)) == PRESETS
    random.seed(17)
    r = ref.Scene(data, ref.GaussianModel(opt.sh_degree), opt)
    state = random.getstate()
    random.seed(17)
    o = scene.build_scene(data, ref.GaussianModel(opt.sh_degree), opt, presets)
    assert random.getstate() == state
    assert [c.uid for c in o.getTrainCameras()] == [c.uid for c in r.getTrainCameras()]
    same_cameras(r.getTrainCameras(), o.getTrainCameras(), TRAIN_ATTRS, "train")
    assert list(r.preset_cameras) == list(o.preset_cameras)
    for k in r.preset_cameras:
        same_cameras(r.getPresetCameras(k), o.getPresetCameras(k), PRESET_ATTRS, k)
    same(r.cameras_extent, o.cameras_extent, "cameras_extent")
    same_gaussians(r.gaussians, o.gaussians)


def test_one_train_step_over_either_scene_is_identical(ref):
    from luciddreamer_b200 import optim, train
    from luciddreamer_b200 import rasterizer as R
    data, _ = aligned_traindata(False)
    opt = ref.GSParams()
    random.seed(23)
    r = ref.Scene(data, ref.GaussianModel(opt.sh_degree), opt)
    random.seed(23)
    o = scene.build_scene(data, ref.GaussianModel(opt.sh_degree), opt, ref.get_camerapaths())
    # the same fresh model trains over either scene's cameras: FusedAdam wants contiguous parameters, and
    # create_from_pcd keeps the strides of `pcd_points.T`, so the model is made from a contiguous copy
    cloud = scene.PointCloud(np.ascontiguousarray(data["pcd_points"].T), data["pcd_colors"], None)
    bg = torch.zeros(3, device="cuda")
    models = []
    with R.deterministic():
        for sc in (r, o):
            gm = ref.GaussianModel(opt.sh_degree)
            gm.create_from_pcd(cloud, sc.cameras_extent)
            gm.training_setup(opt)
            optim.attach(gm)
            ts = train.TrainStep(gm, sc.getTrainCameras(), bg, opt)
            ts.run(1, 0)
            ts.check()
            models.append(gm)
    torch.cuda.synchronize()
    a, b = models
    for n in ("_xyz", "_features_dc", "_features_rest", "_scaling", "_rotation", "_opacity"):
        same(getattr(a, n).detach(), getattr(b, n).detach(), n)
    assert float(b.optimizer.state[b._xyz]["step"]) == 1.0
    assert not torch.equal(b._xyz.detach(), torch.from_numpy(cloud.points).float().cuda())
