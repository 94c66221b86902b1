"""Device colour mapping of depth clips (gs_colorize_depth via video.colorize_frames) against the host restatement
video.colorize and np.percentile itself: every byte equal, vmin / vmax equal (== , so -0.0 == +0.0), on rendered clips
and on frames built to hit numpy's float32 percentile arithmetic."""
import numpy as np
import pytest
import torch
from numpy.lib import _function_base_impl as npf

from luciddreamer_b200 import GaussianRasterizationSettings, synthetic as syn, video

pytestmark = pytest.mark.gpu

INVALID = np.float32(-99)
BG = (128, 128, 128, 255)


def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return torch.device("cuda:0")


def host(frame):
    """video.colorize of one [H,W] frame, as [H,W,4] (colorize squeezes unit dimensions).  A 1x1 frame squeezes to a
    0-d array, which colorize cannot index; it is coloured as a 1x2 frame whose second pixel is invalid (invalid pixels
    take no part in the percentiles), and the first pixel is kept."""
    if frame.size == 1:
        return video.colorize(np.array([[frame.reshape(-1)[0], INVALID]], np.float32))[:1].reshape(frame.shape + (4,))
    return video.colorize(frame).reshape(frame.shape + (4,))


def device(frames):
    rgba, vmm = video.colorize_frames(torch.from_numpy(np.ascontiguousarray(frames, np.float32)).to(dev()))
    torch.cuda.synchronize()
    return rgba.cpu().numpy(), vmm.cpu().numpy()


def check(frames, rgba=None, vmm=None):
    """Every frame of `frames` [F,H,W] through the device equals the host, byte for byte, and its percentiles."""
    frames = np.asarray(frames, np.float32)
    if rgba is None:
        rgba, vmm = device(frames)
    assert rgba.shape == frames.shape + (4,) and rgba.dtype == np.uint8 and vmm.shape == (frames.shape[0], 2)
    for k, fr in enumerate(frames):
        np.testing.assert_array_equal(rgba[k], host(fr), err_msg=f"frame {k}")
        valid = fr[fr != INVALID]
        assert vmm[k, 0] == np.percentile(valid, 2), (k, vmm[k, 0], np.percentile(valid, 2))
        assert vmm[k, 1] == np.percentile(valid, 98), (k, vmm[k, 1], np.percentile(valid, 98))
    return rgba, vmm


def linear_index(n, p):
    """numpy's own float32 virtual index of np.percentile(float32 data of size n, p) (method 'linear')."""
    return npf._QuantileMethods["linear"]["get_virtual_index"](n, np.float32(p) / np.float32(100))


# ------------------------------------------------------------------------------------------------ rendered clips
def _clip(W, H, F, P=20_000, seed=77):
    d = dev()
    sc = {k: v.to(d) for k, v in syn.make_scene(P, seed, scale_mult=2.0).items()}
    poses = syn.rotate360_poses(F)
    settings = []
    for k in range(F):
        cam = syn.make_camera(W, H, c2w=poses[k])
        settings.append(GaussianRasterizationSettings(H, W, cam.tanfovx, cam.tanfovy, torch.zeros(3, device=d), 1.0,
                                                      cam.viewmatrix.to(d), cam.projmatrix.to(d), 3, cam.campos.to(d),
                                                      False, False))
    return sc, settings


@pytest.mark.parametrize("W,H", [(160, 90), (512, 512)])
def test_rendered_clip_depth_rgba_equals_host_colorize(W, H):
    F = 8
    sc, settings = _clip(W, H, F)
    frames, depths, dmin, dmax, idx = video.render_video_frames(sc, settings)
    frames_c, rgba, dmin_c, dmax_c, idx_c = video.render_video_frames(sc, settings, depth_rgba=True)
    assert idx == idx_c == list(range(F))
    assert rgba.shape == (F, H, W, 4) and rgba.dtype == np.uint8
    np.testing.assert_array_equal(frames_c, frames)
    assert (dmin_c, dmax_c) == (dmin, dmax)
    for k in range(F):
        np.testing.assert_array_equal(rgba[k], host(depths[k]), err_msg=f"frame {k}")
    assert len({host(depths[k]).tobytes() for k in range(F)}) > 1          # the clip is not one repeated frame
    f1, rgba1, _a, _b, idx1 = video.render_video_frames(sc, settings, rank=1, world=2, depth_rgba=True)
    assert idx1 == list(range(1, F, 2))
    np.testing.assert_array_equal(f1, frames[1::2])
    np.testing.assert_array_equal(rgba1, rgba[1::2])


def test_depth_rgba_needs_depth():
    sc, settings = _clip(64, 48, 1, P=100)
    with pytest.raises(ValueError):
        video.render_video_frames(sc, settings, with_depth=False, depth_rgba=True)


# ------------------------------------------------------------------------------------------------ crafted frames
def _with_invalid(rng, frame, n_valid):
    """frame with all but n_valid pixels (random positions) set to invalid_val."""
    out = frame.copy().reshape(-1)
    keep = rng.permutation(out.size)[:n_valid]
    mask = np.ones(out.size, bool)
    mask[keep] = False
    out[mask] = INVALID
    return out.reshape(frame.shape)


def test_ties_on_the_selected_ranks():
    rng = np.random.default_rng(1)
    H, W = 37, 41
    n = H * W
    frames = []
    for levels in (2, 3, 5, 50):                              # few distinct values: every rank sits inside a tie
        frames.append(rng.integers(0, levels, n).astype(np.float32).reshape(H, W) - 2.5)
    i2, i98 = int(np.floor(linear_index(n, 2))), int(np.floor(linear_index(n, 98)))
    for lo_tie, hi_tie in ((True, False), (False, True), (True, True)):
        s = np.arange(n, dtype=np.float32) * 0.25 - 100.0     # distinct, then ties put exactly across lo / lo+1
        if lo_tie:
            s[i2 - 3: i2 + 1] = s[i2 - 3]                     # tie ends on the lower order statistic
            s[i2 + 1: i2 + 6] = s[i2 + 1]                     # a new tie starts at the upper one
        if hi_tie:
            s[i98: i98 + 2] = s[i98]                          # lower and upper order statistic tied
        frames.append(rng.permutation(s).reshape(H, W))
    check(np.stack(frames))


def test_constant_frames_map_to_the_first_colour():
    rng = np.random.default_rng(2)
    H, W = 24, 40
    c = np.full((H, W), 3.5, np.float32)
    z = np.full((H, W), -0.0, np.float32)
    z.reshape(-1)[rng.permutation(H * W)[:300]] = 0.0          # +0 and -0 are one value
    frames = np.stack([c, _with_invalid(rng, c, 17), z, _with_invalid(rng, z, 500)])
    rgba, vmm = check(frames)
    lut0 = tuple(video.jet_lut()[0])
    for k, fr in enumerate(frames):
        assert (rgba[k][fr != INVALID] == lut0).all() and (rgba[k][fr == INVALID] == BG).all()
        assert vmm[k, 0] == vmm[k, 1]


def test_invalid_pixels_down_to_one_and_two_valid():
    rng = np.random.default_rng(3)
    H, W = 19, 23
    base = -rng.uniform(0.5, 8.0, (H, W)).astype(np.float32)
    counts = [1, 2, 3, 4, 7, 50, 51, 52, 200, H * W - 1, H * W]
    check(np.stack([_with_invalid(rng, base, c) for c in counts]))


def test_signs_of_zero():
    """What gs_pack_frame writes: -0.0 background, +0.0 where depth <= 0, negative depths elsewhere."""
    rng = np.random.default_rng(4)
    H, W = 64, 48
    frames = []
    for frac_bg, frac_pos in ((0.9, 0.05), (0.5, 0.3), (0.02, 0.01), (0.97, 0.0), (0.0, 0.97)):
        u = rng.uniform(size=(H, W))
        fr = -rng.uniform(0.1, 5.0, (H, W)).astype(np.float32)
        fr[u < frac_bg] = -0.0
        fr[(u >= frac_bg) & (u < frac_bg + frac_pos)] = 0.0
        frames.append(fr)
    frames.append(_with_invalid(rng, frames[0], 1000))
    check(np.stack(frames))


def test_magnitudes_from_1e_30_to_1e30_and_denormals():
    rng = np.random.default_rng(5)
    H, W = 50, 60
    n = H * W
    mags = (10.0 ** rng.uniform(-30, 30, n)) * rng.choice([-1.0, 1.0], n)
    den = (rng.integers(1, 1 << 23, n).astype(np.uint32) | (rng.integers(0, 2, n).astype(np.uint32) << 31)).view(np.float32)
    assert (np.abs(den) < np.finfo(np.float32).tiny).all()
    mixed = np.where(rng.uniform(size=n) < 0.5, mags, den).astype(np.float32)
    small = (10.0 ** rng.uniform(-30, -25, n)).astype(np.float32)
    frames = [a.astype(np.float32).reshape(H, W) for a in (mags, den, mixed, small)]
    frames.append(_with_invalid(rng, frames[2], 777))
    check(np.stack(frames))


def _gammas(p, limit=20_000):
    return [(n, float(linear_index(n, p) - np.floor(linear_index(n, p)))) for n in range(2, limit)]


def test_integer_index_and_gamma_around_one_half():
    """Sizes where numpy's float32 index is an integer (gamma = 0), where gamma is exactly 0.5 (the b - (b-a)*(1-t)
    branch of _lerp), and where it is closest to 0.5 from below and from above."""
    rng = np.random.default_rng(6)
    H, W = 100, 200
    sizes = set()
    for p in (2, 98):
        g = _gammas(p)
        exact = [n for n, t in g if t == 0.0][:6]
        half = [n for n, t in g if t == 0.5][:3]
        below = [n for n, t in sorted((x for x in g if x[1] < 0.5), key=lambda x: 0.5 - x[1])][:3]
        above = [n for n, t in sorted((x for x in g if x[1] > 0.5), key=lambda x: x[1] - 0.5)][:3]
        assert len(exact) == 6 and len(half) == 3 and len(below) == 3 and len(above) == 3, (p, exact, half, below, above)
        sizes.update(exact + half + below + above)
    sizes = sorted(sizes)
    frames = []
    for n in sizes:
        fr = np.full(H * W, INVALID, np.float32)
        fr[rng.permutation(H * W)[:n]] = -rng.uniform(0.1, 9.0, n).astype(np.float32)
        frames.append(fr.reshape(H, W))
    check(np.stack(frames))


def _float64_indexes(n, p):
    """The percentile index under three double-precision restatements of numpy's: (n-1) * p/100, (n-1) * float32(p/100),
    and numpy's _compute_virtual_index evaluated in double."""
    q32 = float(np.float32(p) / np.float32(100))
    return [(n - 1) * (p / 100.0), (n - 1) * q32, npf._compute_virtual_index(float(n), p / 100.0, 1.0, 1.0)]


def _sizes_float32_vs_float64(p, limit=300_000):
    out = []
    for n in range(2, limit):
        lo = int(np.floor(linear_index(n, p)))
        if any(int(np.floor(v)) != lo for v in _float64_indexes(n, p)):
            out.append(n)
    return out


def _double_percentile(s, v):
    """Linear interpolation at index v in double precision (s sorted), rounded to float32 once."""
    lo = int(np.floor(v))
    a, b = float(s[lo]), float(s[min(lo + 1, len(s) - 1)])
    return np.float32(a + (b - a) * (v - lo))


@pytest.mark.parametrize("p", [2, 98])
def test_sizes_where_float32_and_float64_index_arithmetic_pick_different_ranks(p):
    """numpy evaluates the percentile index in float32 for float32 data; a double restatement takes another order
    statistic at these sizes.  Each frame puts a wide gap right below numpy's lower order statistic, so taking the other
    one changes vmin / vmax (checked here against a double-precision evaluation)."""
    sizes = _sizes_float32_vs_float64(p)
    assert len(sizes) >= 50, len(sizes)
    rng = np.random.default_rng(7 + p)
    pick = sorted(set(sizes[:10]) | set(sizes[:: max(1, len(sizes) // 50)]))[:60]
    H, W = 550, 550
    assert max(pick) <= H * W
    frames = []
    for n in pick:
        lo = int(np.floor(linear_index(n, p)))
        s = (np.arange(n, dtype=np.float64) - lo + 0.5).astype(np.float32)    # s[lo] = 0.5, s[lo + 1] = 1.5
        s[:lo] -= np.float32(1e6)                                             # wide gap below numpy's rank
        fr = np.full(H * W, INVALID, np.float32)
        fr[rng.permutation(H * W)[:n]] = rng.permutation(s)
        frames.append(fr.reshape(H, W))
        want = np.percentile(s, p)
        others = [v for v in _float64_indexes(n, p) if int(np.floor(v)) != lo]
        assert others and all(_double_percentile(s, v) != want for v in others), n
    check(np.stack(frames))


@pytest.mark.parametrize("H,W", [(1, 1), (7, 13), (1080, 1920), (1, 300), (300, 1)])
def test_frame_shapes(H, W):
    rng = np.random.default_rng(H * 7919 + W)
    fr = -rng.uniform(0.1, 20.0, (H, W)).astype(np.float32)
    fr[rng.uniform(size=(H, W)) < 0.3] = -0.0
    frames = [fr]
    if H * W > 1:
        frames.append(_with_invalid(rng, fr, max(1, H * W // 3)))
    check(np.stack(frames))


# ------------------------------------------------------------------------------------------------ batches
@pytest.mark.parametrize("F", [1, 64])
def test_each_frame_of_a_batch_equals_that_frame_alone(F):
    rng = np.random.default_rng(F)
    H, W = 45, 67                                              # H * W odd: frames after the first are unaligned
    frames = []
    for k in range(F):
        fr = -rng.uniform(0.1, 10.0, (H, W)).astype(np.float32)
        fr[rng.uniform(size=(H, W)) < 0.2] = -0.0
        frames.append(_with_invalid(rng, fr, int(rng.integers(1, H * W + 1))))
    frames = np.stack(frames)
    rgba, vmm = check(frames)
    for k in range(F):
        r1, v1 = device(frames[k: k + 1])
        np.testing.assert_array_equal(r1[0], rgba[k])
        np.testing.assert_array_equal(v1[0], vmm[k])
    # the same batch from a base pointer that is not 16-byte aligned (scalar loads / stores for every frame)
    flat = torch.from_numpy(frames.reshape(-1)).to(dev())
    buf = torch.empty(flat.numel() + 1, dtype=torch.float32, device=dev())
    buf[1:] = flat
    r2, v2 = video.colorize_frames(buf[1:].view(F, H, W))
    np.testing.assert_array_equal(r2.cpu().numpy(), rgba)
    np.testing.assert_array_equal(v2.cpu().numpy(), vmm)
    assert r2.is_contiguous()


def test_frame_without_valid_pixels_is_background_with_nan_percentiles():
    rng = np.random.default_rng(9)
    H, W = 33, 20
    good = -rng.uniform(0.5, 3.0, (H, W)).astype(np.float32)
    empty = np.full((H, W), INVALID, np.float32)
    frames = np.stack([good, empty, good[::-1].copy(), empty])
    with pytest.raises(IndexError):
        video.colorize(empty)                                  # numpy: percentile of an empty selection
    rgba, vmm = device(frames)
    for k in (1, 3):
        assert (rgba[k] == BG).all()
        assert np.isnan(vmm[k]).all()
    check(frames[[0, 2]], rgba[[0, 2]], vmm[[0, 2]])


def test_graph_capture_replays_the_same_bytes():
    rng = np.random.default_rng(10)
    F, H, W = 6, 90, 160
    frames = -rng.uniform(0.1, 10.0, (F, H, W)).astype(np.float32)
    frames[rng.uniform(size=frames.shape) < 0.1] = INVALID
    static_in = torch.from_numpy(frames).to(dev())
    eager = video.colorize_frames(static_in)                   # warm-up (copies the colour table) and reference
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out_rgba, out_vmm = video.colorize_frames(static_in)
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(out_rgba, eager[0]) and torch.equal(out_vmm, eager[1])
    frames2 = frames[::-1].copy()
    frames2[0, :5] = INVALID
    static_in.copy_(torch.from_numpy(frames2))
    for _ in range(2):
        g.replay()
    torch.cuda.synchronize()
    check(frames2, out_rgba.cpu().numpy(), out_vmm.cpu().numpy())
