"""The deterministic backward without a GPU: its two C entry points are declared, exported and sized within budget, its
kernels carry no float global reductions in the machine code, and the Python switch restores its previous state."""
import collections
import os
import re
import shutil
import subprocess

import pytest
import torch

from luciddreamer_b200 import _native as N

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "luciddreamer_b200", "csrc")
NEW = ("gs_backward_deterministic", "gs_backward_deterministic_scratch_bytes")


def test_header_declares_and_library_exports_the_deterministic_backward():
    src = open(os.path.join(ROOT, "include", "gsraster.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    L = N.lib()
    for name in NEW:
        assert re.search(r"\b" + name + r"\s*\(", src), name
        assert hasattr(L, name), name
        assert name in [s[0] for s in N.SYMBOLS], name
    assert L.gs_abi_version() == 2
    assert L.gs_profile_num_kernels() == 12


def test_scratch_grows_with_both_arguments_and_stays_within_budget():
    L = N.lib()
    f = L.gs_backward_deterministic_scratch_bytes
    for nvis in (1, 1000, 250_000, 2_000_000):
        for cap in (64, 100_000, 8_000_000):
            total, base = f(nvis, cap), L.gs_backward_scratch_bytes(nvis)
            assert total >= base
            # extra: at most ~64 B per pair of capacity + 16 B per visible Gaussian (+ alignment)
            assert total - base <= 64 * cap + 16 * nvis + 4096, (nvis, cap, total - base)
            assert f(nvis + 10_000, cap) > total and f(nvis, cap + 10_000) > total


def test_deterministic_backward_rejects_bad_arguments():
    L = N.lib()
    f = N.GsFrame()
    f.P, f.W, f.H = 0, 16, 16
    g = N.GsGrads()
    assert L.gs_backward_deterministic(None, f, None, None, None, 64, None, None, 0, None, None, None, None) == -1
    assert b"NULL" in L.gs_last_error()
    g.peer_world = 2
    assert L.gs_backward_deterministic(None, f, None, None, None, 64, None, None, 0, None, None, g, None) == -1
    assert b"peer" in L.gs_last_error()
    g.peer_world = 0
    assert L.gs_backward_deterministic(None, f, None, None, None, 64, None, None, 16, None, None, g, None) == -1
    assert b"scratch" in L.gs_last_error()


def _sass(obj):
    path = os.path.join(CSRC, obj)
    if not os.path.exists(path) or shutil.which("cuobjdump") is None:
        pytest.skip(f"{obj} or cuobjdump not available")
    out = subprocess.run(["cuobjdump", "-sass", path], capture_output=True, text=True, check=True).stdout
    per, fn = {}, None
    for line in out.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            fn = m.group(1)
            per[fn] = collections.Counter()
            continue
        m = re.match(r"\s+/\*[0-9a-f]{4}\*/\s+(?:@!?U?P\d\s+)?([A-Za-z0-9_.]+)", line)
        if m and fn:
            per[fn][m.group(1)] += 1
    return per


def test_running_deterministic_kernels_issue_no_float_reductions():
    per = {**_sass("gs_blend_bwd.o"), **_sass("gs_det_bwd.o")}
    new = {k: v for k, v in per.items() if "k_tile_partials" in k or "k_det_" in k}
    assert len([k for k in new if "k_tile_partials" in k]) == 2          # both warp geometries
    for name in ("k_det_count", "k_det_scan_reduce", "k_det_scan_down", "k_det_place", "k_det_sort_warp",
                 "k_det_sort_big", "k_det_gather"):
        assert any(name in k for k in new), name
    for fn, c in new.items():
        bad = [op for op in c if (op.startswith("REDG") or op.startswith("ATOMG") or op.startswith("RED.")
                                  or op.startswith("ATOM.")) and ".F32" in op]
        assert not bad, (fn, bad)
    # the partial-storing tile pass leaves the CTA through 128-bit stores
    for fn, c in new.items():
        if "k_tile_partials" in fn:
            assert any(op.startswith("STG.E.128") for op in c), fn


def test_switch_restores_the_previous_state():
    from luciddreamer_b200 import rasterizer as R
    assert not R.is_deterministic(0)
    with R.deterministic(device=0):
        assert R.is_deterministic(0)
        with R.deterministic(False, device=0):
            assert not R.is_deterministic(0)
        assert R.is_deterministic(0)
        R.set_deterministic(False, 0)
        assert not R.is_deterministic(0)
    assert not R.is_deterministic(0)
    R.set_deterministic(True, 0)
    with R.deterministic(device=0):
        pass
    assert R.is_deterministic(0)
    R.set_deterministic(False, 0)
    assert not R.is_deterministic(0)


def test_cpu_tensors_still_raise_in_deterministic_mode():
    from luciddreamer_b200 import GaussianRasterizationSettings, GaussianRasterizer
    from luciddreamer_b200 import rasterizer as R
    z = torch.zeros(3)
    rs = GaussianRasterizationSettings(8, 8, 0.4, 0.4, z, 1.0, torch.eye(4), torch.eye(4), 0, z, False, False)
    m = torch.zeros(4, 3)
    with R.deterministic(device=0):
        with pytest.raises(RuntimeError, match="no CPU fallback"):
            GaussianRasterizer(rs)(m, m, torch.zeros(4, 1), colors_precomp=m, scales=m, rotations=torch.zeros(4, 4))
