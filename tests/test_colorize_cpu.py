"""Depth colour mapping without a GPU: the two C entry points are declared and exported, reject bad arguments with
GS_EINVAL before touching the device, size their scratch monotonically, compile without spills or float atomics, and
video.colorize_frames rejects what it cannot take."""
import collections
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

from luciddreamer_b200 import _native as N, video

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "luciddreamer_b200", "csrc")
NEW = ("gs_colorize_depth", "gs_colorize_scratch_bytes")
FAKE = 1 << 20          # a well-aligned non-NULL address; never dereferenced because every call below is rejected


def test_header_declares_and_library_exports_the_colorize_entry_points():
    src = open(os.path.join(ROOT, "include", "gsraster.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    L = N.lib()
    for name in NEW:
        assert re.search(r"\b" + name + r"\s*\(", src), name
        assert hasattr(L, name), name
        assert name in [s[0] for s in N.SYMBOLS], name
    assert L.gs_abi_version() == 2
    assert L.gs_profile_num_kernels() == 12


def test_scratch_size_is_monotone_in_frames():
    f = N.lib().gs_colorize_scratch_bytes
    assert f(0) == 0 and f(-3) == 0
    sizes = [f(F) for F in (1, 2, 3, 8, 64, 720, 1440, 100_000)]
    assert all(b > a for a, b in zip(sizes, sizes[1:]))
    assert f(1) <= 64 * 1024 and f(1440) == 1440 * f(1)


def _call(F=2, H=8, W=8, value=FAKE, lut=FAKE, scratch=FAKE, nbytes=None, rgba=FAKE, vmm=FAKE):
    L = N.lib()
    if nbytes is None:
        nbytes = L.gs_colorize_scratch_bytes(F) if F > 0 else 0
    return L.gs_colorize_depth(None, F, H, W, value, -99.0, lut, 0xff808080, scratch, nbytes, rgba, vmm, None)


@pytest.mark.parametrize("kw,msg", [
    (dict(F=0), b"sizes"), (dict(F=-1), b"sizes"), (dict(H=0), b"sizes"), (dict(W=-5), b"sizes"),
    (dict(H=65536, W=65536), b"too large"),
    (dict(value=None), b"NULL"), (dict(lut=None), b"NULL"), (dict(scratch=None), b"NULL"), (dict(rgba=None), b"NULL"),
    (dict(value=FAKE + 2), b"aligned"), (dict(lut=FAKE + 1), b"aligned"), (dict(rgba=FAKE + 3), b"aligned"),
    (dict(vmm=FAKE + 2), b"aligned"), (dict(scratch=FAKE + 8), b"aligned"),
    (dict(nbytes=0), b"scratch"),
])
def test_bad_arguments_return_einval(kw, msg):
    assert _call(**kw) == -1
    assert msg in N.lib().gs_last_error(), N.lib().gs_last_error()


def test_short_scratch_is_rejected_by_one_byte():
    need = N.lib().gs_colorize_scratch_bytes(5)
    assert _call(F=5, nbytes=need - 1) == -1
    assert b"scratch" in N.lib().gs_last_error()


def test_colorize_frames_rejects_cpu_wrong_dtype_and_wrong_shape():
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        video.colorize_frames(torch.zeros(2, 4, 4))
    with pytest.raises(ValueError, match="float32"):
        video.colorize_frames(torch.zeros(2, 4, 4, dtype=torch.float64))
    with pytest.raises(ValueError, match=r"\[F,H,W\]"):
        video.colorize_frames(torch.zeros(4, 4))
    with pytest.raises(ValueError, match=r"\[F,H,W\]"):
        video.colorize_frames(torch.zeros(1, 2, 4, 4))
    with pytest.raises(ValueError):
        video.colorize_frames(np.zeros((2, 4, 4), np.float32))


def test_device_defaults_come_from_the_host_colorize():
    assert video._INVALID_VAL == -99
    assert video._BACKGROUND_RGBA.to_bytes(4, "little") == bytes((128, 128, 128, 255))


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


def test_colorize_kernels_use_no_float_atomics_and_no_double_precision():
    per = _sass("gs_colorize.o")
    for name in ("k_cz_hist", "k_cz_select", "k_cz_color"):
        assert any(name in k for k in per), name
    assert len([k for k in per if "k_cz_hist" in k]) == 3 and len([k for k in per if "k_cz_select" in k]) == 3
    for fn, c in per.items():
        bad = [op for op in c if (op.startswith(("REDG", "ATOMG", "RED.", "ATOM.", "ATOMS")) and ".F32" in op)
               or op.startswith(("DADD", "DMUL", "DFMA"))]
        assert not bad, (fn, bad)
    # one 128-bit store per four pixels in the colour pass
    assert any(op.startswith("STG.E.128") for op in next(c for k, c in per.items() if "k_cz_color" in k))


def test_colorize_kernels_do_not_spill():
    log = os.path.join(CSRC, "gs_colorize.o.ptxas.log")
    if not os.path.exists(log):
        pytest.skip("ptxas log not available (library not built by csrc/Makefile)")
    text = open(log).read()
    entries = re.findall(r"Function properties for (\S+)\n(.*spill.*)\n", text)
    assert len([e for e in entries if "k_cz_" in e[0]]) == 7
    for name, props in entries:
        assert "0 bytes spill stores, 0 bytes spill loads" in props, (name, props)
