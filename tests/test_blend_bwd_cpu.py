"""The backward tile pass (gs_blend_bwd.cu) on its machine code, without a GPU: spills and shared memory within the
bounds of the shuffle-butterfly pass it replaced, the occupancy targets it launches with, no double precision beyond
the two prologue products, and 128-bit vector reductions leaving k_blend_bwd."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "luciddreamer_b200", "csrc")


def _ptxas(obj):
    log = os.path.join(CSRC, obj + ".ptxas.log")
    if not os.path.exists(log):
        pytest.skip(f"{obj}.ptxas.log not built")
    per, fn = {}, None
    for line in open(log):
        m = re.search(r"Compiling entry function '(\S+)'", line)
        if m:
            fn = m.group(1)
            continue
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and fn:
            per.setdefault(fn, {})["spill"] = (int(m.group(1)), int(m.group(2)))
        m = re.search(r"Used (\d+) registers.*?(\d+) bytes smem", line)
        if m and fn:
            per.setdefault(fn, {}).update(regs=int(m.group(1)), smem=int(m.group(2)))
    return per


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
            per[fn] = []
            continue
        m = re.match(r"\s+/\*[0-9a-f]{4}\*/\s+(?:@!?U?P\w+\s+)?([A-Za-z0-9_.]+)", line)
        if m and fn:
            per[fn].append(m.group(1))
    return per


def test_resources_stay_within_the_butterfly_bounds_and_keep_the_occupancy_targets():
    per = _ptxas("gs_blend_bwd.o")
    assert len(per) == 4
    for fn, r in per.items():
        nh2 = "ILi2ELi13E" in fn
        assert nh2 or "ILi1ELi7E" in fn, fn
        # spills: at most the butterfly pass's (4 bytes stored, 8 loaded by its k_blend_bwd<2,13>), 4 bytes each way
        # for the kernels where it spilled nothing
        max_st, max_ld = (4, 8) if nh2 and "k_blend_bwd" in fn else (4, 4)
        assert r["spill"][0] <= max_st and r["spill"][1] <= max_ld, (fn, r)
        # 13 CTAs of 64 threads / 7 of 128 per SM: registers and shared memory (1 KB reserved per CTA) both fit
        ctas, threads = (13, 64) if nh2 else (7, 128)
        assert r["regs"] * threads * ctas <= 65536, (fn, r)
        assert (r["smem"] + 1024) * ctas <= 228 * 1024, (fn, r)
        if nh2:
            assert r["smem"] <= 15432 + 128, (fn, r["smem"])                  # the butterfly pass's 15 432 B + 128


def test_vector_reductions_and_no_double_precision_in_the_loop():
    per = _sass("gs_blend_bwd.o")
    assert len(per) == 4
    for fn, ops in per.items():
        assert not [o for o in ops if o.startswith(("HMMA", "HGMMA", "DFMA", "DADD"))], fn
        assert sum(o.startswith("DMUL") for o in ops) <= 2, fn          # 0.5 * W, 0.5 * H of the prologue
        assert not [o for o in ops if o.startswith("SHFL")] or ops.count("SHFL.BFLY") <= 5, fn   # n_contrib max only
        if "k_blend_bwd" in fn:
            assert any(o.startswith("REDG.E.ADD.F32x4") for o in ops), fn
        else:
            assert not [o for o in ops if o.startswith(("RED", "ATOM"))], fn
