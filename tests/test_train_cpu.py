"""The training-step entry points without a GPU: exports, argument checks, the machine code of gs_train.cu, the unchanged
machine code of every kernel, and the host-built schedule tables."""
import ctypes as C
import glob
import json
import os
import re
import shutil
import subprocess
import sys

import numpy as np
import pytest

from luciddreamer_b200 import _native as N
from luciddreamer_b200 import optim, train

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "luciddreamer_b200", "csrc")
GOLDEN = os.path.join(ROOT, "tests", "golden")
NEW = ("gs_activate", "gs_adam_sched_scratch_bytes", "gs_adam_bias_table_len", "gs_adam_bias_table",
       "gs_gaussian_adam_sched_step", "gs_densify_stats_guarded", "gs_forward_release_graph_slot")
FAKE = 1 << 20          # a plausible, 256-byte aligned device address; every call below fails before touching it


def test_header_declares_and_library_exports_the_training_step():
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "gsraster.h")).read(), flags=re.S)
    L = N.lib()
    for name in NEW:
        assert re.search(r"\b" + name + r"\s*\(", src), name
        assert hasattr(L, name), name
        assert name in [s[0] for s in N.SYMBOLS], name
    assert L.gs_abi_version() == 2
    assert L.gs_profile_num_kernels() == 12
    assert C.sizeof(N.GsAdamSchedGroup) == 80


def test_activate_rejects_bad_arguments():
    L = N.lib()
    ok = [FAKE] * 9
    assert L.gs_activate(None, 0, 16, *[None] * 9, None) == 0                   # P = 0: nothing to do
    assert L.gs_activate(None, -1, 16, *ok, None) == -1
    assert L.gs_activate(None, 4, 0, *ok, None) == -1
    assert L.gs_activate(None, 4, 17, *ok, None) == -1
    for k in range(9):
        args = list(ok)
        args[k] = None
        assert L.gs_activate(None, 4, 16, *args, None) == -1, k
        assert b"NULL" in L.gs_last_error()
    for k in (4, 5, 8):                          # rotation, shs, rotations: 128-bit accesses
        args = list(ok)
        args[k] = FAKE + 4
        assert L.gs_activate(None, 4, 16, *args, None) == -1, k
        assert b"16-byte" in L.gs_last_error()
    args = list(ok)
    args[1] = FAKE + 2
    assert L.gs_activate(None, 4, 16, *args, None) == -1


def test_graph_slot_release_rejects_bad_arguments():
    L = N.lib()
    assert L.gs_forward_release_graph_slot(None, 0x40000000) == -1
    assert L.gs_forward_release_graph_slot(None, 5) == -1


def test_fused_adam_refuses_the_adam_options_it_does_not_implement():
    import torch
    p = torch.nn.Parameter(torch.zeros(4, 3))
    for kw in ({"weight_decay": 1e-2}, {"amsgrad": True}, {"maximize": True}):
        with pytest.raises(RuntimeError, match=next(iter(kw))):
            optim.FusedAdam([dict(params=[p], name="xyz", **kw)])
    o = optim.FusedAdam([dict(params=[p], name="xyz")], lr=0.0, eps=1e-15)
    with pytest.raises(RuntimeError, match="amsgrad"):
        o.add_param_group(dict(params=[torch.nn.Parameter(torch.zeros(2))], name="f_dc", amsgrad=True))


def _group(**kw):
    g = N.GsAdamSchedGroup()
    g.param, g.grad, g.exp_avg, g.exp_avg_sq, g.step = FAKE, FAKE, FAKE, FAKE, FAKE
    g.rows, g.row_width, g.grad_row_width, g.grad_offset, g.activation, g.lr = 10, 3, 3, 0, 0, 1e-3
    for k, v in kw.items():
        setattr(g, k, v)
    arr = (N.GsAdamSchedGroup * 1)()
    arr[0] = g
    return arr


def _sched(groups, n=1, betas=(0.9, 0.999), bias=(FAKE, FAKE, 100), it=None, lr_len=0, guard=(None, 0, 0, 0),
           scratch=(FAKE, 256)):
    L = N.lib()
    return L.gs_gaussian_adam_sched_step(None, groups, n, betas[0], betas[1], 1e-15, bias[0], bias[1], bias[2], it, lr_len,
                                         guard[0], guard[1], guard[2], guard[3], scratch[0], scratch[1], None)


def test_scheduled_adam_rejects_bad_arguments():
    L = N.lib()
    assert L.gs_adam_sched_scratch_bytes() >= 68
    assert _sched(None) == -1
    assert _sched(_group(), n=0) == -1 and _sched(_group(), n=9) == -1
    assert _sched(_group(), betas=(1.0, 0.999)) == -1
    assert _sched(_group(), bias=(None, FAKE, 100)) == -1 and _sched(_group(), bias=(FAKE, FAKE, 1)) == -1
    assert _sched(_group(), bias=(FAKE + 4, FAKE, 100)) == -1
    assert _sched(_group(), scratch=(None, 256)) == -1 and _sched(_group(), scratch=(FAKE, 16)) == -1
    assert _sched(_group(), scratch=(FAKE + 8, 256)) == -1
    for field in ("param", "grad", "exp_avg", "exp_avg_sq", "step"):
        assert _sched(_group(**{field: None})) == -1, field
        assert b"malformed" in L.gs_last_error()
    for field in ("param", "exp_avg", "exp_avg_sq"):
        assert _sched(_group(**{field: FAKE + 4})) == -1, field
    assert _sched(_group(step=FAKE + 2)) == -1 and _sched(_group(lr_table=FAKE + 4)) == -1
    assert _sched(_group(rows=-1)) == -1 and _sched(_group(activation=4)) == -1
    assert _sched(_group(row_width=0)) == -1 and _sched(_group(grad_row_width=2)) == -1
    assert _sched(_group(grad_offset=-1)) == -1
    assert _sched(_group(lr_table=FAKE)) == -1                          # a table needs the device iteration
    assert b"iteration" in L.gs_last_error()
    assert _sched(_group(lr_table=FAKE), it=FAKE, lr_len=0) == -1
    assert _sched(_group(), guard=(FAKE, 0, 16, 64)) == -1 and _sched(_group(), guard=(FAKE, 16, 16, -1)) == -1
    assert _sched(_group(), guard=(FAKE + 4, 16, 16, 64)) == -1
    assert b"guard" in L.gs_last_error()


def test_guarded_densify_stats_rejects_bad_arguments():
    L = N.lib()
    f = L.gs_densify_stats_guarded
    assert f(None, 0, None, None, None, None, None, None, 0, 0, 0, None) == 0
    assert f(None, -1, FAKE, FAKE, FAKE, FAKE, FAKE, None, 0, 0, 0, None) == -1
    for k in range(5):
        args = [FAKE] * 5
        args[k] = None
        assert f(None, 8, *args, None, 0, 0, 0, None) == -1, k
        args[k] = FAKE + 2
        assert f(None, 8, *args, None, 0, 0, 0, None) == -1, k
    assert f(None, 8, *[FAKE] * 5, FAKE, 0, 16, 64, None) == -1
    assert b"guard" in L.gs_last_error()


def test_bias_tables_match_torch_adams_python_formation():
    """torch.optim.Adam forms 1 - beta1 ** step and (1 - beta2 ** step) ** 0.5 in Python doubles (the latter is cast to
    float32 where it divides the float32 sqrt(exp_avg_sq)); the host table must agree bit for bit."""
    L = N.lib()
    for b1, b2 in ((0.9, 0.999), (0.8, 0.99), (0.0, 0.5)):
        n = L.gs_adam_bias_table_len(b1, b2)
        assert n > 3001 or (b1, b2) != (0.9, 0.999)
        bc1, bc2 = np.empty(n, np.float64), np.empty(n, np.float32)
        N.check(L.gs_adam_bias_table(b1, b2, n, bc1.ctypes.data, bc2.ctypes.data))
        for s in range(1, min(n, 3001)):
            assert bc1[s] == 1 - b1 ** float(s), (b1, s)
            assert bc2[s] == np.float32((1 - b2 ** float(s)) ** 0.5), (b2, s)
        # saturated: the entry every later step uses is exactly the correction of those steps
        assert bc1[n - 1] == 1.0 and bc2[n - 1] == np.float32(1.0) and (bc1[n - 2] != 1.0 or bc2[n - 2] != 1.0)
        for s in (n, n + 1, 10 * n):
            assert 1 - b1 ** float(s) == 1.0 and np.float32((1 - b2 ** float(s)) ** 0.5) == 1.0
    assert L.gs_adam_bias_table_len(1.0, 0.999) == 0 and L.gs_adam_bias_table_len(0.9, -0.1) == 0
    assert L.gs_adam_bias_table(0.9, 0.999, 1, None, None) == -1


def test_xyz_table_matches_the_reference_schedule_golden():
    for case in json.load(open(os.path.join(GOLDEN, "lr_golden.json"))):
        a = case["args"]

        def sched(step, a=a):
            return optim.expon_lr(step, a["lr_init"], a["lr_final"], a.get("lr_delay_steps", 0),
                                  a.get("lr_delay_mult", 1.0), a["max_steps"])
        table = train.lr_schedule(sched, max(case["steps"]))
        assert np.array(table, dtype=np.float64).tolist() == table          # doubles, as the device table holds them
        for step, want in zip(case["steps"], case["lr"]):
            if step >= 0:
                assert table[step] == want, (a, step)


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


def test_train_kernels_have_no_spills_no_float_atomics_and_one_double_division():
    log = os.path.join(CSRC, "gs_train.o.ptxas.log")
    if not os.path.exists(log):
        pytest.skip("gs_train.o.ptxas.log not built")
    text = open(log).read()
    assert text.count("Compiling entry function") == 4
    for m in re.finditer(r"(\d+) bytes spill stores, (\d+) bytes spill loads", text):
        assert m.group(1) == "0" and m.group(2) == "0", text
    per = _sass("gs_train.o")
    assert len(per) == 4
    fp64 = re.compile(r"^(DADD|DMUL|DFMA|DSETP|DMNMX|DSET)(\..*)?$|^MUFU\.(RCP|RSQ)64H$|^[FI]2[FI]\..*F64")
    for fn, ops in per.items():
        assert not [o for o in ops if o.startswith(("ATOM", "RED"))], fn          # no atomics at all
        used = {o.split(".")[0] if o[0] == "D" else o for o in ops if fp64.match(o)}
        if "k_adam_sched_prep" in fn:
            # lr / bias_correction1: reciprocal seed, Newton steps and their checks, and the final rounding to float
            assert {"MUFU.RCP64H", "F2F.F32.F64"} <= used <= {"DFMA", "DMUL", "DSETP", "MUFU.RCP64H", "F2F.F32.F64"}, used
        else:
            assert not used, (fn, used)


# the kernels of gs_blend.cu's retired shuffle-butterfly backward and alternative register builds: (object, kernel, NH, OCC)
RETIRED = [("gs_blend.o", "k_blend_fwd", 2, 12), ("gs_blend.o", "k_blend_bwd", 2, 13), ("gs_blend.o", "k_blend_bwd", 2, 10),
           ("gs_blend.o", "k_blend_bwd", 1, 7), ("gs_blend.o", "k_tile_partials", 2, 13), ("gs_blend.o", "k_tile_partials", 1, 7)]


def test_machine_code_of_every_surviving_kernel_is_unchanged():
    """Every kernel of every object compiles to the same instructions as in tests/golden/sass_kernels.json
    (tests/golden/make_sass_golden.py on the build before the retired kernels were removed); of the golden's kernels only
    the six retired ones are gone, and there are no new kernels."""
    if shutil.which("cuobjdump") is None:
        pytest.skip("cuobjdump not available")
    sys.path.insert(0, GOLDEN)
    try:
        import make_sass_golden as G
    finally:
        sys.path.remove(GOLDEN)
    gold = json.load(open(os.path.join(GOLDEN, "sass_kernels.json")))
    built = sorted(os.path.basename(o) for o in glob.glob(os.path.join(CSRC, "*.o")))
    if set(gold) - set(built):
        pytest.skip(f"{sorted(set(gold) - set(built))} not built")
    assert sorted(gold) == built, built                                                # no new objects
    gone = []
    for obj, want in gold.items():
        have = G.kernel_fingerprints(os.path.join(CSRC, obj))
        assert set(have) <= set(want), (obj, sorted(set(have) - set(want)))          # no new kernels
        for fn, h in have.items():
            assert h == want[fn], (obj, fn)                                           # the same instructions
        gone += [(obj, fn) for fn in want if fn not in have]
    retired = sorted((o, f"{k}ILi{nh}ELi{occ}E") for o, k, nh, occ in RETIRED)
    names = sorted((o, re.search(r"_cu_X\d+(k_\w+?ILi\d+ELi\d+E)", fn).group(1)) for o, fn in gone)
    assert names == retired, names


def test_library_reads_no_environment_switches():
    """Which device path runs depends on the inputs and the device alone: the library names no GS_* environment
    variable that could force one."""
    lib = os.path.join(CSRC, "libgsraster_b200.so")
    if not os.path.exists(lib):
        pytest.skip("libgsraster_b200.so not built")
    assert not re.findall(rb"GS_[A-Z][A-Z0-9_]+", open(lib, "rb").read())
