"""Densification library (luciddreamer_b200.densify, include/gsdensify.h) without a GPU: it compiles for sm_90a,
exports the header's symbols, refuses bad arguments before reaching a device, and keeps every product and sum of the
restated torch expressions rounded on its own."""
import ctypes as C
import os
import re
import subprocess

import pytest
import torch

from luciddreamer_b200 import densify

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "luciddreamer_b200", "densify_csrc")
KERNELS = ("k_plan", "k_scan", "k_map", "k_apply", "k_reset_opacity")


@pytest.fixture(scope="module", autouse=True)
def built():
    subprocess.check_call(["make", "-C", CSRC, "-j4"], stdout=subprocess.DEVNULL)


def test_header_and_ctypes_symbol_tables_agree():
    header = open(os.path.join(ROOT, "include", "gsdensify.h")).read()
    declared = re.findall(r"^int (gsdensify_\w+)\(", header, re.M)
    assert declared == [s[0] for s in densify.SYMBOLS]
    exported = subprocess.run(["nm", "-D", "--defined-only", densify.LIB_PATH], capture_output=True, text=True,
                              check=True).stdout
    assert sorted(re.findall(r" T (gsdensify_\w+)", exported)) == sorted(declared)
    for name, _, args in densify.SYMBOLS:
        decl = re.search(rf"int {name}\(([^)]*)\)", header).group(1)
        n = 0 if decl.strip() == "void" else decl.count(",") + 1
        assert n == len(args), name
    assert C.sizeof(densify.Tensor) == 24
    for k, v in dict(PARAM=0, XYZ=1, SCALING=2, MOMENT=3, MAX_TENSORS=32).items():
        assert re.search(rf"#define GSDENSIFY_{k} {v}\b", header), k
        assert getattr(densify, k) == v


def test_machine_code_is_sm_90a_without_spills():
    log = open(os.path.join(CSRC, "gs_densify.o.ptxas.log")).read()
    spills = re.findall(r"(\d+) bytes spill stores, (\d+) bytes spill loads", log)
    assert len(spills) == len(KERNELS) and all(s == ("0", "0") for s in spills)
    obj = os.path.join(CSRC, "gs_densify.o")
    sass = subprocess.run(["cuobjdump", "-sass", obj], capture_output=True, text=True, check=True).stdout
    for k in KERNELS:
        assert k in sass
    assert "sm_90a" in subprocess.run(["cuobjdump", "-lelf", obj], capture_output=True, text=True, check=True).stdout
    assert not re.search(r"\b(RED|ATOM|ATOMS)\.", sass)          # offsets come from scans: no atomics at all


def test_no_product_or_sum_is_left_for_the_assembler_to_contract(tmp_path):
    """Built with --fmad=false, every float32 mul / add / sub in the PTX carries an explicit rounding mode (.rn),
    which ptxas never fuses into an FFMA. The fused multiply-adds that remain are written out (the split rows' bmm)
    or belong to expf, logf and the IEEE division and square root."""
    ptx = tmp_path / "gs_densify.ptx"
    subprocess.check_call(["make", "-s", "-C", CSRC, "ptx", f"PTX_OUT={ptx}"], stdout=subprocess.DEVNULL)
    text = ptx.read_text()
    assert re.search(r"\bmul\.rn\.f32", text) and re.search(r"\badd\.rn\.f32", text)
    assert not re.findall(r"\b(mul|add|sub)\.f32\b", text)
    assert not re.findall(r"\b(mul|add|sub)(\.ftz)?\.approx", text)
    assert not re.search(r"\bdiv\.(approx|full)\.f32", text)       # IEEE division only


def test_argument_errors_and_scratch():
    L = densify.lib()
    assert L.gsdensify_abi_version() == 1
    b = C.c_uint64()
    sizes = []
    for P in (0, 1, 255, 256, 2_000_000):
        assert L.gsdensify_scratch_bytes(P, C.byref(b)) == 0
        assert b.value % 256 == 0
        sizes.append(b.value)
    assert sizes == sorted(sizes) and sizes[-1] >= 2_000_000 * (1 + 8 / 256 + 16 / 256)
    for P in (-1, 1 << 30):
        assert L.gsdensify_scratch_bytes(P, C.byref(b)) == -22
    assert L.gsdensify_scratch_bytes(8, None) == -22
    assert L.gsdensify_scratch_bytes(1000, C.byref(b)) == 0
    need = b.value
    A = 1 << 20                                               # fake, well-aligned device addresses: never dereferenced
    f = 0.5

    def plan(P=1000, ptr=A, screen=0, counts=A, scratch=A, nbytes=need):
        return L.gsdensify_plan(P, ptr, ptr, ptr, ptr, f, f, f, screen, f, f, counts, scratch, nbytes, None)
    for kw in (dict(P=-1), dict(ptr=None), dict(screen=2), dict(counts=None), dict(counts=A + 2), dict(scratch=None),
               dict(scratch=A + 128), dict(nbytes=need - 1)):
        assert plan(**kw) == -22, kw

    def mapping(P=1000, S=10, P_new=1000, m=A, stds=A, scratch=A, nbytes=need):
        return L.gsdensify_map(P, A, S, P_new, m, stds, scratch, nbytes, None)
    for kw in (dict(S=-1), dict(S=1001), dict(P_new=3001), dict(P_new=-1), dict(m=None), dict(m=A + 4),
               dict(stds=None), dict(scratch=A + 8), dict(nbytes=0)):
        assert mapping(**kw) == -22, kw

    def apply(descs, P_new=1000, m=A, rot=A, samples=A, S=4):
        arr = (densify.Tensor * max(len(descs), 1))(*descs)
        return L.gsdensify_apply(m, P_new, arr, len(descs), rot, samples, S, None)
    T = densify.Tensor
    for descs, kw in (([T(A, A, 0, 0)], {}), ([T(A, A, 3, 4)], {}), ([T(A, A, 4, densify.XYZ)], {}),
                      ([T(A, A, 2, densify.SCALING)], {}), ([T(None, A, 3, 0)], {}), ([T(A, A + 1, 3, 0)], {}),
                      ([T(A, A, 3, densify.XYZ)], dict(rot=None)), ([T(A, A, 3, densify.XYZ)], dict(samples=None)),
                      ([T(A, A, 3, 0)], dict(m=None)), ([T(A, A, 3, 0)], dict(P_new=-1)),
                      ([T(A, A, 3, 0)] * 33, {}), ([T(A, A, 3000, 0)], dict(P_new=1 << 20))):
        assert apply(descs, **kw) == -22, (descs[0].width, descs[0].kind, kw)
    assert apply([T(A, A, 3, 0)], P_new=0) == 0              # nothing to enqueue
    assert apply([]) == 0
    assert L.gsdensify_reset_opacity(-1, A, A, A, A, None) == -22
    assert L.gsdensify_reset_opacity(8, None, A, A, A, None) == -22
    assert L.gsdensify_reset_opacity(8, A, A + 2, A, A, None) == -22
    assert L.gsdensify_reset_opacity(0, None, None, None, None, None) == 0


def test_python_scalars_become_float32_as_torch_casts_them():
    """The thresholds torch compares a float32 tensor with are the Python scalars rounded to float32."""
    for x in (0.0002, 0.005, 0.01 * 3.7, 0.1 * 2.9, 1e-40, 20, -1):
        v = densify._f32(x)
        assert v == float(torch.tensor(x, dtype=torch.float32))
        t = torch.tensor([v], dtype=torch.float32)
        assert bool(t >= x) and not bool(t < x)              # torch's own comparison agrees with the cast
