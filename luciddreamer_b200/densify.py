"""Densify and prune the reference's GaussianModel on the device (include/gsdensify.h).

    densify.attach(gm)                 # gm.densify_and_prune and gm.reset_opacity become the two functions below
    gm.densify_and_prune(max_grad, min_opacity, extent, max_screen_size)
    gm.reset_opacity()

`densify_and_prune(gm, ...)` and `reset_opacity(gm)` take the arguments of the reference's methods
(scene/gaussian_model.py) and leave the state they leave, bit for bit, the random draw of the split samples included:
new `nn.Parameter` objects in gm and in gm.optimizer.param_groups, the optimiser state re-keyed to them (the same
state dicts, `step` untouched), groups without state still without state, and new statistic tensors. They work with
torch.optim.Adam and with optim.FusedAdam alike. Every Parameter is replaced, so a train.TrainStep re-captures on its
next run(), as it does after the reference's methods.

A densify is three launches on the device, one read of four counts by the host, the reference's own
`torch.normal(mean=zeros, std=stds)` for the split samples (so torch's generator advances exactly as it does there),
and one gather that writes every output tensor once. The output rows are in the reference's order: surviving
originals, clones, split copy 1 and split copy 2 of each selected row, pruned rows left out.

Unlike the reference, densify_and_prune does not call torch.cuda.empty_cache(): the caching allocator keeps its
pool, which the next graph capture allocates from. Allocator state is the one thing it does not reproduce.
"""
from __future__ import annotations

import ctypes as C
import os
import types

import torch
from torch import nn

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "densify_csrc", "libgsdensify.so")

GSDENSIFY_OK = 0
PARAM, XYZ, SCALING, MOMENT = 0, 1, 2, 3
MAX_TENSORS = 32
_P = C.c_void_p
_F = C.c_float


class Tensor(C.Structure):
    """gsdensify_tensor"""
    _fields_ = [("src", _P), ("dst", _P), ("width", C.c_int32), ("kind", C.c_int32)]


SYMBOLS = [
    ("gsdensify_abi_version", C.c_int, []),
    ("gsdensify_scratch_bytes", C.c_int, [C.c_int32, C.POINTER(C.c_uint64)]),
    ("gsdensify_plan", C.c_int, [C.c_int32, _P, _P, _P, _P, _F, _F, _F, C.c_int32, _F, _F, _P, _P, C.c_uint64, _P]),
    ("gsdensify_map", C.c_int, [C.c_int32, _P, C.c_int32, C.c_int32, _P, _P, _P, C.c_uint64, _P]),
    ("gsdensify_apply", C.c_int, [_P, C.c_int32, C.POINTER(Tensor), C.c_int32, _P, _P, C.c_int32, _P]),
    ("gsdensify_reset_opacity", C.c_int, [C.c_int32, _P, _P, _P, _P, _P]),
]

# GaussianModel's attribute of each parameter group (training_setup's names)
ATTRS = {"xyz": "_xyz", "f_dc": "_features_dc", "f_rest": "_features_rest", "opacity": "_opacity",
         "scaling": "_scaling", "rotation": "_rotation"}

_lib = None


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(f"{LIB_PATH} is not built; run __graft_entry__.build()")
        L = C.CDLL(LIB_PATH)
        for name, res, args in SYMBOLS:
            f = getattr(L, name)
            f.restype, f.argtypes = res, args
        _lib = L
    return _lib


def _check(rc: int, what: str) -> None:
    if rc != GSDENSIFY_OK:
        raise RuntimeError(f"{what} failed with code {rc}")


def _stream(dev) -> C.c_void_p:
    return C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)


def _f32(x) -> float:
    """A Python scalar as torch compares a float32 tensor with it: cast to float32."""
    return float(torch.tensor(float(x), dtype=torch.float32))


def _input(t: torch.Tensor, name: str, rows: int, dev) -> torch.Tensor:
    if not (t.is_cuda and t.dtype == torch.float32 and t.device == dev and t.shape[0] == rows):
        raise RuntimeError(f"densify: {name} must be a float32 CUDA tensor of {rows} rows on {dev}, "
                           f"got {tuple(t.shape)} {t.dtype} on {t.device}")
    return t.detach().contiguous()


def _replace(gm, tensors: dict, moments: dict) -> None:
    """Puts each new tensor in its group as a new Parameter and re-keys the group's state dict to it, as the
    reference's _prune_optimizer / cat_tensors_to_optimizer / replace_tensor_to_optimizer do."""
    opt = gm.optimizer
    for group in opt.param_groups:
        name = group["name"]
        if name not in tensors:
            continue
        old = group["params"][0]
        stored = opt.state.get(old, None)
        if stored is not None:
            stored["exp_avg"], stored["exp_avg_sq"] = moments[name]
            del opt.state[old]
        group["params"][0] = nn.Parameter(tensors[name].requires_grad_(True))
        if stored is not None:
            opt.state[group["params"][0]] = stored
        setattr(gm, ATTRS[name], group["params"][0])


@torch.no_grad()
def densify_and_prune(gm, max_grad, min_opacity, extent, max_screen_size) -> dict:
    """GaussianModel.densify_and_prune on the device; see the module docstring. Returns the counts
    {"clones", "splits", "survivors" (originals kept), "P" (rows after)}."""
    opt = gm.optimizer
    dev = gm._xyz.device
    P = gm._xyz.shape[0]
    L = lib()
    with torch.cuda.device(dev):
        s = _stream(dev)
        accum = _input(gm.xyz_gradient_accum, "xyz_gradient_accum", P, dev)
        denom = _input(gm.denom, "denom", P, dev)
        scaling = _input(gm._scaling, "_scaling", P, dev)
        opacity = _input(gm._opacity, "_opacity", P, dev)
        b = C.c_uint64()
        _check(L.gsdensify_scratch_bytes(P, C.byref(b)), "gsdensify_scratch_bytes")
        scratch = torch.empty(b.value, dtype=torch.uint8, device=dev)
        counts = torch.empty(4, dtype=torch.int32, device=dev)
        screen = bool(max_screen_size)
        _check(L.gsdensify_plan(P, accum.data_ptr(), denom.data_ptr(), scaling.data_ptr(), opacity.data_ptr(),
                                _f32(max_grad), _f32(gm.percent_dense * extent), _f32(min_opacity), int(screen),
                                _f32(max_screen_size) if screen else 0.0, _f32(0.1 * extent), counts.data_ptr(),
                                scratch.data_ptr(), scratch.numel(), s), "gsdensify_plan")
        n_clone, S, n_orig, P_new = counts.tolist()

        mapping = torch.empty((P_new, 2), dtype=torch.int32, device=dev)
        stds = torch.empty((2 * S, 3), dtype=torch.float32, device=dev)
        _check(L.gsdensify_map(P, scaling.data_ptr(), S, P_new, mapping.data_ptr(), stds.data_ptr(),
                               scratch.data_ptr(), scratch.numel(), s), "gsdensify_map")
        # densify_and_split's own draw: torch's generator advances exactly as in the reference
        samples = torch.normal(mean=torch.zeros((stds.size(0), 3), device=dev), std=stds)

        descs, news, moments = [], {}, {}

        def gather(src, kind):
            src = src.detach()
            if not src.is_contiguous():
                raise RuntimeError("densify: parameters and moments must be contiguous")
            dst = torch.empty((P_new,) + tuple(src.shape[1:]), dtype=src.dtype, device=dev)
            width = src.numel() // P if P > 0 else 0
            if width > 0:
                descs.append(Tensor(src.data_ptr(), dst.data_ptr(), width, kind))
            return dst

        for group in opt.param_groups:
            if len(group["params"]) != 1:
                raise RuntimeError("densify: every parameter group holds one Parameter")
            name = group["name"]
            p = group["params"][0]
            _input(p, name, P, dev)
            news[name] = gather(p, {"xyz": XYZ, "scaling": SCALING}.get(name, PARAM))
            st = opt.state.get(p, None)
            if st is not None:
                moments[name] = (gather(st["exp_avg"], MOMENT), gather(st["exp_avg_sq"], MOMENT))
        if len(descs) > MAX_TENSORS:
            raise RuntimeError(f"densify: {len(descs)} tensors, at most {MAX_TENSORS}")
        rotation = _input(gm._rotation, "_rotation", P, dev)
        arr = (Tensor * max(len(descs), 1))(*descs)
        _check(L.gsdensify_apply(mapping.data_ptr(), P_new, arr, len(descs), rotation.data_ptr(), samples.data_ptr(),
                                 S, s), "gsdensify_apply")
        stats = [torch.zeros((P_new, 1), device=dev), torch.zeros((P_new, 1), device=dev),
                 torch.zeros((P_new), device=dev)]
        if P + n_clone + S == 1:
            # the reference's final prune mask is `(...).squeeze()` of a single row: a 0-d mask, and indexing with it
            # puts a leading dimension of 1 or 0 rows in front of every tensor the prune touches
            news = {k: v.reshape((P_new, 1) + v.shape[1:]) for k, v in news.items()}
            moments = {k: tuple(m.reshape((P_new, 1) + m.shape[1:]) for m in v) for k, v in moments.items()}
            stats = [t.reshape((P_new, 1) + t.shape[1:]) for t in stats]
        _replace(gm, news, moments)
        gm.xyz_gradient_accum, gm.denom, gm.max_radii2D = stats
    return {"clones": n_clone, "splits": S, "survivors": n_orig, "P": P_new}


@torch.no_grad()
def reset_opacity(gm) -> None:
    """GaussianModel.reset_opacity on the device: opacity = inverse_sigmoid(min(sigmoid(opacity), 0.01)) as a new
    Parameter, the opacity group's moments new zero tensors and its step kept."""
    opt = gm.optimizer
    dev = gm._opacity.device
    P = gm._opacity.shape[0]
    group = next(g for g in opt.param_groups if g["name"] == "opacity")
    stored = opt.state.get(group["params"][0], None)
    if stored is None:             # the reference's replace_tensor_to_optimizer needs the group's state
        raise RuntimeError("reset_opacity: the opacity group has no optimiser state yet")
    with torch.cuda.device(dev):
        src = _input(gm._opacity, "_opacity", P, dev)
        out = torch.empty_like(src)
        m1, m2 = torch.empty_like(src), torch.empty_like(src)
        _check(lib().gsdensify_reset_opacity(P, src.data_ptr(), out.data_ptr(), m1.data_ptr(), m2.data_ptr(),
                                             _stream(dev)), "gsdensify_reset_opacity")
    _replace(gm, {"opacity": out}, {"opacity": (m1, m2)})


def attach(gm):
    """Binds densify_and_prune and reset_opacity to gm in place of the reference's methods; returns gm."""
    gm.densify_and_prune = types.MethodType(densify_and_prune, gm)
    gm.reset_opacity = types.MethodType(reset_opacity, gm)
    return gm
