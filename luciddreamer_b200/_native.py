"""ctypes binding of the C ABI in include/gsraster.h (luciddreamer_b200/csrc/libgsraster_b200.so).

There is NO fallback: if the CUDA library is missing or does not load, importing the product path raises.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

_HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(_HERE, "csrc")
LIB_PATH = os.path.join(CSRC, "libgsraster_b200.so")

GS_OK = 0
GS_ENOTREADY = -5
GS_STATUS_SLOTS = 64
GS_GRAPH_STATUS_SLOTS = 256
GS_GRAPH_TICKET = 1 << 30


class GsFrame(C.Structure):
    _fields_ = [("P", C.c_int32), ("D", C.c_int32), ("M", C.c_int32), ("W", C.c_int32), ("H", C.c_int32),
                ("tan_fovx", C.c_float), ("tan_fovy", C.c_float), ("scale_modifier", C.c_float),
                ("prefiltered", C.c_int32), ("debug", C.c_int32),
                ("bg", C.c_void_p), ("means3D", C.c_void_p), ("shs", C.c_void_p), ("colors_precomp", C.c_void_p),
                ("opacities", C.c_void_p), ("scales", C.c_void_p), ("rotations", C.c_void_p),
                ("cov3D_precomp", C.c_void_p), ("viewmatrix", C.c_void_p), ("projmatrix", C.c_void_p),
                ("campos", C.c_void_p)]


class GsGrads(C.Structure):
    _fields_ = [("dL_dmeans3D", C.c_void_p), ("dL_dmeans2D", C.c_void_p), ("dL_dsh", C.c_void_p),
                ("dL_dcolors", C.c_void_p), ("dL_dopacity", C.c_void_p), ("dL_dscales", C.c_void_p),
                ("dL_drotations", C.c_void_p), ("dL_dcov3D", C.c_void_p),
                ("peer_world", C.c_int32), ("peer_pad", C.c_int32), ("peer_buckets", C.POINTER(C.c_void_p)),
                ("peer_multicast", C.c_void_p), ("peer_seg_off", C.POINTER(C.c_int64)),
                ("peer_signals", C.POINTER(C.c_void_p)), ("peer_rank", C.c_int32), ("peer_epoch_begin", C.c_uint32),
                ("peer_epoch_end", C.c_uint32), ("peer_pad2", C.c_int32)]


class GsAdamGroup(C.Structure):
    _fields_ = [("param", C.c_void_p), ("grad", C.c_void_p), ("exp_avg", C.c_void_p), ("exp_avg_sq", C.c_void_p),
                ("rows", C.c_int64), ("row_width", C.c_int32), ("grad_row_width", C.c_int32),
                ("grad_offset", C.c_int32), ("activation", C.c_int32), ("lr", C.c_double)]


class GsAdamSchedGroup(C.Structure):
    _fields_ = [("param", C.c_void_p), ("grad", C.c_void_p), ("exp_avg", C.c_void_p), ("exp_avg_sq", C.c_void_p),
                ("rows", C.c_int64), ("row_width", C.c_int32), ("grad_row_width", C.c_int32),
                ("grad_offset", C.c_int32), ("activation", C.c_int32), ("lr", C.c_double), ("lr_table", C.c_void_p),
                ("step", C.c_void_p)]


class GsCounts(C.Structure):
    _fields_ = [("num_rendered", C.c_int64), ("num_pairs", C.c_int64), ("num_visible", C.c_int64)]


class GsViewScratch(C.Structure):
    _fields_ = [("geom_buffer", C.c_void_p), ("image_buffer", C.c_void_p), ("binning_buffer", C.c_void_p),
                ("pair_capacity", C.c_int64), ("radii", C.c_void_p)]


class GsViewResult(C.Structure):
    _fields_ = [("out_color", C.c_void_p), ("out_depth", C.c_void_p), ("radii", C.c_void_p), ("counts", GsCounts),
                ("status", C.c_int32), ("pad", C.c_int32)]


# every symbol include/gsraster.h declares: (name, restype, argtypes)
SYMBOLS = [
    ("gs_abi_version", C.c_int, []),
    ("gs_last_error", C.c_char_p, []),
    ("gs_context_create", C.c_int, [C.c_int, C.POINTER(C.c_void_p)]),
    ("gs_context_destroy", None, [C.c_void_p]),
    ("gs_geom_bytes", C.c_size_t, [C.c_int32]),
    ("gs_image_bytes", C.c_size_t, [C.c_int32, C.c_int32]),
    ("gs_binning_bytes", C.c_size_t, [C.c_int64]),
    ("gs_forward_preprocess", C.c_int, [C.c_void_p, C.POINTER(GsFrame), C.c_void_p, C.c_void_p, C.c_void_p,
                                        C.c_void_p, C.POINTER(C.c_int32)]),
    ("gs_forward_counts", C.c_int, [C.c_void_p, C.c_int32, C.POINTER(GsCounts)]),
    ("gs_forward_counts_peek", C.c_int, [C.c_void_p, C.c_int32, C.POINTER(GsCounts)]),
    ("gs_forward_release_graph_slot", C.c_int, [C.c_void_p, C.c_int32]),
    ("gs_forward_render", C.c_int, [C.c_void_p, C.POINTER(GsFrame), C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64,
                                    C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p]),
    ("gs_forward_views", C.c_int, [C.c_void_p, C.POINTER(GsFrame), C.c_int32, C.POINTER(GsViewScratch), C.c_int32,
                                   C.POINTER(GsViewResult), C.c_void_p]),
    ("gs_backward_scratch_bytes", C.c_size_t, [C.c_int64]),
    ("gs_backward", C.c_int, [C.c_void_p, C.POINTER(GsFrame), C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64,
                              C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.POINTER(GsGrads),
                              C.c_void_p]),
    ("gs_backward_deterministic_scratch_bytes", C.c_size_t, [C.c_int64, C.c_int64]),
    ("gs_backward_deterministic", C.c_int, [C.c_void_p, C.POINTER(GsFrame), C.c_void_p, C.c_void_p, C.c_void_p,
                                            C.c_int64, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p,
                                            C.POINTER(GsGrads), C.c_void_p]),
    ("gs_mark_visible", C.c_int, [C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    ("gs_l1_loss_backward", C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_float, C.c_void_p,
                                      C.c_void_p, C.c_void_p]),
    ("gs_pack_frame", C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                C.c_void_p]),
    ("gs_minmax_read", C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    ("gs_colorize_scratch_bytes", C.c_size_t, [C.c_int32]),
    ("gs_colorize_depth", C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_float, C.c_void_p,
                                    C.c_uint32, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p]),
    ("gs_knn_scratch_bytes", C.c_size_t, [C.c_int32]),
    ("gs_knn_mean_dist2", C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    ("gs_densify_stats", C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                   C.c_void_p]),
    ("gs_gaussian_adam_step", C.c_int, [C.c_void_p, C.POINTER(GsAdamGroup), C.c_int32, C.c_double, C.c_double, C.c_double,
                                        C.c_int32, C.c_void_p]),
    ("gs_activate", C.c_int, [C.c_void_p, C.c_int32, C.c_int32] + [C.c_void_p] * 10),
    ("gs_adam_sched_scratch_bytes", C.c_size_t, []),
    ("gs_adam_bias_table_len", C.c_int32, [C.c_double, C.c_double]),
    ("gs_adam_bias_table", C.c_int, [C.c_double, C.c_double, C.c_int32, C.c_void_p, C.c_void_p]),
    ("gs_gaussian_adam_sched_step", C.c_int, [C.c_void_p, C.POINTER(GsAdamSchedGroup), C.c_int32, C.c_double, C.c_double,
                                              C.c_double, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_int32,
                                              C.c_void_p, C.c_int32, C.c_int32, C.c_int64, C.c_void_p, C.c_size_t,
                                              C.c_void_p]),
    ("gs_densify_stats_guarded", C.c_int, [C.c_void_p, C.c_int32] + [C.c_void_p] * 6 + [C.c_int32, C.c_int32, C.c_int64,
                                                                                          C.c_void_p]),
    ("gs_photometric_scratch_bytes", C.c_size_t, [C.c_int32, C.c_int32]),
    ("gs_photometric_loss_backward", C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_float,
                                               C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    ("gs_debug_export_binning", C.c_int, [C.POINTER(GsFrame), C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p,
                                          C.c_void_p, C.c_int64, C.c_void_p]),
    ("gs_debug_blend_rows_per_warp", C.c_int, [C.c_void_p, C.c_int32, C.c_int32]),
    ("gs_profile_enable", C.c_int, [C.c_void_p, C.c_int]),
    ("gs_profile_num_kernels", C.c_int, []),
    ("gs_profile_kernel_name", C.c_char_p, [C.c_int]),
    ("gs_profile_read", C.c_int, [C.c_void_p, C.POINTER(C.c_float)]),
]

_lib = None


def build(force: bool = False, verbose: bool = False) -> str:
    """nvcc -gencode arch=compute_90a,code=sm_90a (see csrc/Makefile); cross-compiles without a GPU."""
    if force:
        subprocess.check_call(["make", "-C", CSRC, "clean"], stdout=None if verbose else subprocess.DEVNULL)
    subprocess.check_call(["make", "-C", CSRC, "-j8"], stdout=None if verbose else subprocess.DEVNULL)
    return LIB_PATH


def lib():
    """Load the CUDA library; raises (never falls back) if it is absent."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                f"{LIB_PATH} is missing: the H100 rasterizer has no CPU fallback. "
                "Build it with `python -c 'import __graft_entry__ as g; g.build()'` (needs nvcc).")
        L = C.CDLL(LIB_PATH)
        for name, res, args in SYMBOLS:
            fn = getattr(L, name)           # AttributeError if the header and the library disagree
            fn.restype = res
            fn.argtypes = args
        _lib = L
    return _lib


def last_error() -> str:
    return lib().gs_last_error().decode("utf-8", "replace")


def check(rc: int) -> None:
    if rc != GS_OK:
        raise RuntimeError(f"gsraster error {rc}: {last_error()}")
