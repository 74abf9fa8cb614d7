"""ctypes declarations of include/gpr.h (the C ABI of libgpr.so).

This is the binding a Python host uses; INTEGRATION.md shows the equivalent Rust ``extern "C"``
block for the reference's own language.  Nothing here computes: it only describes the ABI.
"""
from __future__ import annotations

import ctypes as C
import os

GPR_OK = 0
GPR_E_INVALID, GPR_E_CUDA, GPR_E_NOMEM, GPR_E_CAPACITY = -1, -2, -3, -4
GPR_E_STATE, GPR_E_NCCL, GPR_E_UNSUPPORTED = -5, -6, -7
ERROR_NAMES = {
    -1: "GPR_E_INVALID", -2: "GPR_E_CUDA", -3: "GPR_E_NOMEM", -4: "GPR_E_CAPACITY",
    -5: "GPR_E_STATE", -6: "GPR_E_NCCL", -7: "GPR_E_UNSUPPORTED",
}
GPR_MEM_HOST, GPR_MEM_DEVICE = 0, 1
GPR_KERNEL_AUTO, GPR_KERNEL_LDG, GPR_KERNEL_TMA = 0, 1, 2
GPR_FMT_F32, GPR_FMT_U8B = 0, 1
GPR_F_POWER_PLANE = 0x1
GPR_F_BLOCK_INDEX = 0x2
GPR_GROUP_UTIL = 0x100
GPR_UNIQUE_ID_BYTES = 128
GPR_P2P_HANDLE_BYTES = 64


class gpr_config(C.Structure):
    _fields_ = [
        ("struct_size", C.c_uint32), ("device", C.c_int32),
        ("max_pods", C.c_uint32), ("max_gpus", C.c_uint32), ("max_samples", C.c_uint32),
        ("flags", C.c_uint32), ("kernel_variant", C.c_int32), ("reserved0", C.c_int32),
        ("stream", C.c_void_p),
    ]


class gpr_window(C.Structure):
    _fields_ = [
        ("struct_size", C.c_uint32), ("mem_kind", C.c_int32),
        ("util", C.c_void_p), ("power", C.c_void_p),
        ("eligible", C.c_void_p), ("created_ts", C.c_void_p),
        ("cutoff_ts", C.c_int64),
        ("n_pods", C.c_uint32), ("n_gpus", C.c_uint32), ("n_samples", C.c_uint32),
        ("util_format", C.c_uint32),
        ("row_stride", C.c_uint64), ("power_threshold", C.c_double),
        ("groups", C.c_void_p),
    ]


class gpr_result(C.Structure):
    _fields_ = [
        ("struct_size", C.c_uint32), ("out_mem_kind", C.c_int32),
        ("decision_bits", C.c_void_p), ("candidate_bits", C.c_void_p), ("series_max", C.c_void_p),
        ("veto_bits", C.c_void_p),
        ("n_series", C.c_uint64), ("n_candidates", C.c_uint64), ("n_decisions", C.c_uint64),
        ("kernel_ms", C.c_double),
        ("idle_slots", C.c_void_p),
    ]


class gpr_device_info(C.Structure):
    _fields_ = [
        ("struct_size", C.c_uint32), ("sm_count", C.c_int32),
        ("cc_major", C.c_int32), ("cc_minor", C.c_int32),
        ("l2_bytes", C.c_uint64), ("hbm_bytes", C.c_uint64), ("name", C.c_char * 64),
    ]


class gpr_text_span(C.Structure):
    _fields_ = [
        ("begin", C.c_uint64), ("end", C.c_uint64), ("row", C.c_uint32), ("flags", C.c_uint32),
        ("n_in", C.c_uint32), ("n_oow", C.c_uint32), ("n_tiny", C.c_uint32), ("reserved", C.c_uint32),
    ]


class gpr_text_grid(C.Structure):
    _fields_ = [
        ("struct_size", C.c_uint32), ("flags", C.c_uint32),
        ("t_end", C.c_int64), ("window_seconds", C.c_int64), ("step", C.c_int64),
        ("n_samples", C.c_uint32), ("n_rows", C.c_uint32), ("power_threshold", C.c_double),
    ]


class gpr_sample_batch(C.Structure):
    _fields_ = [
        ("struct_size", C.c_uint32), ("mem_kind", C.c_int32),
        ("offsets", C.c_void_p), ("rows", C.c_void_p), ("ts_ms", C.c_void_p), ("values", C.c_void_p),
        ("n_series", C.c_uint32), ("reserved", C.c_uint32),
    ]


class gpr_sample_stats(C.Structure):
    _fields_ = [("n_in", C.c_uint64), ("n_oow", C.c_uint64), ("n_tiny", C.c_uint64)]


class gpr_chunk_batch(C.Structure):
    _fields_ = [
        ("struct_size", C.c_uint32), ("mem_kind", C.c_int32),
        ("series_chunks", C.c_void_p), ("rows", C.c_void_p), ("chunk_bytes", C.c_void_p), ("data", C.c_void_p),
        ("n_series", C.c_uint32), ("reserved", C.c_uint32),
    ]


class gpr_chunk_export(C.Structure):
    _fields_ = [
        ("struct_size", C.c_uint32), ("mem_kind", C.c_int32),
        ("series_chunks", C.c_void_p), ("rows", C.c_void_p), ("chunk_bytes", C.c_void_p), ("data", C.c_void_p),
        ("cap_series", C.c_uint64), ("cap_chunks", C.c_uint64), ("cap_bytes", C.c_uint64),
        ("n_series", C.c_uint64), ("n_chunks", C.c_uint64), ("n_bytes", C.c_uint64), ("n_samples", C.c_uint64),
    ]


GPR_SPAN_SHARED, GPR_SPAN_HARD = 1, 2
GPR_TEXT_FILL, GPR_TEXT_RESIDENT = 1, 2
GPR_ROW_NONE = 0xFFFFFFFF

_P = C.c_void_p
# name -> (restype, argtypes); must list every symbol include/gpr.h declares
PROTOTYPES = {
    "gpr_version": (C.c_int, []),
    "gpr_create": (C.c_int, [C.POINTER(gpr_config), C.POINTER(_P)]),
    "gpr_destroy": (None, [_P]),
    "gpr_last_error": (C.c_char_p, [_P]),
    "gpr_decide": (C.c_int, [_P, C.POINTER(gpr_window), C.POINTER(gpr_result)]),
    "gpr_decide_async": (C.c_int, [_P, C.POINTER(gpr_window), C.POINTER(gpr_result)]),
    "gpr_sync": (C.c_int, [_P]),
    "gpr_decide_batch_async": (C.c_int, [_P, C.POINTER(gpr_window), C.POINTER(gpr_result), C.c_uint32]),
    "gpr_resident_init": (C.c_int, [_P, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32]),
    "gpr_append": (C.c_int, [_P, _P, _P, C.c_uint32, C.c_uint64, C.c_int32]),
    "gpr_resident_reindex": (C.c_int, [_P]),
    "gpr_resident_advance": (C.c_int, [_P, C.c_uint32]),
    "gpr_resident_head": (C.c_int, [_P, C.POINTER(C.c_uint32)]),
    "gpr_decide_resident": (C.c_int, [_P, C.POINTER(gpr_window), C.POINTER(gpr_result)]),
    "gpr_resident_planes": (C.c_int, [_P, C.POINTER(_P), C.POINTER(_P), C.POINTER(C.c_uint64)]),
    "gpr_resident_remap": (C.c_int, [_P, C.c_uint32, C.c_uint32, _P, C.c_int32]),
    "gpr_resident_live_rows": (C.c_int, [_P, _P, C.c_int32]),
    "gpr_resident_cols": (C.c_int, [_P, C.c_int32, C.c_uint32, C.c_uint32, _P, C.c_int32]),
    "gpr_resident_retime": (C.c_int, [_P, C.c_uint32, C.c_uint32]),
    "gpr_comm_unique_id": (C.c_int, [_P]),
    "gpr_comm_init": (C.c_int, [_P, _P, C.c_int, C.c_int]),
    "gpr_comm_destroy": (C.c_int, [_P]),
    "gpr_p2p_init": (C.c_int, [_P, C.c_int, C.c_int, C.c_uint32, _P]),
    "gpr_p2p_attach": (C.c_int, [_P, _P]),
    "gpr_host_alloc": (C.c_int, [_P, C.c_size_t, C.POINTER(_P)]),
    "gpr_host_free": (C.c_int, [_P, _P]),
    "gpr_device_alloc": (C.c_int, [_P, C.c_size_t, C.POINTER(_P)]),
    "gpr_device_free": (C.c_int, [_P, _P]),
    "gpr_memcpy": (C.c_int, [_P, _P, _P, C.c_size_t, C.c_int32, C.c_int32]),
    "gpr_timer_begin": (C.c_int, [_P]),
    "gpr_timer_end": (C.c_int, [_P, C.POINTER(C.c_double)]),
    "gpr_step_stamps": (C.c_int, [_P, _P, C.c_uint32, C.POINTER(C.c_uint32), C.POINTER(C.c_uint64)]),
    "gpr_p2p_debug": (C.c_int, [_P, C.c_int32]),
    "gpr_phase_stamps": (C.c_int, [_P, _P, C.c_uint32, C.POINTER(C.c_uint32)]),
    "gpr_flush_l2": (C.c_int, [_P]),
    "gpr_launch_count": (C.c_int, [_P, C.POINTER(C.c_uint64)]),
    "gpr_get_device_info": (C.c_int, [_P, C.POINTER(gpr_device_info)]),
    "gpr_text_scan": (C.c_int, [_P, C.c_int32, _P, C.c_uint64, C.c_int32, _P, _P, C.c_uint64,
                                C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]),
    "gpr_text_scan_begin": (C.c_int, [_P, C.c_int32, _P, C.c_uint64, C.c_int32]),
    "gpr_text_scan_next": (C.c_int, [_P, _P, _P, C.c_uint64, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64),
                                     C.POINTER(C.c_uint64), C.POINTER(C.c_int32)]),
    "gpr_text_parse": (C.c_int, [_P, C.c_int32, _P, C.c_uint32, C.POINTER(gpr_text_grid), C.c_int32]),
    "gpr_text_planes": (C.c_int, [_P, C.POINTER(_P), C.POINTER(_P)]),
    "gpr_samples_scatter": (C.c_int, [_P, C.POINTER(gpr_sample_batch), C.POINTER(gpr_text_grid), C.c_int32,
                                      C.POINTER(gpr_sample_stats)]),
    "gpr_chunks_scatter": (C.c_int, [_P, C.POINTER(gpr_chunk_batch), C.POINTER(gpr_text_grid), C.c_int32,
                                     C.POINTER(gpr_sample_stats)]),
    "gpr_resident_export": (C.c_int, [_P, C.POINTER(gpr_text_grid), C.c_int32, C.c_uint32,
                                      C.POINTER(gpr_chunk_export)]),
    "gpr_synth_fill": (C.c_int, [_P, C.c_uint64, C.c_int32, _P, C.c_uint64, C.c_uint32,
                                 C.c_uint32, C.c_uint32, C.c_uint64]),
    "gpr_synth_eligible": (C.c_int, [_P, C.c_uint64, _P, C.c_uint64, C.c_uint32]),
}


def lib_path() -> str:
    return os.path.join(os.path.dirname(os.path.abspath(__file__)), "libgpr.so")


_lib = None


def load() -> C.CDLL:
    """Load libgpr.so (built in-tree by ``__graft_entry__.build()``).  Fails loudly if absent:
    there is no Python or CPU substitute for the CUDA library."""
    global _lib
    if _lib is not None:
        return _lib
    path = lib_path()
    if not os.path.exists(path):
        raise RuntimeError(
            f"{path} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(nvcc, sm_90a).  The idle-decision engine has no CPU fallback.")
    lib = C.CDLL(path)
    for name, (restype, argtypes) in PROTOTYPES.items():
        fn = getattr(lib, name)  # AttributeError here = header/library drift
        fn.restype = restype
        fn.argtypes = argtypes
    _lib = lib
    return lib
