"""ctypes loader for the C oracle (``libgpr_oracle.so``).  TEST INFRASTRUCTURE ONLY — see
``gpr_oracle.h``: parity unpinned; only tests/, smoke() and bench.py's CPU-baseline legs may
import this module."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_DIR = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_DIR, "libgpr_oracle.so")
_lib = None

_P = C.c_void_p


def build(force: bool = False) -> str:
    src = os.path.join(_DIR, "gpr_oracle.c")
    if force or not os.path.exists(_SO) or os.path.getmtime(_SO) < os.path.getmtime(src):
        subprocess.check_call(["make", "-C", _DIR, "-s"] + (["-B"] if force else []))
    return _SO


def load() -> C.CDLL:
    global _lib
    if _lib is None:
        build()
        lib = C.CDLL(_SO)
        lib.gpo_max_over_time.restype = C.c_double
        lib.gpo_max_over_time.argtypes = [_P, C.c_uint32]
        dec_args = [_P, _P, _P, _P, C.c_int64, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint64,
                    C.c_double, _P, _P, _P, _P]
        lib.gpo_decide.restype = C.c_int
        lib.gpo_decide.argtypes = dec_args
        lib.gpo_decide_mt.restype = C.c_int
        lib.gpo_decide_mt.argtypes = [C.c_int] + dec_args
        lib.gpo_synth_cell.restype = C.c_float
        lib.gpo_synth_cell.argtypes = [C.c_uint64, C.c_int, C.c_uint64, C.c_uint32, C.c_uint32]
        lib.gpo_synth_eligible_pod.restype = C.c_uint8
        lib.gpo_synth_eligible_pod.argtypes = [C.c_uint64, C.c_uint64]
        lib.gpo_synth_fill.restype = C.c_int
        lib.gpo_synth_fill.argtypes = [C.c_int, C.c_uint64, C.c_int, _P, C.c_uint64, C.c_uint32,
                                       C.c_uint32, C.c_uint32, C.c_uint64]
        lib.gpo_synth_eligible.restype = C.c_int
        lib.gpo_synth_eligible.argtypes = [C.c_uint64, _P, C.c_uint64, C.c_uint32]
        lib.gpo_decide_synth.restype = C.c_int
        lib.gpo_decide_synth.argtypes = [C.c_int, C.c_uint64, C.c_uint64, C.c_uint32, C.c_uint32,
                                         C.c_uint32, C.c_int, C.c_double, C.c_int, _P, _P, _P]
        lib.gpo_decide_synth_ex.restype = C.c_int
        lib.gpo_decide_synth_ex.argtypes = [C.c_int, C.c_uint64, C.c_uint64, C.c_uint32, C.c_uint32,
                                            C.c_uint32, C.c_int, C.c_double, C.c_int, _P, _P, _P, _P, _P]
        lib.gpo_hardware_threads.restype = C.c_int
        lib.gpo_pool_pin.restype = None
        lib.gpo_pool_pin.argtypes = [C.c_int]
        _lib = lib
    return _lib


def _p(a):
    return None if a is None else a.ctypes.data


def max_over_time(row) -> float:
    row = np.ascontiguousarray(row, dtype=np.float32)
    return float(load().gpo_max_over_time(_p(row), row.size))


def decide(util, power=None, eligible=None, created_ts=None, cutoff_ts=0, power_threshold=0.0,
           n_threads: int = 1, want_series_max: bool = True):
    util = np.ascontiguousarray(util, dtype=np.float32)
    P, G, T = util.shape
    if power is not None:
        power = np.ascontiguousarray(power, dtype=np.float32)
    if eligible is not None:
        eligible = np.ascontiguousarray(eligible, dtype=np.uint8)
    if created_ts is not None:
        created_ts = np.ascontiguousarray(created_ts, dtype=np.int64)
    W = max((P + 31) // 32, 1)
    dbits = np.zeros(W, dtype=np.uint32)
    cbits = np.zeros(W, dtype=np.uint32)
    smax = np.zeros((P, G), dtype=np.float32) if want_series_max else None
    counts = np.zeros(3, dtype=np.uint64)
    thr = 0.0 if power_threshold is None else float(power_threshold)
    lib = load()
    args = (_p(util), _p(power), _p(eligible), _p(created_ts), int(cutoff_ts), P, G, T, 0, thr,
            _p(dbits), _p(cbits), _p(smax), _p(counts))
    rc = lib.gpo_decide(*args) if n_threads <= 1 else lib.gpo_decide_mt(n_threads, *args)
    if rc != 0:
        raise RuntimeError(f"oracle failed rc={rc}")
    W = (P + 31) // 32
    return {"decision_bits": dbits[:W], "candidate_bits": cbits[:W], "series_max": smax,
            "n_series": int(counts[0]), "n_candidates": int(counts[1]),
            "n_decisions": int(counts[2])}


def synth_fill(seed, plane, pod_offset, P, G, T, n_threads: int = 0):
    out = np.empty((P, G, T), dtype=np.float32)
    if n_threads <= 0:
        n_threads = hardware_threads()
    rc = load().gpo_synth_fill(n_threads, seed, plane, _p(out), pod_offset, P, G, T, 0)
    if rc != 0:
        raise RuntimeError("gpo_synth_fill failed")
    return out


def synth_eligible(seed, pod_offset, P):
    out = np.empty(P, dtype=np.uint8)
    load().gpo_synth_eligible(seed, _p(out), pod_offset, P)
    return out


def decide_synth(seed, pod_offset, P, G, T, use_power=False, power_threshold=0.0, use_elig=False,
                 n_threads: int = 0, want_series_max: bool = False, want_veto: bool = False):
    """want_series_max: also the window max of every util series ([P, G] float32); want_veto: also the packed
    bitmap of the pods the power clause vetoes"""
    if n_threads <= 0:
        n_threads = hardware_threads()
    W = max((P + 31) // 32, 1)
    dbits = np.zeros(W, dtype=np.uint32)
    cbits = np.zeros(W, dtype=np.uint32)
    vbits = np.zeros(W, dtype=np.uint32) if want_veto else None
    smax = np.empty((P, G), dtype=np.float32) if want_series_max else None
    counts = np.zeros(3, dtype=np.uint64)
    rc = load().gpo_decide_synth_ex(n_threads, seed, pod_offset, P, G, T, int(use_power),
                                    float(power_threshold), int(use_elig), _p(dbits), _p(cbits),
                                    _p(smax), _p(vbits), _p(counts))
    if rc != 0:
        raise RuntimeError("gpo_decide_synth failed")
    W = (P + 31) // 32
    out = {"decision_bits": dbits[:W], "candidate_bits": cbits[:W], "n_series": int(counts[0]),
           "n_candidates": int(counts[1]), "n_decisions": int(counts[2])}
    if want_series_max:
        out["series_max"] = smax
    if want_veto:
        out["veto_bits"] = vbits[:W]
    return out


def pool_pin(on: bool = True):
    """timed baseline only: pin the pool's workers to distinct CPUs (see gpr_oracle.h)"""
    load().gpo_pool_pin(1 if on else 0)


def hardware_threads() -> int:
    return int(load().gpo_hardware_threads())
