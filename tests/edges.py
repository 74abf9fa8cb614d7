"""Sample values where f32 and float64 part ways, with the text Prometheus puts on the wire.  TEST INFRASTRUCTURE.

The engine stores samples as f32; Prometheus decides on float64.  The two agree on integers and short decimals,
so tests built only from those cannot tell a kernel that rounds at the wrong place from a correct one.  This module
produces the values that can: power readings within an f32 ulp of the veto threshold (on either side, and for
thresholds that are not themselves f32), utilisation and PROF ratios that are non-zero but vanish in f32, 17-digit
ratios, NaN / +-Inf, numbers the device parser declines (more than 19 significant digits), and timestamps with
millisecond fractions.  Used by tests/test_promql_semantics.py (CPU ingest, emulated device) and
tests/test_gpu_promql.py (H100) against the float64 evaluation of tests/promql_mini.py.
"""
from __future__ import annotations

import math
from decimal import Decimal

import numpy as np

# veto thresholds: exact in f32, and not (the sample equal to a non-f32 threshold must still veto)
THRESHOLDS = [150.0, 150.5, 149.99, 0.1, 100.7]

# values at zero: `== 0` must survive the rounding to f32 for every one of them
ZEROISH = [-0.0, 5e-324, 1e-320, 1e-46, 1.4e-45, 1e-39, 1.1754942e-38, -5e-324, -1e-46, -1e-39]
# DCGM_FI_DEV_GPU_UTIL is divided by 100 before `== 0`; below ~2.5e-322 that division underflows to 0 in float64,
# which the f32 plane (non-zero kept non-zero) does not reproduce.  Not a value DCGM can report (an integer
# percentage) and not handled yet: utilisation draws stay above it
UTIL_ZEROISH = [x for x in ZEROISH if x == 0 or x / 100 != 0]
# DCGM_FI_PROF_GR_ENGINE_ACTIVE: shortest-round-trip doubles, up to 17 significant digits
RATIOS = [0.30000000000000004, 0.12345678901234568, 0.9999999999999999, 1e-07, 2.220446049250313e-16,
          0.010000000000000002]
SPECIAL = [math.nan, math.inf, -math.inf]


def go_float(x: float) -> str:
    """The text Prometheus writes for a sample value (util/jsonutil MarshalFloat): Go's strconv.FormatFloat with
    the shortest round-trip digits, 'e' format below 1e-6 and from 1e21 up, 'f' format otherwise."""
    if math.isnan(x):
        return "NaN"
    if math.isinf(x):
        return "+Inf" if x > 0 else "-Inf"
    sign = "-" if math.copysign(1.0, x) < 0 else ""
    if x == 0:
        return sign + "0"
    mant, _, exp = repr(abs(x)).partition("e")      # repr: the same shortest digits as Go's precision -1
    point = mant.index(".") if "." in mant else len(mant)
    digits = mant.replace(".", "")
    pos = point + (int(exp) if exp else 0)          # decimal point after `pos` digits
    while len(digits) > 1 and digits[0] == "0":
        digits, pos = digits[1:], pos - 1
    digits = digits.rstrip("0") or "0"
    if 1e-6 <= abs(x) < 1e21:
        if pos <= 0:
            body = "0." + "0" * -pos + digits
        elif pos >= len(digits):
            body = digits + "0" * (pos - len(digits))
        else:
            body = digits[:pos] + "." + digits[pos:]
    else:
        e = pos - 1
        body = digits[0] + ("." + digits[1:] if len(digits) > 1 else "") + "e" + ("-" if e < 0 else "+") + "%02d" % abs(e)
    out = sign + body
    assert float(out) == x
    return out


def long_spelling(x: float) -> str:
    """x spelt with more than 19 significant digits (the device parser declines it and the CPU re-parses the row);
    reads back as exactly x.  For values of moderate magnitude only."""
    assert 1e-3 <= abs(x) < 1e6, x
    s = format(Decimal(x), ".22f")
    assert float(s) == x and len(s.lstrip("-").replace(".", "").lstrip("0")) > 19, s
    return s


def f32_up(thr: float) -> float:
    """smallest f32 >= thr, as float64"""
    f = np.float32(thr)
    if float(f) < thr:
        f = np.nextafter(f, np.float32(np.inf))
    return float(f)


def power_edges(thr: float) -> list:
    """power readings around the threshold `thr`: thr itself, the f32 neighbours of its f32 rounding on both sides,
    the float64 neighbours of thr, thr - 2**-18 and thr - 1e-6 (149.999999 for 150)"""
    f = np.float32(thr)
    lo, hi = np.nextafter(f, np.float32(-np.inf)), np.nextafter(f, np.float32(np.inf))
    vals = [thr, float(f), float(lo), float(hi), math.nextafter(thr, -math.inf), math.nextafter(thr, math.inf),
            thr - 2.0 ** -18, float(repr(thr - 1e-6))]
    return sorted(set(vals))


def f32_rounding_flips(thr: float) -> list:
    """the readings below thr whose nearest f32 compares >= the threshold: the ones a plain rounding would veto"""
    up = np.float32(f32_up(thr))
    return [v for v in power_edges(thr) if v < thr and np.float32(v) >= up]
