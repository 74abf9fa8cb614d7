"""ctypes access to libgprhost.so (the C++ host logic) for the CPU tests."""
import ctypes as C
import json
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HOST_DIR = os.path.join(ROOT, "gpu-pruner_b200", "host")
SO = os.path.join(ROOT, "gpu-pruner_b200", "libgprhost.so")
BIN = os.path.join(ROOT, "gpu-pruner_b200", "gpu-pruner")
_lib = None
CAP = 1 << 22


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(SO):
            subprocess.check_call(["make", "-C", HOST_DIR, "-s", "../libgprhost.so"])
        _lib = C.CDLL(SO)
        _lib.gph_parse_rfc3339.restype = C.c_longlong
        _lib.gph_format_float.argtypes = [C.c_double, C.c_char_p, C.c_int]
        _lib.gph_rfc3339.argtypes = [C.c_longlong, C.c_char_p, C.c_int]
    return _lib


def _args(argv):
    blob = b"".join(a.encode() + b"\0" for a in argv)
    return blob, len(argv)


def _call(fn, *args):
    buf = C.create_string_buffer(CAP)
    rc = fn(*args, buf, CAP)
    return rc, buf.value.decode()


def parse_cli(argv):
    blob, n = _args(argv)
    rc, s = _call(lib().gph_parse_cli, blob, n)
    assert rc >= 0
    return json.loads(s)


def render_query(argv):
    blob, n = _args(argv)
    rc, s = _call(lib().gph_render_query, blob, n)
    assert rc >= 0, s
    return s


def render_selectors(argv):
    blob, n = _args(argv)
    rc, s = _call(lib().gph_render_selectors, blob, n)
    assert rc >= 0
    return json.loads(s)


def enabled_resources(letters):
    return lib().gph_enabled_resources(letters.encode())


def format_float(v):
    rc, s = _call(lib().gph_format_float, C.c_double(v))
    return s


def find_root(fixture_dir, pod_meta):
    rc, s = _call(lib().gph_find_root, fixture_dir.encode(), json.dumps(pod_meta).encode())
    assert rc >= 0
    return json.loads(s)


def scale_requests(kind, obj, now_ns=1_700_000_000_123_456_789, uuid="0123456789abcdef0123456789abcdef", pod_name=""):
    rc, s = _call(lib().gph_scale_requests, kind.encode(), json.dumps(obj).encode(), C.c_longlong(now_ns),
                  uuid.encode(), pod_name.encode())
    assert rc >= 0, rc
    return json.loads(s)


def generate_event(kind, obj, now_ns=0, uuid="", pod_name=""):
    rc, s = _call(lib().gph_generate_event, kind.encode(), json.dumps(obj).encode(), C.c_longlong(now_ns),
                  uuid.encode(), pod_name.encode())
    assert rc >= 0, rc
    return json.loads(s)


def scalekind_eq(kind_a, a, kind_b, b):
    h = (C.c_ulonglong * 2)()
    rc = lib().gph_scalekind_eq(kind_a.encode(), json.dumps(a).encode(), kind_b.encode(), json.dumps(b).encode(), h)
    assert rc >= 0
    return bool(rc), h[0], h[1]


def rfc3339(ns):
    rc, s = _call(lib().gph_rfc3339, C.c_longlong(ns))
    return s


def parse_rfc3339(s):
    return lib().gph_parse_rfc3339(s.encode())


def ingest_mode(threads):
    """-1: DOM reference path; >= 0: text path with that many parser threads (0 = all cores)"""
    lib().gph_ingest_mode(threads)


def ingest_dmi(dmi):
    """response of the node_dmi_info query applied by the following ingest() calls (None = none)"""
    lib().gph_ingest_dmi(None if dmi is None else json.dumps(dmi).encode())


def resolve_groups(series_max, candidate_bits, decision_bits, counts, veto_bits=None, eligible=None, created_ts=None,
                   cutoff=0):
    """exact `sum by` on the window of the last ingest(): returns corrected (candidate_bits, decision_bits, counts, changed)"""
    import numpy as np
    sm = np.ascontiguousarray(series_max, dtype=np.float32)
    cb = np.array(candidate_bits, dtype=np.uint32)
    db = np.array(decision_bits, dtype=np.uint32)
    cn = np.array(counts, dtype=np.uint64)
    p = lambda a, dt: None if a is None else np.ascontiguousarray(a, dtype=dt).ctypes.data_as(C.c_void_p)
    vb, el, cr = (None if veto_bits is None else np.ascontiguousarray(veto_bits, dtype=np.uint32),
                  None if eligible is None else np.ascontiguousarray(eligible, dtype=np.uint8),
                  None if created_ts is None else np.ascontiguousarray(created_ts, dtype=np.int64))
    rc = lib().gph_resolve_groups(sm.ctypes.data_as(C.c_void_p), p(vb, np.uint32), p(el, np.uint8), p(cr, np.int64),
                                  C.c_longlong(int(cutoff)), cb.ctypes.data_as(C.c_void_p), db.ctypes.data_as(C.c_void_p),
                                  cn.ctypes.data_as(C.c_void_p))
    assert rc >= 0
    return cb, db, tuple(int(x) for x in cn), rc


def group_values(series_max):
    import numpy as np
    sm = np.ascontiguousarray(series_max, dtype=np.float32)
    out = np.zeros(sm.shape, np.float64)
    assert lib().gph_group_values(sm.ctypes.data_as(C.c_void_p), out.ctypes.data_as(C.c_void_p)) == 0
    return out


def ingest(util, prof=None, power=None, duration_min=30, step=0, t_end=0, power_threshold=None):
    """power_threshold: what the power plane will be decided with (its samples are snapped to it; None = none)"""
    import numpy as np
    dims = (C.c_uint * 3)()
    enc = lambda j: None if j is None else json.dumps(j).encode()
    thr = C.c_double(0.0 if power_threshold is None else float(power_threshold))
    meta = C.create_string_buffer(CAP)
    rc = lib().gph_ingest_for_threshold(enc(util), enc(prof), enc(power), C.c_longlong(duration_min),
                                        C.c_longlong(step), C.c_longlong(t_end), thr, dims, None, None, meta, CAP)
    if rc != 0:
        raise RuntimeError(json.loads(meta.value.decode()).get("error", "ingest failed"))
    P, G, T = dims[0], dims[1], dims[2]
    u = np.zeros((P, G, T), np.float32)
    w = np.zeros((P, G, T), np.float32) if power is not None else None
    rc = lib().gph_ingest_for_threshold(enc(util), enc(prof), enc(power), C.c_longlong(duration_min),
                                        C.c_longlong(step), C.c_longlong(t_end), thr, dims, u.ctypes.data_as(C.c_void_p),
                                        None if w is None else w.ctypes.data_as(C.c_void_p), meta, CAP)
    assert rc == 0
    return u, w, json.loads(meta.value.decode())


def run_tick(argv, candidate_bits, series_max, n_series, fail=False, log_path=""):
    """one Controller::run_query_and_scale with a RECORDED verdict (no GPU): see capi.cpp gph_run_tick"""
    import numpy as np
    blob, n = _args(argv)
    cb = np.ascontiguousarray(candidate_bits, dtype=np.uint32)
    sm = np.ascontiguousarray(series_max, dtype=np.float32)
    buf = C.create_string_buffer(CAP)
    rc = lib().gph_run_tick(blob, n, cb.ctypes.data_as(C.c_void_p), sm.ctypes.data_as(C.c_void_p),
                            C.c_ulonglong(int(n_series)), int(fail), log_path.encode(), buf, CAP)
    assert rc >= 0, buf.value.decode()
    return json.loads(buf.value.decode())
