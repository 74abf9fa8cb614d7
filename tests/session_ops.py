"""Seeded random call sequences on one context, and the plain references they are checked against.  TEST
INFRASTRUCTURE, shared by tests/test_gpu_session.py (the sequences on an H100) and tests/test_session_plan.py (the
generator on the CPU).

A sequence is a list of operations (dicts with a "kind") drawn from a fixed seed.  Nothing here touches a device: a
window is a spec (shape, source, gates, table, outputs, data seed) and `window_data` / `expected` turn it into numpy
arrays and the result the engine must return.  The generator keeps a small model of the context (pending results,
the resident ring, the largest window so far) so that every sequence stays valid where it means to be valid, and
fails exactly where it means to fail:

  * decisions: blocking, async and batches of async, over device f32 (dense, strided, 4 bytes off alignment), device
    bytes, pinned f32 / bytes and (blocking only) pageable host windows; power, gates and `sum by` tables on and off;
    every optional output on or off, in host or device memory;
  * sync at random points;
  * the resident ring: init, append (host or device columns, n_new > T, power_cols NULL), advance, a text slice
    parsed into the ring then reindexed, decisions in whole and early mode, with and without a table;
  * the text planes: a scan and parse of util (and power) text, then async decisions on the plane pointers;
  * failing calls (FAILURES), each with the ABI's code.
"""
from __future__ import annotations

import math

import numpy as np

import edges
import groups_ref as R
import kat

SEEDS = list(range(12))
N_OPS = 60
MAX_CELLS = 3 << 20          # cells of the largest window (and the host staging capacity the engines get)
MAX_TABLE_SLOTS = 4200       # P * G of a window with a `sum by` table (the reference is a plain Python loop)
MAX_TEXT_CELLS = 60_000      # cells of a text plane (the text is built in Python)
MAX_PENDING = 256            # gpr.h: at most 256 results outstanding between two gpr_sync calls
GUARD = 16                   # words after every output buffer that must stay untouched
POISON = 0x7BADBEEF
POISON_F32 = np.float32(-777.0)
SENTINEL = 0xA5A5A5A5A5A5A5A5   # gpr_result counters before a call: still there = never retired
T_END = 1_700_000_000
STEP = 10                    # seconds per bucket of the text slices and planes

PS, GS, TS = [1, 31, 33, 1000, 9000], [1, 4, 33], [4, 181, 1800]
SOURCES = ["dev", "dev_strided", "dev_misaligned", "dev_u8", "pin", "pin_u8", "pageable", "pageable_u8"]
ASYNC_SOURCES = [s for s in SOURCES if not s.startswith("pageable")]
OUTPUTS = ("cand", "smax", "veto", "islots")

# code of every failing call (include/gpr.h)
E_INVALID, E_CAPACITY, E_STATE, E_UNSUPPORTED = -1, -4, -5, -7
FAILURES = {
    "struct_size": E_INVALID,          # blocking gpr_decide, gpr_window.struct_size wrong
    "g257": E_UNSUPPORTED,             # blocking, n_gpus = 257
    "bad_host_table": E_INVALID,       # blocking host window, malformed table
    "row_stride": E_INVALID,           # blocking, 0 < row_stride < n_samples
    "over_capacity": E_CAPACITY,       # blocking host window larger than the staging
    "resident_no_ring": E_STATE,       # gpr_decide_resident before gpr_resident_init
    "resident_stale": E_STATE,         # gpr_decide_resident on a stale block index
    "batch_fail": E_INVALID,           # a batch whose window k is invalid
    "async_bad_device_table": E_INVALID,  # async, malformed device table: the next gpr_sync fails
    "slots_full": E_STATE,             # the 257th outstanding result (async, then blocking)
}
BLOCKING_FAILURES = ("struct_size", "g257", "bad_host_table", "row_stride", "over_capacity", "resident_no_ring",
                     "resident_stale")
KINDS = ("decide", "async", "batch", "sync", "resident_init", "append", "advance", "text_resident", "reindex",
         "decide_resident", "text_planes", "fail")

# the engines every sequence runs on: (id, stream, GPR_PDL, kernel)
ENGINES = [("own-pdl-auto", "own", 1, "auto"), ("own-pdl-tma", "own", 1, "tma"), ("own-pdl-ldg", "own", 1, "ldg"),
           ("own-nopdl-auto", "own", 0, "auto"), ("caller-auto", "caller", 1, "auto")]


# ---- windows --------------------------------------------------------------------------------------------------
def is_host(src):
    return src.startswith("pin") or src.startswith("pageable")


def is_u8(src):
    return src.endswith("u8")


def cells(w):
    return w["P"] * w["G"] * w["T"]


def draw_window(rng, blocking=True, src=None, table=None, small=False):
    """a window spec; `table`: None = draw, False = none, "bad" = a malformed device table"""
    src = src or str(rng.choice(SOURCES if blocking else ASYNC_SOURCES))
    while True:
        P, G, T = int(rng.choice(PS)), int(rng.choice(GS)), int(rng.choice(TS))
        if small and P * G * T > 40_000:
            continue
        if P * G * T <= MAX_CELLS:
            break
    if table == "bad":
        G = max(G, 4)
    elif table is None:
        table = bool(G > 1 and P * G <= MAX_TABLE_SLOTS and rng.random() < 0.4)
    outs = {k: bool(rng.random() < 0.5) for k in OUTPUTS}
    return dict(src=src, P=P, G=G, T=T, seed=int(rng.integers(1 << 31)),
                thr=float(rng.choice(edges.THRESHOLDS)) if rng.random() < 0.5 else None,
                gates=bool(rng.random() < 0.5), table=table, outs=outs,
                out_kind="host" if rng.random() < 0.5 else "dev")


UTIL_F32 = np.array([0, 1, 50, 100, np.nan, -0.0, -3, 1e-45], np.float32)
UTIL_U8 = np.array([0, 1, 50, 100, np.nan], np.float32)
POWER = np.array([40, 60, 100.7, 149.99, 150, 150.5, np.nan], np.float32)


def _util(rng, P, G, T, u8):
    pal = UTIL_U8 if u8 else UTIL_F32
    u = rng.choice(pal, size=(P, G, T), p=[.85, .02, .01, .01, .09, .01, .005, .005][:len(pal)]
                   if not u8 else [.86, .02, .01, .02, .09])
    idle = rng.random((P, G)) < 0.5
    u[idle] = np.where(rng.random((int(idle.sum()), T)) < 0.05, np.nan, 0).astype(np.float32)
    burst = np.flatnonzero(rng.random(P) < 0.2)
    u[burst, rng.integers(0, G, burst.size), rng.integers(0, T, burst.size)] = 1.0
    return u.astype(np.float32)


def _power(rng, P, G, T):
    w = rng.choice(POWER[[0, 1, 6]], size=(P, G, T), p=[.5, .46, .04]).astype(np.float32)
    hot = np.flatnonzero(rng.random(P) < 0.4)
    w[hot, rng.integers(0, G, hot.size), rng.integers(0, T, hot.size)] = rng.choice(POWER[2:6], size=hot.size)
    return w


def window_data(w):
    """the arrays of a window spec: util f32 [P, G, T] (NaN = no sample; integer values for byte sources), power or
    None, eligible / created_ts / cutoff, table uint32 [P, G] or None"""
    rng = np.random.default_rng(w["seed"])
    P, G, T = w["P"], w["G"], w["T"]
    d = dict(util=_util(rng, P, G, T, is_u8(w["src"])), power=_power(rng, P, G, T) if w["thr"] else None,
             eligible=None, created_ts=None, cutoff_ts=0, table=None)
    if w["gates"]:
        d["eligible"] = (rng.random(P) < 0.9).astype(np.uint8)
        d["created_ts"] = rng.integers(1000, 2000, P).astype(np.int64)
        d["cutoff_ts"] = 1500
    if w["table"]:
        t = R.random_table(rng, P, G, share=0.6)
        if w["table"] == "bad":
            p = int(rng.integers(0, P))
            t[p, 2] = 3                                 # a leader above its slot
        d["table"] = t
    return d


def power_cell(x, thr):
    """the f32 a power reading x is stored as for the threshold thr (the POWER RULE of gpr.h)"""
    up = np.float32(edges.f32_up(thr))
    f = np.float32(x)
    if x >= thr and f < up:
        f = up
    if x < thr and f >= up:
        f = np.nextafter(up, np.float32(-np.inf))
    return f


def gate_mask(P, eligible, created_ts, cutoff_ts):
    ok = np.ones(P, bool)
    if eligible is not None:
        ok &= np.asarray(eligible).astype(bool)
    if created_ts is not None:
        ok &= ~(np.asarray(created_ts, np.int64) >= np.int64(cutoff_ts))
    return ok


def pack(b):
    pad = np.zeros(((len(b) + 31) // 32) * 32, bool)
    pad[:len(b)] = b
    return np.packbits(pad, bitorder="little").view("<u4").astype(np.uint32)


def expected(util, power=None, thr=None, eligible=None, created_ts=None, cutoff_ts=0, table=None):
    """what a decision must return: the C oracle without a table, groups_ref with one (gates on top), veto in float64,
    idle_slots from the row maxima or the group sums, series_max per row"""
    from oracle import oracle_c, oracle_np
    P, G, _ = util.shape
    use_power = power is not None and thr is not None and thr != 0 and not math.isnan(thr)
    veto = np.zeros(P, bool)
    if use_power:
        with np.errstate(invalid="ignore"):
            veto = (oracle_np.window_max(power) >= float(thr)).any(axis=1)
    if table is None:
        o = oracle_c.decide(util, power if use_power else None, eligible, created_ts, cutoff_ts,
                            thr if use_power else 0.0)
        smax = o["series_max"]
        g = R.decide(None, m=smax)
        out = dict(decision_bits=o["decision_bits"], candidate_bits=o["candidate_bits"], n_series=o["n_series"],
                   n_candidates=o["n_candidates"], n_decisions=o["n_decisions"])
    else:
        g = R.decide(util, power if use_power else None, thr if use_power else 0.0, table)
        smax = R.row_max(util)
        dec = g["candidate"] & gate_mask(P, eligible, created_ts, cutoff_ts)
        out = dict(decision_bits=pack(dec), candidate_bits=g["candidate_bits"], n_series=g["n_series"],
                   n_candidates=g["n_candidates"], n_decisions=int(dec.sum()))
    out.update(series_max=np.asarray(smax, np.float32), veto_bits=pack(veto), idle_slots=g["idle_slots"])
    return out


def expected_of(w):
    d = window_data(w)
    return expected(d["util"], d["power"], w["thr"], d["eligible"], d["created_ts"], d["cutoff_ts"], d["table"])


# ---- the resident ring and text ----------------------------------------------------------------------------------
def ring_columns(seed, rows, n, power):
    """host/device append columns [rows, n] (util, power or None): exact f32 values, so no power rule applies"""
    rng = np.random.default_rng(seed)
    u = rng.choice(np.array([0, 0, 0, 0, 3, np.nan], np.float32), size=(rows, n))
    u[rng.random(rows) < 0.5] = 0.0
    p = rng.choice(np.array([40, 60, 149.5, 150, 200, np.nan], np.float32), size=(rows, n),
                   p=[.5, .44, .02, .01, .01, .02]) if power else None
    return u.astype(np.float32), None if p is None else p.astype(np.float32)


TEXT_VALUES = ["0", "0", "0", "0", "0.0", "3", "1.5", "100", "NaN", "1e-3"]


def text_slice(seed, rows, n_new, t_end):
    """samples of the newest n_new buckets for a ring slice: [(row, [(ts, value text)])]; some buckets twice"""
    rng = np.random.default_rng(seed)
    out = []
    for r in range(rows):
        if rng.random() < 0.2:
            continue
        s = []
        for b in range(n_new):
            for _ in range(int(rng.integers(0, 3))):
                s.append((t_end - b * STEP - int(rng.integers(0, STEP)), str(rng.choice(TEXT_VALUES))))
        if s:
            out.append((r, s))
    if not out:            # every slice merges something, so a block index always goes stale
        out.append((0, [(t_end, "0")]))
    return out


def merge_slice(plane_bits, spans, t_end, window, T, col_end):
    """the ring plane (uint32 [rows, T]) after gpr_text_parse of `spans`: bucket back = (t_end - ts) // STEP,
    inside iff t_end - window < ts <= t_end, NaN-aware max per cell"""
    v = plane_bits.view(np.float32)
    for row, samples in spans:
        for ts, txt in samples:
            if not (t_end - window < ts <= t_end) or txt == "NaN":
                continue
            col = (col_end - (t_end - ts) // STEP) % T
            x = np.float32(float(txt))
            if np.isnan(v[row, col]) or v[row, col] < x:
                v[row, col] = x
    return plane_bits


def text_bytes(spans):
    """bare sample lists, one per span: (text, [(begin, end, row)])"""
    buf, out = [], []
    n = 0
    for row, samples in spans:
        body = ",".join('[%d,"%s"]' % (ts, v) for ts, v in samples)
        begin = n + 1
        buf.append("[" + body + "]\n")
        out.append((begin, begin + len(body), row))
        n += len(body) + 3
    return "".join(buf).encode(), out


def plane_text(seed, P, G, T, thr):
    """a context-plane window as text: util (and power) samples at the bucket times, some absent.
    -> (util spans, power spans or None, util f32 [P, G, T], power cells f32 [P, G, T] or None)"""
    rng = np.random.default_rng(seed)
    rows = P * G
    u = rng.choice(np.array([0, 0, 0, 0, 2, np.nan], np.float32), size=(rows, T))
    u[rng.random(rows) < 0.5] = 0.0
    u[rng.random((rows, T)) < 0.05] = np.nan
    ts = T_END - (T - 1 - np.arange(T)) * STEP
    uspans = [(r, [(int(ts[c]), "%d" % u[r, c]) for c in range(T) if not np.isnan(u[r, c])]) for r in range(rows)]
    if not thr:
        return uspans, None, u.reshape(P, G, T), None
    readings = [40.0, 60.0] + edges.power_edges(thr)
    x = np.array(readings)[rng.choice(len(readings), size=(rows, T), p=None)]
    x[rng.random((rows, T)) < 0.97] = 40.0
    wspans = [(r, [(int(ts[c]), edges.go_float(float(x[r, c]))) for c in range(T)]) for r in range(rows)]
    cellsf = np.array([[power_cell(float(v), thr) for v in row] for row in x], np.float32)
    return uspans, wspans, u.reshape(P, G, T), cellsf.reshape(P, G, T)


# ---- the generator ---------------------------------------------------------------------------------------------
def _ring_spec(rng, index=None):
    return dict(P=int(rng.choice([1, 3, 33])), G=int(rng.choice([1, 4])), T=int(rng.choice(TS)),
                power=bool(rng.random() < 0.6), index=bool(rng.random() < 0.5) if index is None else index)


def plan(seed, n_ops=N_OPS):
    """the operations of sequence `seed`"""
    rng = np.random.default_rng([seed, 0x5E55])
    ops = []
    st = dict(pending=0, ring=None, stale=False, t_end=T_END, max_cells=0)
    # every failure at least once, at random places (no ring before "resident_no_ring")
    fails = list(FAILURES)
    rng.shuffle(fails)
    fails.remove("resident_no_ring")
    slots = sorted(rng.choice(np.arange(6, n_ops - 2), size=len(fails), replace=False).tolist())
    scheduled = dict(zip(slots, fails))
    no_ring_at = int(rng.integers(0, 3))
    scheduled[no_ring_at] = "resident_no_ring"

    def add(op):
        ops.append(op)
        k = op["kind"]
        if k in ("decide", "decide_resident"):
            st["pending"] = 0
        elif k == "async":
            st["pending"] += 1
        elif k == "batch":
            st["pending"] += len(op["wins"])
        elif k == "text_planes":
            st["pending"] += len(op["decisions"])
        elif k == "sync":
            st["pending"] = 0
        elif k == "fail":
            f = op["fail"]
            if f == "batch_fail":
                st["pending"] += op["k"]
            elif f in ("async_bad_device_table", "slots_full"):
                st["pending"] = 0                     # both end with the gpr_sync they test
        for w in op.get("wins", []) + ([op["win"]] if "win" in op else []):
            st["max_cells"] = max(st["max_cells"], cells(w))

    def decision(kind):
        blocking = kind == "decide"
        return dict(kind=kind, win=draw_window(rng, blocking))

    i = 0
    while len(ops) < n_ops or i <= max(scheduled):
        f = scheduled.get(i)
        i += 1
        if st["pending"] > MAX_PENDING - 40:
            add(dict(kind="sync"))
            continue
        if f is not None:
            if f in BLOCKING_FAILURES and st["pending"] == 0:
                add(decision("async"))                # something pending that the failure must not drop
            if f == "resident_stale":
                if st["ring"] is None or not st["ring"]["index"]:
                    st["ring"] = _ring_spec(rng, index=True)
                    add(dict(kind="resident_init", ring=st["ring"]))
                n_new = int(rng.integers(1, 4))
                add(dict(kind="text_resident", n_new=n_new, seed=int(rng.integers(1 << 31))))
                st["stale"] = True
            if f == "resident_no_ring":
                assert st["ring"] is None
            op = dict(kind="fail", fail=f, code=FAILURES[f])
            if f == "batch_fail":
                n = int(rng.integers(3, 7))
                op["wins"] = [draw_window(rng, False, small=True) for _ in range(n)]
                op["k"] = int(rng.integers(0, n))
                op["how"] = str(rng.choice(["row_stride", "struct_size"]))
            elif f == "async_bad_device_table":
                op["before"] = [draw_window(rng, False, small=True) for _ in range(int(rng.integers(0, 3)))]
                op["win"] = draw_window(rng, False, src="dev", table="bad", small=True)
                op["after"] = [draw_window(rng, False, small=True) for _ in range(int(rng.integers(1, 3)))]
            elif f == "slots_full":
                op["wins"] = [draw_window(rng, False, src=str(rng.choice(["dev", "pin"])), table=False, small=True)
                              for _ in range(4)]
            elif f in ("struct_size", "row_stride", "bad_host_table", "resident_stale"):
                op["win"] = draw_window(rng, True, src="pageable" if f == "bad_host_table" else None,
                                        table=True if f == "bad_host_table" else None, small=True)
                if f == "bad_host_table" and op["win"]["G"] < 4:
                    op["win"]["G"] = 4
            add(op)
            continue
        r = rng.random()
        if i <= no_ring_at and 0.56 <= r < 0.78:
            r = 0.2                                   # no ring before the call that needs none
        if r < 0.14:
            add(decision("decide"))
        elif r < 0.36:
            add(decision("async"))
        elif r < 0.46:
            n = int(rng.integers(2, 7))
            add(dict(kind="batch", wins=[draw_window(rng, False) for _ in range(n)]))
        elif r < 0.56:
            add(dict(kind="sync"))
        elif r < 0.62 or (r < 0.78 and st["ring"] is None):
            st["ring"] = _ring_spec(rng)
            st["stale"] = False
            add(dict(kind="resident_init", ring=st["ring"]))
        elif r < 0.78:
            ring = st["ring"]
            q = rng.random()
            if st["stale"]:
                add(dict(kind="reindex"))
                st["stale"] = False
            elif q < 0.3:
                T = ring["T"]
                n_new = int(rng.choice([1, 3, max(1, T - 1), T, T + 5]))
                add(dict(kind="append", n_new=n_new, src=str(rng.choice(["host", "dev"])),
                         power_cols=bool(ring["power"] and rng.random() < 0.7),
                         stride=int(rng.choice([0, 0, n_new + 3])), seed=int(rng.integers(1 << 31))))
            elif q < 0.45:
                add(dict(kind="advance", n_new=int(rng.choice([1, 7, ring["T"] + 2]))))
            elif q < 0.6:
                add(dict(kind="text_resident", n_new=int(rng.integers(1, 4)), seed=int(rng.integers(1 << 31))))
                st["stale"] = ring["index"]
            else:
                P, G = ring["P"], ring["G"]
                add(dict(kind="decide_resident", mode=str(rng.choice(["whole", "early"])),
                         table=bool(G > 1 and rng.random() < 0.5), gates=bool(rng.random() < 0.5),
                         thr=float(rng.choice(edges.THRESHOLDS)) if ring["power"] and rng.random() < 0.7 else None,
                         gates_kind=str(rng.choice(["host", "dev"])), seed=int(rng.integers(1 << 31))))
        elif r < 0.84:
            while True:
                P, G, T = int(rng.choice(PS[:4])), int(rng.choice(GS)), int(rng.choice(TS[:2]))
                if P * G * T <= MAX_TEXT_CELLS:
                    break
            thr = float(rng.choice(edges.THRESHOLDS)) if rng.random() < 0.5 else None
            decs = []
            for _ in range(int(rng.integers(1, 4))):
                w = draw_window(rng, False, src="dev", table=False)
                decs.append(dict(outs=w["outs"], out_kind=w["out_kind"], power=bool(thr)))
            add(dict(kind="text_planes", P=P, G=G, T=T, thr=thr, seed=int(rng.integers(1 << 31)), decisions=decs))
        else:
            add(decision("async"))
    return ops


def ring_after_slice(model, op, t_end):
    """advance the model ring by op["n_new"] buckets and merge the op's text slice; -> (spans, window)"""
    n_new = op["n_new"]
    model.advance(n_new)
    spans = text_slice(op["seed"], model.rows, n_new, t_end)
    window = n_new * STEP
    merge_slice(model.planes[0], spans, t_end, window, model.T, (model.head + model.T - 1) % model.T)
    return spans, window


# ---- what a plan exercises (tests/test_session_plan.py) -----------------------------------------------------------
def transitions(ops):
    """the transitions a plan reaches (each needs only the plan, not the engine)"""
    seen = set()
    pending, biggest = 0, 0
    last = None
    for op in ops:
        k = op["kind"]
        wins = ([op["win"]] if "win" in op and k in ("decide", "async") else []) + (op["wins"] if k == "batch" else [])
        for w in wins:
            if last is not None and last["kind"] == "async" and not last["win"]["table"] and k in ("async", "batch") \
                    and w["table"]:
                seen.add("grouped after ungrouped async")
            if last is not None and last["kind"] == "async" and last["win"]["out_kind"] == "dev" \
                    and w["out_kind"] == "host":
                seen.add("host-out after device-out")
            if pending and cells(w) > biggest:
                seen.add("growth while results are pending")
            biggest = max(biggest, cells(w))
            last = dict(kind="async" if k != "decide" else "decide", win=w)
            pending = 0 if k == "decide" else pending + 1
        if k == "fail" and op["fail"] == "batch_fail" and op["k"] > 0:
            seen.add("batch failing at k > 0")
        if k == "text_planes" and pending:
            seen.add("text planes parsed while results are pending")
        if k == "text_planes":
            pending += len(op["decisions"])
        if k in ("sync", "decide_resident") or (k == "fail" and op["fail"] in ("async_bad_device_table",
                                                                                "slots_full")):
            pending = 0
        if k not in ("decide", "async", "batch"):
            last = None
    return seen


TRANSITIONS = ("grouped after ungrouped async", "host-out after device-out", "growth while results are pending",
               "batch failing at k > 0", "text planes parsed while results are pending")
