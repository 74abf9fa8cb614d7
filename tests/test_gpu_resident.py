"""The resident ring of daemon mode through libgpr.so on an H100, against the numpy ring model of
tests/ring_scripts.py and the float64 oracle.

Every script of tests/test_ring_emul.py runs on two engines per kernel variant (GPR_KERNEL=ldg / tma / auto): one whose
ring keeps the block index (GPR_F_BLOCK_INDEX, deciding on idx_ld = ceil(T / 64) padded to a multiple of 4 "samples"
per series, a TMA-able row) and one that rescans the ring.  After every operation the ring is read back and must equal
the model bit for bit, and gpr_decide_resident (power threshold 150 W) must give the oracle's verdict on the unrolled
window twice: once with series_max (every row read whole) and once with idle_slots and no series_max (rows stop at
their first settling sample; AUTO runs the probe kernel), every row's idle slot checked; the two engines must agree.
The appended columns come from pageable and pinned host memory and from device memory, at a 16-byte and at a 4-byte
aligned address."""
import json

import numpy as np
import pytest

import kat
import ring_scripts as RS
from test_gpu_parity import assert_ran, expected_idle_slots, plan_exe, resident_ld  # noqa: F401 (a fixture)

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")
VARIANTS = ["ldg", "tma", "auto"]
CASES = RS.cases()
SOURCES = ["pageable", "pinned", "device", "device+4"]
_MAX_CELLS = 1 << 20    # the largest source of any script: rows * ld per plane


@pytest.fixture(scope="module")
def engines():
    import gpu_pruner_b200 as g
    if not torch.cuda.is_available():
        pytest.fail("-m gpu tests need a CUDA device; the engine has no CPU fallback")
    e = {(v, ix): g.IdleEngine(device=0, kernel=v) for v in VARIANTS for ix in (True, False)}
    bufs = {k: (x.host_array((2 * _MAX_CELLS,), np.uint32),
                torch.empty(2 * _MAX_CELLS + 4, dtype=torch.int32, device="cuda:0")) for k, x in e.items()}
    yield e, bufs
    for x in e.values():
        x.close()


def _pack(flags):
    w = np.zeros(max((len(flags) + 31) // 32, 1), np.uint32)
    for p in np.flatnonzero(flags):
        w[p >> 5] |= np.uint32(1 << (int(p) & 31))
    return w[:(len(flags) + 31) // 32]


def expected(m: RS.Ring):
    """the oracle on the unrolled window, and the veto bits by float64 comparison"""
    from oracle import oracle_c
    power = m.window(1) if len(m.planes) > 1 else None
    exp = oracle_c.decide(m.window(0), power, power_threshold=RS.THR if power is not None else 0.0)
    veto = np.zeros(m.P, bool) if power is None else np.any(power.astype(np.float64) >= RS.THR, axis=(1, 2))
    exp["veto_bits"] = _pack(veto)
    return exp


def decide(eng, m: RS.Ring, early=False):
    """gpr_decide_resident with series_max, or (early) with idle_slots and no series_max"""
    from gpu_pruner_b200 import ffi
    W = max((m.P + 31) // 32, 1)
    db, cb, vb = (np.full(W, 0xDEADBEEF, np.uint32) for _ in range(3))
    sm = None if early else np.full((m.P, m.G), -777.0, np.float32)
    isl = np.full((max(m.P, 1), (m.G + 31) // 32), 0xDEADBEEF, np.uint32) if early else None
    r = eng.decide_ptr(None, 0, 0, 0, db, candidate_bits=cb, series_max=sm, veto_bits=vb, idle_slots=isl,
                       power_threshold=RS.THR if len(m.planes) > 1 else 0.0, in_kind=ffi.GPR_MEM_HOST,
                       out_kind=ffi.GPR_MEM_HOST, resident=True)
    W = (m.P + 31) // 32
    out = {"decision_bits": db[:W], "candidate_bits": cb[:W], "veto_bits": vb[:W],
           "n_series": r.n_series, "n_candidates": r.n_candidates, "n_decisions": r.n_decisions}
    if early:
        out["idle_slots"] = isl[:m.P]
    else:
        out["series_max"] = sm
    return out


def same_verdict(got, exp):
    """None, or the first output of `got` that differs from `exp` (an oracle result or another engine's)"""
    for k in ("decision_bits", "candidate_bits", "veto_bits"):
        if not np.array_equal(got[k], exp[k]):
            return k
    if (got["n_series"], got["n_candidates"], got["n_decisions"]) != \
            (exp["n_series"], exp["n_candidates"], exp["n_decisions"]):
        return "counts"
    if "series_max" in got and not kat.smax_equal(got["series_max"], exp["series_max"]):
        return "series_max"
    if "idle_slots" in got:
        want = exp["idle_slots"] if "idle_slots" in exp else expected_idle_slots(exp["series_max"])
        if not np.array_equal(got["idle_slots"], want):
            return "idle_slots"
    return None


def _read_ring(eng, m):
    from gpu_pruner_b200 import ffi
    u, p, ld = eng.resident_planes()
    assert ld == m.T
    out = []
    for ptr in (u, p)[:len(m.planes)]:
        a = np.empty((m.rows, m.T), np.uint32)
        eng.memcpy(a, ptr, a.nbytes, ffi.GPR_MEM_HOST, ffi.GPR_MEM_DEVICE)
        out.append(a)
    return out


def _append(eng, bufs, kind, op):
    """gpr_append of the op's columns (rows x ld, uint32 bits) from memory of the given kind"""
    from gpu_pruner_b200 import ffi
    _, n_new, ld, util, power = op
    host, dev = bufs
    srcs = [a for a in (util, power) if a is not None]
    if kind == "pageable":
        ptrs = [a.ctypes.data for a in srcs]
        mk = ffi.GPR_MEM_HOST
    elif kind == "pinned":
        ptrs, off = [], 0
        for a in srcs:
            host[off:off + a.size] = a.ravel()
            ptrs.append(host.ctypes.data + 4 * off)
            off += a.size + 4
        mk = ffi.GPR_MEM_HOST
    else:
        shift = 1 if kind == "device+4" else 0       # 4 bytes off the 16-byte alignment of the allocation
        ptrs, off = [], shift
        for a in srcs:
            dev[off:off + a.size].copy_(torch.from_numpy(a.ravel().view(np.int32)))
            ptrs.append(dev.data_ptr() + 4 * off)
            off += a.size + 4
        torch.cuda.synchronize()
        mk = ffi.GPR_MEM_DEVICE
    eng.append(ptrs[0], ptrs[1] if power is not None else None, n_new=n_new, row_stride=ld, mem_kind=mk)


def run_script(eng, bufs, case, index):
    """run the case on one engine, the ring checked after every operation; returns the verdicts"""
    from gpu_pruner_b200 import ffi
    flags = (case.flags | 2) if index else (case.flags & ~2)
    ops = [("init", case.P, case.G, case.T, flags)] + case.ops[1:]
    out, n_app = [], 0
    m = None
    for i, op in enumerate(ops):
        last_write = op[0] == "write" and (i + 1 == len(ops) or ops[i + 1][0] != "write")
        if op[0] == "init":
            eng.resident_init(op[1], op[2], op[3], power_plane=bool(op[4] & 1), block_index=bool(op[4] & 2))
            m = RS.Ring(*op[1:])
        elif op[0] == "append":
            _append(eng, bufs, SOURCES[n_app % len(SOURCES)], op)
            n_app += 1
            m.append(op[1], op[3], op[4])
        elif op[0] == "advance":
            eng.resident_advance(op[1])
            m.advance(op[1])
        elif op[0] == "write":              # direct writes, as a generator would make them
            u, p, _ = eng.resident_planes()
            eng.memcpy((u, p)[op[1]], op[2], op[2].nbytes, ffi.GPR_MEM_DEVICE, ffi.GPR_MEM_HOST)
            m.write(op[1], op[2])
            if index and last_write and not case.flags & 2:
                eng.resident_reindex()      # the script was written for a ring without an index
        else:
            eng.resident_reindex()
        assert eng.resident_head() == m.head, (case.name, i, op[0])
        for pl, (got, want) in enumerate(zip(_read_ring(eng, m), m.planes)):
            if not np.array_equal(got, want):
                r, t = np.argwhere(got != want)[0]
                raise AssertionError(f"{case.name} op {i} ({op[0]}): plane {pl} row {r} position {t}: "
                                     f"{got[r, t]:#010x} != {want[r, t]:#010x}")
        if op[0] == "write" and index and not (last_write and not case.flags & 2):
            out.append(None)                # the index is rebuilt by the reindex that follows (gpr.h)
            continue
        exp = expected(m)
        got = [decide(eng, m), decide(eng, m, early=True)]
        for g, mode in zip(got, ("whole", "early")):
            bad = same_verdict(g, exp)
            assert bad is None, \
                f"{case.name} op {i} ({op[0]} {op[1:2]}), index={index}, {mode}: {bad} differs from the oracle"
        out.append(got)
    return out


@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("case", CASES, ids=[c.name for c in CASES])
def test_ring_scripts(case, variant, engines, plan_exe):
    e, bufs = engines
    sm_count = e[(variant, True)].device_info()["sm_count"]
    for index in (True, False):
        for mode in ("whole", "early"):
            assert_ran(plan_exe, sm_count, variant, mode, resident_ld(case.T, index),
                       case.P * case.G * (2 if case.flags & 1 else 1), resident_ld(case.T, index) % 4 == 0)
    a = run_script(e[(variant, True)], bufs[(variant, True)], case, True)
    b = run_script(e[(variant, False)], bufs[(variant, False)], case, False)
    assert len(a) == len(b) == len(case.ops)
    for i, (x, y) in enumerate(zip(a, b)):
        if x is not None:
            for mode, xm, ym in zip(("whole", "early"), x, y):
                assert same_verdict(xm, ym) is None, (case.name, i, mode)


@pytest.mark.parametrize("index", [False, True], ids=["rescan", "block-index"])
def test_append_without_power_columns_opens_them(index, engines):
    """P = G = 1, T = 4: readings of 200 W, then a tick of util zeros with power_cols NULL.  The window has no power
    sample left, so nothing vetoes the pod and it is a candidate (the old readings used to stay and veto it)."""
    e, bufs = engines
    eng = e[("tma", index)]
    T = 4
    eng.resident_init(1, 1, T, power_plane=True, block_index=index)
    eng.append(np.zeros((1, 1, T), np.float32), np.full((1, 1, T), 200.0, np.float32))
    m = RS.Ring(1, 1, T, 1 | (2 if index else 0))
    assert decide(eng, m)["n_candidates"] == 0
    eng.append(np.zeros((1, 1, T), np.float32), None)
    got = decide(eng, m)
    assert got["n_candidates"] == 1 and got["veto_bits"][0] == 0
    u, p = _read_ring(eng, m)
    assert (p == RS.NO_SAMPLE).all()


def test_advance_recomputes_the_block_index(engines):
    """T = 128 with the index: 64 columns of 5, 64 of 0, then gpr_resident_advance(64) opens the columns of 5.  The
    window holds zeros and no-sample buckets, so the series is idle with series_max 0 (the index used to keep 5)."""
    e, _ = engines
    eng = e[("tma", True)]
    T = 128
    eng.resident_init(1, 1, T, block_index=True)
    eng.append(np.full((1, 1, 64), 5.0, np.float32))
    eng.append(np.zeros((1, 1, 64), np.float32))
    eng.resident_advance(64)
    got = decide(eng, RS.Ring(1, 1, T, 2))
    assert got["n_candidates"] == 1 and got["series_max"][0, 0] == 0.0


def test_text_parse_marks_the_index_stale(engines):
    """advance + gpr_text_parse(GPR_TEXT_RESIDENT) on an index ring: deciding is refused until gpr_resident_reindex,
    then the verdict and series_max equal those of the rescan engine on the same text"""
    import gpu_pruner_b200 as g
    from test_gpu_text import T_END, _labels, _spans_from_markers
    e, _ = engines
    rng = np.random.default_rng(21)
    P, G, T, n_new = 40, 2, 192, 30
    vals = rng.choice(np.array([0, 0, 0, 0, 3, 100], np.float32), size=(P * G, T + 3 * n_new))
    vals[rng.random(vals.shape) < 0.1] = np.nan
    vals[: P * G // 2, T - 20:] = 0.0      # a burst early in the window that later ticks push out
    vals[: P * G // 2, T - 40:T - 20] = 7.0
    t0 = T_END - vals.shape[1]

    def text_for(lo, hi):
        parts = []
        for r in range(P * G):
            body = ",".join('[%d,"%s"]' % (t0 + i + 1, "NaN" if np.isnan(vals[r, i]) else "%g" % vals[r, i])
                            for i in range(lo, hi))
            parts.append('{"metric":' + json.dumps(_labels(r // G, r % G), separators=(",", ":")) + ',"values":['
                         + body + "]}")
        return ('{"status":"success","data":{"resultType":"matrix","result":[' + ",".join(parts) + "]}}").encode()

    engs = [e[("tma", True)], e[("tma", False)]]
    for x, ix in zip(engs, (True, False)):
        x.resident_init(P, G, T, block_index=ix)
    hi = T
    for tick in range(4):
        lo = 0 if tick == 0 else hi - n_new
        text = text_for(lo, hi)
        res = []
        for x, ix in zip(engs, (True, False)):
            opens, closes = x.text_scan(text)
            spans = _spans_from_markers(text, opens, closes, x)
            x.resident_advance(T if tick == 0 else n_new)
            x.text_parse(spans, t0 + hi, 1, T, P * G, resident=True, window_seconds=T if tick == 0 else n_new)
            if ix:
                with pytest.raises(g.GprError) as ei:
                    decide(x, RS.Ring(P, G, T, 2))
                assert ei.value.code == g.ffi.GPR_E_STATE and "gpr_resident_reindex" in str(ei.value)
                x.resident_reindex()
            res.append(decide(x, RS.Ring(P, G, T, 0)))
        assert same_verdict(res[0], res[1]) is None, tick
        win = vals[:, hi - T:hi].reshape(P, G, T)
        from oracle import oracle_c
        exp = oracle_c.decide(win)
        exp["veto_bits"] = _pack(np.zeros(P, bool))
        assert same_verdict(res[1], exp) is None, tick
        hi += n_new


def test_c2_sized_daemon_run(engines, oracle_c):
    """10,000 pods x 4 GPUs x 1,800 samples with power and the index (0.6 GB of HBM): a full window, then 12 ticks of
    180 columns from pinned memory, so the head wraps; the oracle's verdict at every tick"""
    e, _ = engines
    eng = e[("tma", True)]
    P, G, T, n_new, ticks = 10000, 4, 1800, 180, 12
    total = T + ticks * n_new
    seed = 0x5EED0C02
    util = oracle_c.synth_fill(seed, 0, 0, P, G, total)
    power = oracle_c.synth_fill(seed, 1, 0, P, G, total)
    eng.resident_init(P, G, T, power_plane=True, block_index=True)
    cols_u = eng.host_array((P, G, n_new), np.float32)
    cols_w = eng.host_array((P, G, n_new), np.float32)
    eng.append(np.ascontiguousarray(util[:, :, :T]), np.ascontiguousarray(power[:, :, :T]))
    t = T
    heads = set()
    for k in range(ticks + 1):
        m = RS.Ring(P, G, T, 3)
        got = decide(eng, m)
        exp = oracle_c.decide(util[:, :, t - T:t], power[:, :, t - T:t], power_threshold=RS.THR, n_threads=8)
        exp["veto_bits"] = _pack(np.any(power[:, :, t - T:t].astype(np.float64) >= RS.THR, axis=(1, 2)))
        assert same_verdict(got, exp) is None, k
        heads.add(eng.resident_head())
        if k == ticks:
            break
        cols_u[...] = util[:, :, t:t + n_new]
        cols_w[...] = power[:, :, t:t + n_new]
        eng.append(cols_u.ctypes.data, cols_w.ctypes.data, n_new=n_new)
        t += n_new
    assert len(heads) == 10 and 0 in heads      # the head went round the ring and wrapped
