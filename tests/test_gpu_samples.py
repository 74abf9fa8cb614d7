"""gpr_samples_scatter on the H100 against the device text parser it must equal (include/gpr.h): the same samples
rendered as matrix JSON (round-trip repr values, whole-millisecond timestamps) and run through gpr_text_scan +
gpr_text_parse give bit-identical planes, for the util plane and for the power plane with its threshold, and the
span counters add up to the scatter's stats.  Then: every source memory (pageable, pinned, device, and a batch of
more than 10 M samples whose 2 Mi-sample upload pieces cut inside and between series), a daemon timeline into the
resident ring next to a text-fed twin, the C2 synthetic window turned into samples and decided, and every invalid
batch leaving a pre-filled plane byte-identical."""
import ctypes as C
import os

import numpy as np
import pytest

import kat

pytestmark = pytest.mark.gpu

FILL = np.uint32(0xFFFFFFFF)
T_END = 1_700_000_040            # s
STEP = 1
THR = 150.0


def _engine():
    import gpu_pruner_b200 as g
    torch = pytest.importorskip("torch")
    if not torch.cuda.is_available():
        pytest.fail("-m gpu tests need a CUDA device; the engine has no CPU fallback")
    return g.IdleEngine(device=0)


@pytest.fixture(scope="module")
def eng():
    e = _engine()
    yield e
    e.close()


def _read(eng, ptr, n_rows, T):
    out = np.empty((n_rows, T), np.uint32)
    eng.memcpy(out, ptr, out.nbytes, 0, 1)
    return out


def _plane(eng, n_rows, T, plane=0):
    return _read(eng, eng.text_planes()[plane], n_rows, T)


# ---- the same samples as text ------------------------------------------------------------------------------------
def _value_text(v):
    if np.isnan(v):
        return "NaN"
    if np.isinf(v):
        return "+Inf" if v > 0 else "-Inf"
    return repr(float(v))


def _render(offsets, rows, ts, vals):
    """matrix JSON of the non-empty series (Prometheus emits no empty sample list); -> (bytes, [(row, series)])"""
    parts, order = [], []
    for s in range(len(rows)):
        a, e = int(offsets[s]), int(offsets[s + 1])
        if a == e:
            continue
        samples = ",".join(f'[{t // 1000}.{t % 1000:03d},"{_value_text(v)}"]' for t, v in zip(ts[a:e].tolist(),
                                                                                            vals[a:e].tolist()))
        parts.append('{"metric":{"__name__":"DCGM_FI_DEV_GPU_UTIL","pod":"p%d"},"values":[%s]}' % (s, samples))
        order.append(int(rows[s]))
    text = '{"status":"success","data":{"resultType":"matrix","result":[' + ",".join(parts) + "]}}"
    return text.encode(), order


def _text_parse(eng, text, order, T, n_rows, plane, thr, resident=False, window=None, slot=0):
    opens, closes = eng.text_scan(text, slot=slot)
    assert len(opens) == len(order)
    import gpu_pruner_b200 as g
    sp = np.zeros(len(order), g.IdleEngine.SPAN_DTYPE)
    for i, o in enumerate(opens):
        b = int(o) + 12
        sp[i]["begin"], sp[i]["end"], sp[i]["row"] = b, int(closes[np.searchsorted(closes, b)]) + 2, order[i]
    out = eng.text_parse(sp, T_END, STEP, T, n_rows, slot=slot, plane=plane, power_threshold=thr, resident=resident,
                         window_seconds=window)
    assert not (out["flags"] & 2).any(), "a span went to the CPU parser: keep values within the device grammar"
    return {"n_in": int(out["n_in"].sum()), "n_oow": int(out["n_oow"].sum()), "n_tiny": int(out["n_tiny"].sum())}


SPECIAL = np.array([0.0, -0.0, -3.5, -7.25, 1e-50, -1e-50, 1e39, -1e39, np.nan, np.inf, -np.inf, 149.999999, 150.0,
                    150.0000001, 149.99999999999997, 7e-46, 0.1, 1 / 3, 0.30000000000000004, 2.5e-07, 1e21])


def _random_batch(rng, n_series, n_rows, T, max_len=400, window=None):
    window = T * STEP if window is None else window
    lengths = rng.integers(0, max_len, n_series)
    lengths[rng.random(n_series) < 0.05] = 0
    offsets = np.concatenate([[0], np.cumsum(lengths)]).astype(np.uint64)
    n = int(offsets[-1])
    ts = T_END * 1000 - rng.integers(-3000, window * 1000 + 5000, n)          # some outside on both sides
    ts[rng.random(n) < 0.05] = T_END * 1000 - window * 1000                    # the open edge
    ts[rng.random(n) < 0.05] = T_END * 1000                                     # the closed edge
    v = rng.integers(0, 101, n).astype(np.float64)                               # integer percentages
    ratio = rng.random(n) < 0.3
    v[ratio] = rng.random(int(ratio.sum()))                                      # 17-digit PROF ratios
    pick = rng.random(n) < 0.3
    v[pick] = rng.choice(SPECIAL, int(pick.sum()))
    rows = rng.integers(0, n_rows, n_series).astype(np.uint32)                  # several series per row
    return offsets, rows, ts.astype(np.int64), v


@pytest.mark.parametrize("plane,thr", [(0, 0.0), (1, THR), (1, 149.99)])
def test_bit_identical_to_the_text_path(eng, plane, thr):
    rng = np.random.default_rng(11 + plane)
    T, n_rows = 120, 300
    offsets, rows, ts, vals = _random_batch(rng, 700, n_rows, T)
    text, order = _render(offsets, rows, ts, vals)
    counts = _text_parse(eng, text, order, T, n_rows, plane, thr)
    want = _plane(eng, n_rows, T, plane)
    st = eng.samples_scatter(offsets, rows, ts, vals, T_END, STEP, T, n_rows, plane=plane, power_threshold=thr)
    got = _plane(eng, n_rows, T, plane)
    assert np.array_equal(got, want), np.argwhere(got != want)[:8]
    assert st == counts and st["n_in"] == len(ts) and st["n_tiny"] > 0 and st["n_oow"] > 0
    assert (want != FILL).sum() > n_rows * T // 2


def _torch_dev(a):
    import torch
    t = torch.from_numpy(np.ascontiguousarray(a)).cuda()
    torch.cuda.synchronize()   # the context's stream is not ordered with torch's (include/gpr.h)
    return t


def test_every_source_gives_the_same_plane(eng):
    """pageable, pinned and device batches; 10.8 M samples in ragged series, so the 2 Mi-sample upload pieces of the
    host batches end inside series and next to empty ones; the device batch once at an address 8 bytes off a 16-byte
    boundary (scalar loads)"""
    import gpu_pruner_b200 as g
    rng = np.random.default_rng(21)
    T, n_rows = 1800, 6000
    lengths = rng.integers(1500, 2100, n_rows)
    lengths[rng.random(n_rows) < 0.02] = 0
    offsets = np.concatenate([[0], np.cumsum(lengths)]).astype(np.uint64)
    n = int(offsets[-1])
    assert n >= 10_000_000
    rows = rng.permutation(n_rows).astype(np.uint32)
    ts = T_END * 1000 - rng.integers(-2000, T * 1000 + 2000, n).astype(np.int64)
    vals = rng.integers(0, 101, n).astype(np.float64)
    vals[rng.random(n) < 0.1] = 0.0
    ratio = rng.random(n) < 0.2
    vals[ratio] = rng.random(int(ratio.sum()))
    vals[rng.random(n) < 0.2] = np.nan
    cuts = np.arange(1, n // (2 << 20) + 1) * (2 << 20)
    starts = offsets[:-1][lengths > 0]
    assert len(cuts) >= 4 and not np.isin(cuts, starts).all()    # pieces end inside series

    planes, stats = {}, {}
    stats["pageable"] = eng.samples_scatter(offsets, rows, ts, vals, T_END, STEP, T, n_rows)
    planes["pageable"] = _plane(eng, n_rows, T)
    pts, pvals = eng.host_array(n, np.int64), eng.host_array(n, np.float64)
    pts[:], pvals[:] = ts, vals
    stats["pinned"] = eng.samples_scatter(offsets, rows, pts, pvals, T_END, STEP, T, n_rows)
    planes["pinned"] = _plane(eng, n_rows, T)
    d_off, d_rows = _torch_dev(offsets.view(np.int64)), _torch_dev(rows.view(np.int32))
    d_ts, d_vals = _torch_dev(ts), _torch_dev(vals)
    stats["device"] = eng.samples_scatter(d_off, d_rows, d_ts, d_vals, T_END, STEP, T, n_rows,
                                          mem_kind=g.ffi.GPR_MEM_DEVICE, n_series=n_rows)
    planes["device"] = _plane(eng, n_rows, T)
    import torch
    raw_t = torch.empty(n + 1, dtype=torch.int64, device="cuda")
    raw_v = torch.empty(n + 1, dtype=torch.float64, device="cuda")
    raw_t[1:], raw_v[1:] = d_ts, d_vals
    torch.cuda.synchronize()
    assert raw_t[1:].data_ptr() % 16 == 8
    stats["device, unaligned"] = eng.samples_scatter(d_off, d_rows, raw_t[1:], raw_v[1:], T_END, STEP, T, n_rows,
                                                     mem_kind=g.ffi.GPR_MEM_DEVICE, n_series=n_rows)
    planes["device, unaligned"] = _plane(eng, n_rows, T)
    for k in planes:
        assert np.array_equal(planes[k], planes["pageable"]), k
        assert stats[k] == stats["pageable"], (k, stats[k], stats["pageable"])
    # a spot check of the plane against the rule itself: each row's max over its in-window samples
    inw = (ts <= T_END * 1000) & (ts > (T_END - T * STEP) * 1000)
    assert stats["pageable"]["n_oow"] == int((~inw).sum())
    sidx = np.repeat(np.arange(n_rows), lengths)
    for s in rng.choice(np.flatnonzero(lengths), 20, replace=False):
        m = inw & (sidx == s) & ~np.isnan(vals)
        got = planes["pageable"][rows[s]].view(np.float32)
        assert np.nanmax(got) == vals[m].max() if m.any() else np.isnan(got).all()


def _ring(eng, P, G, T):
    u, p, _ = eng.resident_planes()
    return _read(eng, u, P * G, T), _read(eng, p, P * G, T)


@pytest.mark.parametrize("block_index", [False, True])
def test_daemon_timeline_matches_the_text_fed_ring(block_index):
    """two contexts run the same ticks — advance + text parse, advance + gpr_samples_scatter — into rings with a power
    plane; the rings wrap several times and stay bit-identical; with the block index deciding before the reindex is
    GPR_E_STATE; after it gpr_decide_resident equals the oracle on the ring's samples"""
    import gpu_pruner_b200 as g
    from oracle import oracle_c
    rng = np.random.default_rng(31 + block_index)
    P, G, T = 40, 2, 90
    a, b = _engine(), _engine()
    try:
        for e in (a, b):
            e.resident_init(P, G, T, power_plane=True, block_index=block_index)
        advanced = 0
        for tick in range(9):
            n_new = int(rng.integers(5, 40))
            advanced += n_new
            t_end = T_END + 100 * tick
            for e in (a, b):
                e.resident_advance(n_new)
            for plane, thr in ((0, 0.0), (1, THR)):
                offsets, rows, ts, vals = _random_batch(rng, 60, P * G, n_new, max_len=3 * n_new, window=n_new)
                ts += (t_end - T_END) * 1000
                if plane == 1:
                    vals = np.where(rng.random(len(vals)) < 0.5, rng.choice([149.999999, 150.0, 150.0000001, 80.0],
                                                                         len(vals)), vals)
                text, order = _render(offsets, rows, ts, vals)
                opens, closes = a.text_scan(text, slot=plane)
                sp = np.zeros(len(order), g.IdleEngine.SPAN_DTYPE)
                for i, o in enumerate(opens):
                    bg = int(o) + 12
                    sp[i]["begin"], sp[i]["end"], sp[i]["row"] = bg, int(closes[np.searchsorted(closes, bg)]) + 2, order[i]
                a.text_parse(sp, t_end, STEP, T, P * G, slot=plane, plane=plane, power_threshold=thr, resident=True,
                             window_seconds=n_new)
                b.samples_scatter(offsets, rows, ts, vals, t_end, STEP, T, P * G, plane=plane, power_threshold=thr,
                                  resident=True, window_seconds=n_new)
            ra, rb = _ring(a, P, G, T), _ring(b, P, G, T)
            assert a.resident_head() == b.resident_head()
            assert np.array_equal(ra[0], rb[0]) and np.array_equal(ra[1], rb[1]), tick
            dbits = np.zeros(2, np.uint32)
            cbits = np.zeros(2, np.uint32)
            smax = np.zeros((P, G), np.float32)
            kw = dict(power_threshold=THR, candidate_bits=cbits, series_max=smax, in_kind=g.ffi.GPR_MEM_HOST,
                      out_kind=g.ffi.GPR_MEM_HOST, resident=True)
            if block_index:
                with pytest.raises(g.GprError) as ei:
                    b.decide_ptr(None, P, G, T, dbits, **kw)
                assert ei.value.code == g.ffi.GPR_E_STATE
            b.resident_reindex()
            r = b.decide_ptr(None, P, G, T, dbits, **kw)
            want = oracle_c.decide(rb[0].view(np.float32).reshape(P, G, T), rb[1].view(np.float32).reshape(P, G, T),
                                   power_threshold=THR)
            assert np.array_equal(dbits[:2], want["decision_bits"]) and np.array_equal(cbits[:2], want["candidate_bits"])
            assert (r.n_series, r.n_candidates) == (want["n_series"], want["n_candidates"])
            assert kat.smax_equal(smax, want["series_max"])
        assert advanced > T   # the ring wrapped
    finally:
        a.close()
        b.close()


def test_c2_window_from_samples_decides_like_the_window(eng):
    """the C2 synthetic window (10,000 pods x 4 GPUs x 1,800 samples), every present cell a sample at its bucket's
    timestamp, scattered from the device into the context planes and decided with the power veto and the gates:
    bitmaps, counts and series_max equal deciding the synthetic planes directly, and the oracle"""
    import torch
    import gpu_pruner_b200 as g
    from oracle import oracle_c
    P, G, T, SEED = 10_000, 4, 1800, 7
    rows = P * G
    util = torch.empty((rows, T), dtype=torch.float32, device="cuda")
    power = torch.empty((rows, T), dtype=torch.float32, device="cuda")
    eng.synth_fill(SEED, 0, util, 0, P, G, T)
    eng.synth_fill(SEED, 1, power, 0, P, G, T)
    elig = torch.empty(P, dtype=torch.uint8, device="cuda")
    eng.synth_eligible(SEED, elig, 0, P)

    def decide(u, w):
        W = (P + 31) // 32
        out = [np.zeros(W, np.uint32), np.zeros(W, np.uint32), np.zeros((P, G), np.float32)]
        r = eng.decide_ptr(u, P, G, T, out[0], power=w, eligible=elig, power_threshold=THR, candidate_bits=out[1],
                           series_max=out[2], out_kind=g.ffi.GPR_MEM_HOST)
        return out, (r.n_series, r.n_candidates, r.n_decisions)

    direct = decide(util, power)
    for plane, src in ((0, util), (1, power)):
        present = ~torch.isnan(src)
        counts = present.sum(1)
        offsets = torch.zeros(rows + 1, dtype=torch.int64, device="cuda")
        offsets[1:] = torch.cumsum(counts, 0)
        r_idx, c_idx = present.nonzero(as_tuple=True)
        ts = T_END * 1000 - (T - 1 - c_idx).to(torch.int64) * STEP * 1000
        vals = src[r_idx, c_idx].to(torch.float64)
        r_ids = torch.arange(rows, dtype=torch.int32, device="cuda")
        torch.cuda.synchronize()   # the context's stream is not ordered with torch's (include/gpr.h)
        st = eng.samples_scatter(offsets, r_ids, ts, vals, T_END, STEP, T, rows, plane=plane,
                                 power_threshold=THR if plane else 0.0, mem_kind=g.ffi.GPR_MEM_DEVICE, n_series=rows)
        assert st["n_in"] == int(counts.sum()) and st["n_oow"] == 0
    tu, tw = eng.text_planes()
    got = decide(tu, tw)
    for k in range(3):
        assert np.array_equal(got[0][k].view(np.uint32), direct[0][k].view(np.uint32)), k
    assert got[1] == direct[1]
    want = oracle_c.decide(util.cpu().numpy().reshape(P, G, T), power.cpu().numpy().reshape(P, G, T),
                           eligible=elig.cpu().numpy(), power_threshold=THR, n_threads=os.cpu_count() or 1)
    assert np.array_equal(got[0][0], want["decision_bits"]) and np.array_equal(got[0][1], want["candidate_bits"])
    assert got[1] == (want["n_series"], want["n_candidates"], want["n_decisions"])
    assert kat.smax_equal(got[0][2], want["series_max"])


def _raw_scatter(eng, batch, grid_flags, n_rows, T, plane=0):
    import gpu_pruner_b200 as g
    grid = g.ffi.gpr_text_grid()
    grid.struct_size = C.sizeof(g.ffi.gpr_text_grid)
    grid.flags, grid.t_end, grid.window_seconds, grid.step = grid_flags, T_END, T * STEP, STEP
    grid.n_samples, grid.n_rows = T, n_rows
    return eng._lib.gpr_samples_scatter(eng.handle, C.byref(batch), C.byref(grid), plane, None)


def test_invalid_batches_leave_the_plane_untouched(eng):
    import torch
    import gpu_pruner_b200 as g
    rng = np.random.default_rng(41)
    T, n_rows = 60, 20
    offsets, rows, ts, vals = _random_batch(rng, 30, n_rows, T)
    eng.samples_scatter(offsets, rows, ts, vals, T_END, STEP, T, n_rows)
    before = _plane(eng, n_rows, T)
    assert (before != FILL).any()
    dev = {k: _torch_dev(v) for k, v in (("offsets", offsets.view(np.int64)), ("rows", rows.view(np.int32)),
                                          ("ts", ts), ("values", vals))}
    # an async decision enqueued before the failing calls completes at gpr_sync
    W = 1
    P_d, G_d = 4, 5
    dbits = torch.zeros(W, dtype=torch.int32, device="cuda")
    r_async = eng.decide_ptr(eng.text_planes()[0], P_d, G_d, T, dbits, blocking=False)

    def make(kind, offs, rws, struct_size=None):
        b = g.ffi.gpr_sample_batch()
        b.struct_size = C.sizeof(g.ffi.gpr_sample_batch) if struct_size is None else struct_size
        b.mem_kind = kind
        if kind == g.ffi.GPR_MEM_HOST:
            b.offsets, b.rows, b.ts_ms, b.values = offs.ctypes.data, rws.ctypes.data, ts.ctypes.data, vals.ctypes.data
        else:
            b.offsets, b.rows = offs.data_ptr(), rws.data_ptr()
            b.ts_ms, b.values = dev["ts"].data_ptr(), dev["values"].data_ptr()
        b.n_series = len(rows)
        return b

    bad_row = rows.copy()
    bad_row[7] = n_rows
    dec = offsets.copy()
    dec[5], dec[6] = offsets[6] + 1, offsets[6]
    start = offsets + np.uint64(1)
    keep = []
    cases = []
    for kind in (g.ffi.GPR_MEM_HOST, g.ffi.GPR_MEM_DEVICE):
        conv = (lambda a: a) if kind == g.ffi.GPR_MEM_HOST else \
            (lambda a: _torch_dev(a.view(np.int64) if a.dtype == np.uint64 else a.view(np.int32)))
        for name, offs, rws in (("row >= n_rows", offsets, bad_row), ("decreasing offsets", dec, rows),
                                ("offsets[0] != 0", start, rows)):
            o, r = conv(offs), conv(rws)
            keep.append((o, r))
            cases.append((f"{name} ({kind})", make(kind, o, r), g.ffi.GPR_E_INVALID, g.ffi.GPR_TEXT_FILL))
        o, r = conv(offsets), conv(rows)
        keep.append((o, r))
        cases.append((f"struct_size ({kind})", make(kind, o, r, struct_size=8), g.ffi.GPR_E_INVALID,
                      g.ffi.GPR_TEXT_FILL))
    for name, b, code, flags in cases:
        rc = _raw_scatter(eng, b, flags, n_rows, T)
        assert rc == code, (name, rc, eng._lib.gpr_last_error(eng.handle))
        assert np.array_equal(_plane(eng, n_rows, T), before), name
    # the resident ring without gpr_resident_init
    fresh = _engine()
    try:
        b = make(g.ffi.GPR_MEM_HOST, offsets, rows)
        assert _raw_scatter(fresh, b, g.ffi.GPR_TEXT_RESIDENT, n_rows, T) == g.ffi.GPR_E_STATE
    finally:
        fresh.close()
    eng.sync()
    assert r_async.n_decisions >= 0 and r_async.n_series >= 0
    want = eng.decide_ptr(eng.text_planes()[0], P_d, G_d, T, torch.zeros(W, dtype=torch.int32, device="cuda"))
    assert (r_async.n_series, r_async.n_candidates) == (want.n_series, want.n_candidates)
