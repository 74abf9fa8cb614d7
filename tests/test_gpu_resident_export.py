"""gpr_resident_export through libgpr.so on an H100: the resident ring encoded as Prometheus XOR chunks on the GPU, and
restored from them through gpr_chunks_scatter.

  * bytes: the C2 ring (10,000 x 4 x 1,800 with power) exported byte for byte as tests/cpp/chunks_encode.cpp, the C++
    mirror of Prometheus' appender, encodes the same (ts_ms, value) lists, for both planes;
  * round trip: rings built by gpr_append at random heads, exported and restored into a fresh context, both planes,
    with and without GPR_F_BLOCK_INDEX: the unrolled ring is bit-identical (every NaN as the fill), and
    gpr_decide_resident gives identical bitmaps, counters, series_max and idle_slots;
  * a restore into a reshaped ring through `rows` equals gpr_resident_remap with the same map;
  * a daemon timeline: a snapshot at tick k, a restart some ticks later that advances by the gap and scatters only
    the gap; from then on the running ring and the restored one are identical at every tick, and equal a fresh
    full-window scatter;
  * the export leaves the ring bytes, the head, the index state and pending _async results untouched, on the
    context's own stream and on a caller-owned one;
  * every error code, with the destination untouched; host (pageable and pinned) and device outputs."""
import ctypes as C

import numpy as np
import pytest

import export_ref as X
import ring_scripts as RS
from test_gpu_resident import decide, expected, same_verdict
from test_remap_emul import NONE, remap_model

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

T_END, STEP = 1_700_000_000, 10


def _engine(**kw):
    import gpu_pruner_b200 as g
    if not torch.cuda.is_available():
        pytest.fail("-m gpu tests need a CUDA device; the engine has no CPU fallback")
    return g.IdleEngine(device=0, **kw)


def _read_ring(eng, rows, T, n_planes):
    from gpu_pruner_b200 import ffi
    u, p, ld = eng.resident_planes()
    assert ld == T
    out = []
    for ptr in (u, p)[:n_planes]:
        a = np.empty((rows, T), np.uint32)
        eng.memcpy(a, ptr, a.nbytes, ffi.GPR_MEM_HOST, ffi.GPR_MEM_DEVICE)
        out.append(a)
    return out


def _model_ring(rng, eng, P, G, T, flags):
    """a ring filled by gpr_append at random heads, and its model (tests/ring_scripts.py)"""
    m = RS.Ring(P, G, T, flags)
    eng.resident_init(P, G, T, power_plane=bool(flags & 1), block_index=bool(flags & 2))
    for _ in range(int(rng.integers(1, 4))):
        n = int(rng.integers(1, 2 * T + 2))
        util = RS._mixed(rng, 0, m.rows, n)
        power = RS._mixed(rng, 1, m.rows, n) if flags & 1 and rng.random() < 0.8 else None
        m.append(n, util, power)
        eng.append(util.view(np.float32), None if power is None else power.view(np.float32))
    assert eng.resident_head() == m.head
    return m


def _grid(T, t_end=T_END, step=STEP, window_seconds=None, thr=0.0):
    from gpu_pruner_b200 import ffi
    g = ffi.gpr_text_grid()
    g.struct_size = C.sizeof(ffi.gpr_text_grid)
    g.t_end, g.step, g.n_samples = t_end, step, T
    g.window_seconds = T * step if window_seconds is None else window_seconds
    g.power_threshold = thr
    return g


def _raw_export(eng, grid, plane, M, arrays, mem_kind, caps=None):
    """gpr_resident_export into four caller arrays (numpy or CUDA tensors) -> (rc, the struct)"""
    from gpu_pruner_b200 import ffi
    o = ffi.gpr_chunk_export()
    o.struct_size = C.sizeof(ffi.gpr_chunk_export)
    o.mem_kind = mem_kind

    def ptr(a):
        if a is None:
            return None
        return a.data_ptr() if hasattr(a, "data_ptr") else (a.ctypes.data if a.size else None)
    o.series_chunks, o.rows, o.chunk_bytes, o.data = (ptr(a) for a in arrays)
    sizes = [(a.numel() if hasattr(a, "numel") else a.size) for a in arrays]
    o.cap_series, o.cap_chunks, o.cap_bytes = caps if caps is not None else (sizes[1], sizes[2] - 1, sizes[3])
    rc = eng._lib.gpr_resident_export(eng._h, C.byref(grid), plane, M, C.byref(o))
    return rc, o


def _restore(eng, out, P, G, T, flags, rows=None):
    """a fresh ring of [P][G][T] restored from exports {plane: Engine.resident_export(...)} (rows: per exported series
    of each plane, its new row or NONE), reindexed"""
    eng.resident_init(P, G, T, power_plane=bool(flags & 1), block_index=bool(flags & 2))
    for pl, ex in out.items():
        sc, rr, cb, data = ex["series_chunks"], ex["rows"], ex["chunk_bytes"], ex["data"]
        if rows is not None:
            sc, rr, cb, data = _keep(ex, rows[pl])
        gr = dict(ex["grid"])
        eng.chunks_scatter(sc, rr, cb, data, gr["t_end"], gr["step"], gr["T"], P * G, plane=pl, resident=True,
                           window_seconds=gr["window_seconds"], power_threshold=gr["power_threshold"])
    eng.resident_reindex()


def _keep(ex, new_rows):
    """the export's series whose new row is not NONE, fed to those rows"""
    sc, cb, data = ex["series_chunks"], ex["chunk_bytes"], ex["data"]
    keep = np.nonzero(new_rows != NONE)[0]
    chunks, counts = [], []
    for s in keep:
        c0, c1 = int(sc[s]), int(sc[s + 1])
        chunks += [data[int(cb[c]):int(cb[c + 1])] for c in range(c0, c1)]
        counts.append(c1 - c0)
    sc2 = np.concatenate([[0], np.cumsum(counts)]).astype(np.uint64)
    cb2 = np.concatenate([[0], np.cumsum([len(c) for c in chunks])]).astype(np.uint64)
    data2 = np.concatenate(chunks).astype(np.uint8) if chunks else np.zeros(0, np.uint8)
    return sc2, new_rows[keep].astype(np.uint32), cb2, data2


def _unrolled(planes, head):
    return [X.canonical(X.unroll(p, head)) for p in planes]


def _verdicts(eng, m):
    return decide(eng, m), decide(eng, m, early=True)


def _same_outputs(a, b, where):
    """two engines' gpr_decide_resident outputs: bitmaps, counters, series_max (bits) and idle_slots"""
    for x, y in zip(a, b):
        assert same_verdict(x, y) is None, where
    assert np.array_equal(a[0]["series_max"].view(np.uint32), b[0]["series_max"].view(np.uint32)), where
    assert np.array_equal(a[1]["idle_slots"], b[1]["idle_slots"]), where


def _export_planes(eng, n_planes, M=120):
    return {pl: eng.resident_export(T_END, STEP, plane=pl, max_per_chunk=M, power_threshold=RS.THR if pl else 0.0)
            for pl in range(n_planes)}


# ---- 1. bytes --------------------------------------------------------------------------------------------------
def test_c2_ring_byte_equal_to_the_reference_encoder():
    P, G, T = 10_000, 4, 1800
    eng = _engine()
    try:
        eng.resident_init(P, G, T, power_plane=True)
        u, p, _ = eng.resident_planes()
        eng.synth_fill(0x5EED0002, 0, u, 0, P, G, T)
        eng.synth_fill(0x5EED0002, 1, p, 0, P, G, T)
        torch.cuda.synchronize()
        eng.resident_advance(777)     # a head inside the ring: the newest 777 buckets hold no sample
        head = eng.resident_head()
        planes = _read_ring(eng, P * G, T, 2)
        for pl in (0, 1):
            got = eng.resident_export(T_END, STEP, plane=pl)
            sc, rows, cb, data, n = X.export_native(planes[pl], head, T_END, STEP, 120)
            assert got["n_samples"] == n > 0
            assert np.array_equal(got["series_chunks"], sc) and np.array_equal(got["rows"], rows), pl
            assert np.array_equal(got["chunk_bytes"], cb), pl
            assert np.array_equal(got["data"], data), pl
            assert got["data"].size < 2.0 * n      # well under the 4 B per cell of the plane
    finally:
        eng.close()


# ---- 2. round trip ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("flags", [0, 1, 2, 3], ids=["util", "power", "index", "power+index"])
def test_round_trip_into_a_fresh_context(flags):
    rng = np.random.default_rng(200 + flags)
    a, b = _engine(), _engine()
    try:
        for trial in range(6):
            P, G = int(rng.integers(1, 60)), int(rng.integers(1, 5))
            T = int(rng.choice([1, 2, 63, 64, 65, 120, 121, 240, 1800]))
            m = _model_ring(rng, a, P, G, T, flags)
            M = int(rng.choice([1, 2, 119, 120, 65535]))
            out = _export_planes(a, len(m.planes), M)
            _restore(b, out, P, G, T, flags)
            want = _unrolled(m.planes, m.head)
            got = _read_ring(b, m.rows, T, len(m.planes))
            assert b.resident_head() == 0
            for pl in range(len(want)):
                assert np.array_equal(got[pl], want[pl]), (flags, trial, pl)
            r = RS.Ring(P, G, T, flags)
            r.planes = got
            _same_outputs(_verdicts(a, m), _verdicts(b, r), (flags, trial))
            assert same_verdict(decide(b, r), expected(m)) is None
    finally:
        a.close()
        b.close()


# ---- 3. a reshaped restore -------------------------------------------------------------------------------------
def test_restore_through_rows_equals_the_remap():
    rng = np.random.default_rng(31)
    a, b = _engine(), _engine()
    try:
        P0, G0, T = 40, 3, 130
        for kind in range(3):
            m = _model_ring(rng, a, P0, G0, T, 3)
            out = _export_planes(a, 2)
            if kind == 0:   # grow and widen
                P, G = P0 + 9, G0 + 1
                src = np.full((P, G), NONE, np.uint32)
                src[:P0, :G0] = np.arange(P0 * G0, dtype=np.uint32).reshape(P0, G0)
            elif kind == 1:  # compaction
                kept = np.sort(rng.choice(P0, P0 // 2, replace=False))
                P, G = kept.size, G0
                src = np.arange(P0 * G0, dtype=np.uint32).reshape(P0, G0)[kept]
            else:            # a permutation with rows dropped
                P, G = P0, G0
                src = rng.permutation(P0 * G0).astype(np.uint32)
                src[rng.random(src.size) < 0.2] = NONE
            src = np.ascontiguousarray(src, np.uint32).ravel()
            new_of_old = np.full(P0 * G0, NONE, np.uint32)
            new_of_old[src[src != NONE]] = np.nonzero(src != NONE)[0]
            rows = {pl: new_of_old[out[pl]["rows"]] for pl in out}
            _restore(b, out, P, G, T, 3, rows=rows)
            a.resident_remap(P, G, src)
            remapped = remap_model(m.planes, src)
            assert all(np.array_equal(x, y) for x, y in zip(_read_ring(a, P * G, T, 2), remapped))
            want = _unrolled(remapped, m.head)
            got = _read_ring(b, P * G, T, 2)
            for pl in (0, 1):
                assert np.array_equal(got[pl], want[pl]), (kind, pl)
            mr = RS.Ring(P, G, T, 3)
            mr.planes, mr.head = remapped, m.head
            r = RS.Ring(P, G, T, 3)
            r.planes = got
            _same_outputs(_verdicts(a, mr), _verdicts(b, r), kind)
    finally:
        a.close()
        b.close()


# ---- 4. a daemon timeline ----------------------------------------------------------------------------------------
def _samples(rng, rows, t_lo_ms, t_hi_ms, step_ms):
    """a scrape per row every ~step_ms in (t_lo_ms, t_hi_ms], some rows silent: CSR (offsets, rows, ts, values)"""
    ts_all, v_all, counts = [], [], []
    for r in range(rows):
        if r % 9 == 4:
            counts.append(0)
            continue
        ts = np.arange(t_lo_ms + 1 + (r * 37) % step_ms, t_hi_ms + 1, step_ms, dtype=np.int64)
        v = rng.integers(0, 101, ts.size).astype(np.float64)
        v[rng.random(ts.size) < 0.1] = np.nan
        if r % 5 == 1:
            v = np.where(rng.random(ts.size) < 0.5, 0.0, v)
        ts_all.append(ts)
        v_all.append(v)
        counts.append(ts.size)
    return (np.concatenate([[0], np.cumsum(counts)]).astype(np.uint64), np.arange(rows, dtype=np.uint32),
            np.concatenate(ts_all), np.concatenate(v_all))


def test_daemon_timeline_restart_from_a_snapshot():
    rng = np.random.default_rng(41)
    P, G, T, step, tick = 30, 2, 240, 1, 20        # a 240 s window, a tick every 20 s
    rows = P * G
    t0 = T_END
    history = _samples(rng, rows, (t0 - T * step - 600) * 1000, (t0 + 20 * tick) * 1000, 7_000)
    off, rr, ts, vals = history
    row_of = np.repeat(np.arange(rows), np.diff(off).astype(np.int64))

    def between(lo_s, hi_s):
        """the history's samples with lo < ts <= hi (seconds)"""
        keep = (ts > lo_s * 1000) & (ts <= hi_s * 1000)
        counts = np.bincount(row_of[keep], minlength=rows)
        return np.concatenate([[0], np.cumsum(counts)]).astype(np.uint64), rr, ts[keep], vals[keep]

    def scatter(eng, lo_s, hi_s, resident=True):
        o, r_, t_, v_ = between(lo_s, hi_s)
        eng.samples_scatter(o, r_, t_, v_, hi_s, step, T, rows, window_seconds=hi_s - lo_s, resident=resident,
                            fill=not resident)

    run, res, fresh = _engine(), _engine(), _engine()
    try:
        run.resident_init(P, G, T, block_index=True)
        scatter(run, t0 - T * step, t0)
        run.resident_reindex()
        k, gap = 3, 4
        snapshot = None
        for i in range(1, 15):
            t = t0 + i * tick
            run.resident_advance(tick // step)
            scatter(run, t - tick, t)
            run.resident_reindex()
            if i == k:
                snapshot = run.resident_export(t, step, window_seconds=T * step)
            if i == k + gap:   # the restart: restore, advance by the gap, query only the gap
                t_snap = t0 + k * tick
                res.resident_init(P, G, T, block_index=True)
                s = snapshot
                res.chunks_scatter(s["series_chunks"], s["rows"], s["chunk_bytes"], s["data"], t_snap, step, T, rows,
                                   window_seconds=T * step, resident=True)
                res.resident_advance((t - t_snap) // step)
                scatter(res, t_snap, t)
                res.resident_reindex()
            elif i > k + gap:
                res.resident_advance(tick // step)
                scatter(res, t - tick, t)
                res.resident_reindex()
            if i >= k + gap:
                a = X.canonical(X.unroll(_read_ring(run, rows, T, 1)[0], run.resident_head()))
                b = X.canonical(X.unroll(_read_ring(res, rows, T, 1)[0], res.resident_head()))
                assert np.array_equal(a, b), i
                scatter(fresh, t - T * step, t, resident=False)
                plane = np.empty((rows, T), np.uint32)
                fresh.memcpy(plane, fresh.text_planes()[0], plane.nbytes, 0, 1)
                assert np.array_equal(a, plane), i
                _same_outputs(_verdicts(run, _as_ring(run, P, G, T)), _verdicts(res, _as_ring(res, P, G, T)), i)
    finally:
        run.close()
        res.close()
        fresh.close()


def _as_ring(eng, P, G, T):
    r = RS.Ring(P, G, T, 2)
    r.planes = _read_ring(eng, P * G, T, 1)
    r.head = eng.resident_head()
    return r


# ---- 5. the export changes nothing --------------------------------------------------------------------------------
def _async_on_ring(eng, m, db, cb, smax):
    u, p, _ = eng.resident_planes()
    return eng.decide_ptr(u, m.P, m.G, m.T, db, power=p if len(m.planes) > 1 else None, candidate_bits=cb,
                          series_max=smax, power_threshold=RS.THR if len(m.planes) > 1 else 0.0, in_kind=1,
                          out_kind=0, blocking=False)


@pytest.mark.parametrize("stream", ["context", "caller"])
def test_export_leaves_ring_head_index_and_pending_results(stream):
    import kat
    import gpu_pruner_b200 as g
    rng = np.random.default_rng(51)
    s = torch.cuda.Stream() if stream == "caller" else None
    eng = _engine(stream=s.cuda_stream if s is not None else None)
    try:
        m = _model_ring(rng, eng, 300, 4, 1800, 3)
        exp = expected(m)
        before = _read_ring(eng, m.rows, m.T, 2)
        W = (m.P + 31) // 32
        outs = []
        for _ in range(3):
            o = (eng.host_array((W,), np.uint32), eng.host_array((W,), np.uint32), eng.host_array((m.P, m.G), np.float32))
            outs.append((o, _async_on_ring(eng, m, *o)))
        ex = _export_planes(eng, 2)
        eng.sync()
        for (db, cb, smax), r in outs:
            assert np.array_equal(db, exp["decision_bits"]) and np.array_equal(cb, exp["candidate_bits"])
            assert (r.n_series, r.n_candidates) == (exp["n_series"], exp["n_candidates"])
            assert kat.smax_equal(smax, exp["series_max"])
        assert all(np.array_equal(x, y) for x, y in zip(before, _read_ring(eng, m.rows, m.T, 2)))
        assert eng.resident_head() == m.head and ex[0]["n_samples"] > 0
        assert same_verdict(decide(eng, m), exp) is None      # the index is current and unchanged
        # a stale index stays stale through an export
        eng.samples_scatter([0, 1], [0], [T_END * 1000], [55.0], T_END, 1, m.T, m.rows, resident=True,
                            window_seconds=1)
        eng.resident_export(T_END, STEP)
        with pytest.raises(g.GprError) as ei:
            decide(eng, m)
        assert ei.value.code == g.ffi.GPR_E_STATE
        if s is not None:
            s.synchronize()
    finally:
        eng.close()


# ---- 6, 7. errors, and where the outputs live ---------------------------------------------------------------------
def test_errors_leave_the_destination_untouched():
    from gpu_pruner_b200 import ffi
    rng = np.random.default_rng(61)
    eng = _engine()
    try:
        sentinel = (np.full(64, 7, np.uint64), np.full(63, 7, np.uint32), np.full(1000, 7, np.uint64),
                    np.full(20000, 7, np.uint8))
        arrays = tuple(a.copy() for a in sentinel)

        def untouched():
            return all(np.array_equal(a, b) for a, b in zip(arrays, sentinel))

        rc, o = _raw_export(eng, _grid(65), 0, 120, arrays, ffi.GPR_MEM_HOST)
        assert rc == ffi.GPR_E_STATE and untouched()              # no resident window
        m = _model_ring(rng, eng, 21, 3, 65, 0)
        rc, _ = _raw_export(eng, _grid(65), 1, 120, arrays, ffi.GPR_MEM_HOST)
        assert rc == ffi.GPR_E_STATE and untouched()              # no power plane
        bad = [(_grid(64), 0, 120, ffi.GPR_MEM_HOST), (_grid(65, step=0), 0, 120, ffi.GPR_MEM_HOST),
               (_grid(65, step=-10), 0, 120, ffi.GPR_MEM_HOST), (_grid(65), 0, 0, ffi.GPR_MEM_HOST),
               (_grid(65), 0, 65536, ffi.GPR_MEM_HOST), (_grid(65), 2, 120, ffi.GPR_MEM_HOST),
               (_grid(65), 0, 120, 5)]
        for k, (gr, pl, M, kind) in enumerate(bad):
            rc, _ = _raw_export(eng, gr, pl, M, arrays, kind)
            assert rc == ffi.GPR_E_INVALID and untouched(), k
        gr = _grid(65)
        gr.struct_size = 8
        assert _raw_export(eng, gr, 0, 120, arrays, ffi.GPR_MEM_HOST)[0] == ffi.GPR_E_INVALID and untouched()
        o = ffi.gpr_chunk_export()
        o.struct_size = 12
        assert eng._lib.gpr_resident_export(eng._h, C.byref(_grid(65)), 0, 120, C.byref(o)) == ffi.GPR_E_INVALID
        # the size protocol: one short of any need -> GPR_E_CAPACITY, the true counts, nothing written
        want = eng.resident_export(T_END, STEP, max_per_chunk=7)
        ns, nc, nb = want["rows"].size, want["chunk_bytes"].size - 1, want["data"].size
        assert ns <= 63 and nc < 1000 and nb <= 20000
        for caps in ((ns - 1, nc, nb), (ns, nc - 1, nb), (ns, nc, nb - 1), (0, 0, 0)):
            rc, o = _raw_export(eng, _grid(65), 0, 7, arrays, ffi.GPR_MEM_HOST, caps=caps)
            assert rc == ffi.GPR_E_CAPACITY and untouched(), caps
            assert (o.n_series, o.n_chunks, o.n_bytes, o.n_samples) == (ns, nc, nb, want["n_samples"])
        assert m.rows == 63
    finally:
        eng.close()


@pytest.mark.parametrize("where", ["pageable", "pinned", "device"])
def test_host_pinned_and_device_outputs(where):
    from gpu_pruner_b200 import ffi
    rng = np.random.default_rng(71)
    eng = _engine()
    try:
        m = _model_ring(rng, eng, 50, 4, 300, 1)
        for pl in (0, 1):
            want = eng.resident_export(T_END, STEP, plane=pl, max_per_chunk=50)
            sc, rows, cb, data, n = X.export(m.planes[pl], m.head, T_END, STEP, 50)
            assert all(np.array_equal(x, y) for x, y in zip((want["series_chunks"], want["rows"], want["chunk_bytes"],
                                                             want["data"]), (sc, rows, cb, data)))
            sizes = (sc.size + 3, rows.size + 3, cb.size + 3, data.size + 5)   # room to spare, left as it was
            dtypes = (np.uint64, np.uint32, np.uint64, np.uint8)
            if where == "device":
                tdt = (torch.int64, torch.int32, torch.int64, torch.uint8)
                arrays = tuple(torch.full((s,), 7, dtype=t, device="cuda:0") for s, t in zip(sizes, tdt))
                torch.cuda.synchronize()
                kind = ffi.GPR_MEM_DEVICE
            elif where == "pinned":
                arrays = tuple(eng.host_array((s,), d) for s, d in zip(sizes, dtypes))
                for a in arrays:
                    a[:] = 7
                kind = ffi.GPR_MEM_HOST
            else:
                arrays = tuple(np.full(s, 7, d) for s, d in zip(sizes, dtypes))
                kind = ffi.GPR_MEM_HOST
            rc, o = _raw_export(eng, _grid(300, thr=RS.THR if pl else 0.0), pl, 50, arrays, kind)
            assert rc == ffi.GPR_OK
            host = [a.cpu().numpy() if where == "device" else np.asarray(a) for a in arrays]
            for h, w, d in zip(host, (sc, rows, cb, data), dtypes):
                h = h.view(d)
                assert np.array_equal(h[:w.size], w) and np.all(h[w.size:] == 7), (where, pl)
            assert (o.n_series, o.n_chunks, o.n_bytes, o.n_samples) == (rows.size, cb.size - 1, data.size, n)
    finally:
        eng.close()
