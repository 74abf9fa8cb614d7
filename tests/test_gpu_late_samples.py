"""GPU: samples that reach the server late, on an H100.
  * gpr_resident_cols against the ring model of tests/ring_scripts.py: rings filled by gpr_append at several heads,
    both planes, every band edge, host and device outputs between guard words;
  * every error (no ring, plane 1 without a power plane, a bad plane, n_cols 0, a band longer than the ring, NULL out,
    a bad mem_kind) leaves the destination untouched;
  * decisions enqueued before the call keep their verdicts, on the context's stream and on a torch.cuda.Stream;
  * the re-ask recipe of INTEGRATION.md §5 through gpr_samples_scatter and gpr_chunks_scatter: each tick opens only its
    new buckets and merges (t_prev - L, t_now] with window_seconds = t_now - t_prev + L, on a server whose samples
    arrive up to L seconds after their timestamp (L a multiple of the step and not).  At every tick the unrolled ring
    equals a fresh full-window scatter of what the server holds then, bit for bit; with L = 0 it does not."""
import ctypes as C

import numpy as np
import pytest

import chunks_ref as CR
import ring_scripts as RS
from test_gpu_resident import decide, expected, same_verdict
from test_gpu_resident_remap import _async_on_ring, _engine, _model_ring
from test_ring_cols_emul import band_model

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")
GUARD = 0x5EC7AB1E


def _host_call(eng, plane, newer, n_cols, n_cells, kind=None, null=False):
    """the raw call into a host buffer between guard words: (rc, cells, guards intact)"""
    from gpu_pruner_b200 import ffi
    buf = np.full(n_cells + 2, GUARD, np.uint32)
    out = None if null else C.c_void_p(buf.ctypes.data + 4)
    rc = eng._lib.gpr_resident_cols(eng._h, plane, newer, n_cols, out, ffi.GPR_MEM_HOST if kind is None else kind)
    return rc, buf[1:-1].copy(), buf[0] == GUARD and buf[-1] == GUARD


def _device_call(eng, plane, newer, n_cols, n_cells):
    from gpu_pruner_b200 import ffi
    t = torch.full((n_cells + 2,), GUARD, dtype=torch.int32, device="cuda:0")
    rc = eng._lib.gpr_resident_cols(eng._h, plane, newer, n_cols, C.c_void_p(t.data_ptr() + 4), ffi.GPR_MEM_DEVICE)
    torch.cuda.synchronize()
    a = t.cpu().numpy().view(np.uint32)
    return rc, a[1:-1].copy(), a[0] == GUARD and a[-1] == GUARD


def _bands(T):
    out = {(0, 1), (0, T), (T - 1, 1), (1, T - 1), (0, max(1, T // 3)), (T // 2, T - T // 2), (3 % T, 1)}
    return sorted((n, c) for n, c in out if c >= 1 and n + c <= T)


@pytest.mark.parametrize("T", [1, 4, 65, 1800])
def test_band_equals_the_ring_model(T):
    rng = np.random.default_rng(T)
    eng = _engine()
    try:
        for flags in (0, 1, 3):
            for _ in range(3):   # a new ring at a new head each time
                m = _model_ring(rng, eng, 7, 3, T, flags)
                for plane, cells in enumerate(m.planes):
                    for newer, n_cols in _bands(T):
                        want = band_model(cells, m.head, newer, n_cols)
                        where = f"T={T} flags={flags} head={m.head} plane={plane} newer={newer} n_cols={n_cols}"
                        rc, got, guards = _host_call(eng, plane, newer, n_cols, want.size)
                        assert rc == 0 and guards and np.array_equal(got.reshape(want.shape), want), where
                        rc, got, guards = _device_call(eng, plane, newer, n_cols, want.size)
                        assert rc == 0 and guards and np.array_equal(got.reshape(want.shape), want), where
                        band = eng.resident_cols(plane, newer, n_cols)
                        assert np.array_equal(band.view(np.uint32), want), where
    finally:
        eng.close()


def test_errors_leave_the_destination_untouched():
    from gpu_pruner_b200 import ffi
    eng = _engine()
    try:
        for call in (lambda: _host_call(eng, 0, 0, 1, 8), lambda: _device_call(eng, 0, 0, 1, 8)):
            rc, got, guards = call()
            assert rc == ffi.GPR_E_STATE and guards and (got == GUARD).all()
        assert "no resident window" in eng._lib.gpr_last_error(eng._h).decode()
        eng.resident_init(5, 2, 16)   # no power plane
        n = 10 * 16
        bad = [(1, 0, 1, None, ffi.GPR_E_STATE), (2, 0, 1, None, ffi.GPR_E_INVALID), (-1, 0, 1, None, ffi.GPR_E_INVALID),
               (0, 0, 0, None, ffi.GPR_E_INVALID), (0, 0, 17, None, ffi.GPR_E_INVALID),
               (0, 16, 1, None, ffi.GPR_E_INVALID), (0, 0xFFFFFFFF, 2, None, ffi.GPR_E_INVALID),
               (0, 1, 0xFFFFFFFF, None, ffi.GPR_E_INVALID), (0, 0, 4, 2, ffi.GPR_E_INVALID),
               (0, 0, 4, -1, ffi.GPR_E_INVALID)]
        for plane, newer, n_cols, kind, code in bad:
            rc, got, guards = _host_call(eng, plane, newer, n_cols, n, kind)
            assert rc == code and guards and (got == GUARD).all(), (plane, newer, n_cols, kind)
        rc, _, _ = _host_call(eng, 0, 0, 4, n, null=True)
        assert rc == ffi.GPR_E_INVALID
        rc, got, guards = _device_call(eng, 1, 0, 4, n)
        assert rc == ffi.GPR_E_STATE and guards and (got == GUARD).all()
        rc, got, guards = _host_call(eng, 0, 0, 16, n)
        assert rc == 0 and guards and (got == RS.NO_SAMPLE).all()   # a fresh ring: no sample anywhere
    finally:
        eng.close()


@pytest.mark.parametrize("stream", ["context", "caller"])
def test_decisions_enqueued_before_the_call_stay_pending(stream):
    import kat
    rng = np.random.default_rng(37)
    s = torch.cuda.Stream() if stream == "caller" else None
    eng = _engine(stream=s.cuda_stream if s is not None else None)
    try:
        m = _model_ring(rng, eng, 300, 4, 1800, 3)
        exp = expected(m)
        W = (m.P + 31) // 32
        outs = []
        for _ in range(3):
            o = (eng.host_array((W,), np.uint32), eng.host_array((W,), np.uint32), eng.host_array((m.P, m.G), np.float32))
            outs.append((o, _async_on_ring(eng, m, *o)))
        for plane in (0, 1):
            band = eng.resident_cols(plane, 5, 90)
            assert np.array_equal(band.view(np.uint32), band_model(m.planes[plane], m.head, 5, 90))
        eng.sync()
        for (db, cb, smax), r in outs:
            assert np.array_equal(db, exp["decision_bits"]) and np.array_equal(cb, exp["candidate_bits"])
            assert (r.n_series, r.n_candidates) == (exp["n_series"], exp["n_candidates"])
            assert kat.smax_equal(smax, exp["series_max"])
        assert same_verdict(decide(eng, m), exp) is None
        if s is not None:
            s.synchronize()
    finally:
        eng.close()


# ---- the re-ask recipe through the sample and chunk merges ---------------------------------------------------------
T0 = 1_700_000_000
STEP, T, SLICE = 10, 48, 30


class LateStore:
    """samples of `rows` series, every 4 s with jitter, each arriving `lag` seconds after its timestamp"""

    def __init__(self, rng, rows, t_lo, t_hi, max_lag):
        ts, row, lag, val = [], [], [], []
        for r in range(rows):
            t = t_lo + int(rng.integers(0, 4))
            while t <= t_hi:
                ts.append(t * 1000 + int(rng.integers(0, 1000)))
                row.append(r)
                lag.append(float(rng.uniform(0, max_lag)) if rng.random() < 0.5 else 0.0)
                val.append(float(rng.choice([0.0, rng.uniform(0, 100)])))
                t += 4
        self.ts, self.row = np.array(ts, np.int64), np.array(row, np.int64)
        self.arrival = self.ts / 1000.0 + np.array(lag)
        self.val, self.rows = np.array(val, np.float64), rows

    def answer(self, lo, hi, now):
        """what the server returns at `now` for (lo, hi]: CSR by row, every row a series (empty ones included)"""
        keep = (self.ts > lo * 1000) & (self.ts <= hi * 1000) & (self.arrival <= now)
        order = np.lexsort((self.ts[keep], self.row[keep]))
        r, t, v = self.row[keep][order], self.ts[keep][order], self.val[keep][order]
        offsets = np.concatenate([[0], np.cumsum(np.bincount(r, minlength=self.rows))]).astype(np.uint64)
        return offsets, t, v

    def merge(self, eng, plane, how, lo, hi, now):
        offsets, t, v = self.answer(lo, hi, now)
        rows = np.arange(self.rows, dtype=np.uint32)
        kw = dict(window_seconds=hi - lo, plane=plane, resident=True, fill=False)
        if how == "samples":
            eng.samples_scatter(offsets, rows, t, v, hi, STEP, T, self.rows, **kw)
            return
        chunks = [CR.split(t[int(offsets[s]):int(offsets[s + 1])], v[int(offsets[s]):int(offsets[s + 1])])
                  for s in range(self.rows)]
        sc, cb, data = CR.batch(chunks)
        eng.chunks_scatter(sc, rows, cb, data, hi, STEP, T, self.rows, **kw)


@pytest.mark.parametrize("how", ["samples", "chunks"])
@pytest.mark.parametrize("L,max_lag", [(30, 30), (25, 25), (0, 25)])
def test_reask_timeline_equals_a_fresh_scatter(how, L, max_lag):
    rng = np.random.default_rng(L * 7 + max_lag + (how == "chunks"))
    P, G = 6, 2
    rows = P * G
    n_ticks = 24
    t_first = T0
    store = LateStore(rng, rows, t_first - T * STEP - 60, t_first + n_ticks * SLICE, max_lag)
    eng, fresh = _engine(), _engine()
    differed = 0
    try:
        eng.resident_init(P, G, T, power_plane=True)
        for plane in (0, 1):
            store.merge(eng, plane, how, t_first - T * STEP, t_first, t_first)
        t_prev = t_first
        for k in range(1, n_ticks + 1):
            t_now = t_first + k * SLICE
            eng.resident_advance(SLICE // STEP)
            for plane in (0, 1):
                store.merge(eng, plane, how, t_prev - L, t_now, t_now)
            fresh.resident_init(P, G, T, power_plane=True)
            for plane in (0, 1):
                store.merge(fresh, plane, how, t_now - T * STEP, t_now, t_now)
            for plane in (0, 1):
                got = eng.resident_cols(plane, 0, T).view(np.uint32)
                want = fresh.resident_cols(plane, 0, T).view(np.uint32)
                if L >= max_lag:
                    assert np.array_equal(got, want), (how, L, k, plane)
                differed += int((got != want).sum())
            t_prev = t_now
        if L < max_lag:
            assert differed > 0   # the scenario reaches the gap the re-ask closes
    finally:
        eng.close()
        fresh.close()
