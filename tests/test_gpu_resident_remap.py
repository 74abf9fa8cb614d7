"""gpr_resident_remap through libgpr.so on an H100: the resident ring takes a new [P][G] shape and keeps its history.

  * ring model: rings built by gpr_append at random heads, remapped with random maps (grown, widened, shrunk,
    permuted, compacted, rows without a source) from host and device memory; the planes and the head equal the
    model (tests/test_remap_emul.py's remap_model) bit for bit, and gpr_decide_resident, on the block index and on
    the planes, with series_max, with idle_slots, and with a `sum by` table on the new shape, equals the oracle on
    the model's unrolled window (the index is read through those verdicts and series_max);
  * order: decisions enqueued before a remap read the old ring and retire at the next gpr_sync with its verdicts,
    on the context's stream and on a caller-owned torch stream;
  * failure: bad maps and no resident window return their codes, the ring is byte-identical, earlier pending results
    retire, and a stale index stays refused until gpr_resident_reindex;
  * an integrator's timeline through gpr_samples_scatter(GPR_TEXT_RESIDENT): pods join beyond the head-room, a pod
    gains a third slot, departed pods are compacted away, and after every tick the unrolled ring equals a fresh
    GPR_TEXT_FILL scatter of that tick's whole window with the same row layout, and the verdicts the oracle's;
  * the C2 shape (10,000 x 4 x 1,800 with power and index) widened to G = 5 and grown by 25 %."""
import os
import random

import numpy as np
import pytest

import groups_ref as GR
import ring_scripts as RS
from test_gpu_resident import decide, expected, same_verdict
from test_remap_emul import G0, NONE, P0, first_bad, make_map, remap_model
from test_resident_ticks import _series

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")


def _engine(**kw):
    import gpu_pruner_b200 as g
    if not torch.cuda.is_available():
        pytest.fail("-m gpu tests need a CUDA device; the engine has no CPU fallback")
    return g.IdleEngine(device=0, **kw)


def _read_ring(eng, rows, T, n_planes):
    from gpu_pruner_b200 import ffi
    u, p, ld = eng.resident_planes()
    assert ld == T and (p is not None) == (n_planes > 1)
    out = []
    for ptr in (u, p)[:n_planes]:
        a = np.empty((rows, T), np.uint32)
        eng.memcpy(a, ptr, a.nbytes, ffi.GPR_MEM_HOST, ffi.GPR_MEM_DEVICE)
        out.append(a)
    return out


def _model_ring(rng, eng, P, G, T, flags):
    """a ring filled by gpr_append at random heads, and its model"""
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


def _remapped(m, P, G, src):
    n = RS.Ring(P, G, m.T, m.flags)
    n.planes = remap_model(m.planes, src)
    n.head = m.head
    return n


def _check_ring(eng, m, where):
    got = _read_ring(eng, m.rows, m.T, len(m.planes))
    assert eng.resident_head() == m.head, where
    for pl, (a, b) in enumerate(zip(got, m.planes)):
        if not np.array_equal(a, b):
            r, t = np.argwhere(a != b)[0]
            raise AssertionError(f"{where}: plane {pl} row {r} position {t}: {a[r, t]:#010x} != {b[r, t]:#010x}")


def _check_verdicts(eng, m, rng, where):
    exp = expected(m)
    for early in (False, True):
        bad = same_verdict(decide(eng, m, early=early), exp)
        assert bad is None, (where, early, bad)
    # a `sum by` table on the new shape
    if m.G > 1:
        table = GR.random_table(rng, m.P, m.G)
        power = m.window(1) if len(m.planes) > 1 else None
        thr = RS.THR if power is not None else 0.0
        want = GR.decide(m.window(0), power, thr, table)
        W, MW = (m.P + 31) // 32, (m.G + 31) // 32
        db, cb, isl = np.zeros(W, np.uint32), np.zeros(W, np.uint32), np.zeros(m.P * MW, np.uint32)
        r = eng.decide_ptr(None, m.P, m.G, m.T, db, candidate_bits=cb, power_threshold=thr, groups=table,
                           idle_slots=isl, in_kind=0, out_kind=0, resident=True)
        assert np.array_equal(db, want["decision_bits"]) and np.array_equal(cb, want["candidate_bits"]), where
        assert (r.n_series, r.n_candidates) == (want["n_series"], want["n_candidates"]), where
        assert np.array_equal(isl.reshape(m.P, MW), want["idle_slots"]), where


def _random_map(rng, P0, G0):
    """a map of one kind of tests/test_remap_emul.py rescaled to [P0][G0], or a random mix"""
    n_old = P0 * G0
    kind = rng.integers(0, 4)
    if kind == 0:                      # grow P and widen G
        P, G = P0 + int(rng.integers(1, 40)), G0 + int(rng.integers(0, 3))
        src = np.full((P, G), NONE, np.uint32)
        src[:P0, :G0] = np.arange(n_old, dtype=np.uint32).reshape(P0, G0)
    elif kind == 1:                    # compaction: departed pods dropped, the rest keep their order
        kept = np.sort(rng.choice(P0, max(1, P0 // 2), replace=False))
        P, G = kept.size, G0
        src = np.arange(n_old, dtype=np.uint32).reshape(P0, G0)[kept]
    elif kind == 2:                    # a permutation
        P, G = P0, G0
        src = rng.permutation(n_old).astype(np.uint32)
    else:                              # rows without a source among shuffled survivors, a new shape
        P, G = max(1, P0 + int(rng.integers(-5, 20))), max(1, G0 + int(rng.integers(-1, 3)))
        src = np.full(P * G, NONE, np.uint32)
        k = min(P * G, n_old) * 3 // 4
        src[rng.choice(P * G, k, replace=False)] = rng.choice(n_old, k, replace=False)
    return P, G, np.ascontiguousarray(src, np.uint32).ravel()


@pytest.mark.parametrize("flags", [0, 1, 2, 3], ids=["util", "power", "index", "power+index"])
def test_remap_equals_the_model(flags):
    rng = np.random.default_rng(100 + flags)
    eng = _engine()
    try:
        for trial in range(8):
            P0, G0 = int(rng.integers(1, 70)), int(rng.integers(1, 5))
            T = int(rng.choice([1, 3, 4, 63, 64, 65, 130, 240, 1800]))
            m = _model_ring(rng, eng, P0, G0, T, flags)
            for step in range(3):
                P, G, src = _random_map(rng, m.P, m.G)
                if (trial + step) % 2:
                    eng.resident_remap(P, G, torch.from_numpy(src.view(np.int32)).to("cuda:0"))
                else:
                    eng.resident_remap(P, G, src)
                m = _remapped(m, P, G, src)
                where = (flags, trial, step, T, P, G)
                _check_ring(eng, m, where)
                _check_verdicts(eng, m, rng, where)
                # the ring goes on working on its new shape
                n = int(rng.integers(1, T + 2))
                util = RS._mixed(rng, 0, m.rows, n)
                m.append(n, util, None)
                eng.append(util.view(np.float32))
                _check_ring(eng, m, where + ("append",))
                assert same_verdict(decide(eng, m), expected(m)) is None, where
    finally:
        eng.close()


def test_emulator_map_kinds_on_the_device():
    """the six map kinds of the CPU emulator's matrix, from host and from device memory"""
    rng = np.random.default_rng(7)
    eng = _engine()
    try:
        for kind in ("grow P", "widen G", "shrink", "permutation", "compaction", "none rows"):
            for dev in (False, True):
                m = _model_ring(rng, eng, P0, G0, 65, 3)
                P, G, src = make_map(kind, rng)
                eng.resident_remap(P, G, torch.from_numpy(src.view(np.int32)).cuda() if dev else src)
                m = _remapped(m, P, G, src)
                _check_ring(eng, m, (kind, dev))
                _check_verdicts(eng, m, rng, (kind, dev))
    finally:
        eng.close()


def _async_on_ring(eng, m, db, cb, smax):
    """gpr_decide_async over the resident planes as a device window (it reads the ring in stream order)"""
    u, p, _ = eng.resident_planes()
    return eng.decide_ptr(u, m.P, m.G, m.T, db, power=p if len(m.planes) > 1 else None, candidate_bits=cb,
                          series_max=smax, power_threshold=RS.THR if len(m.planes) > 1 else 0.0, in_kind=1,
                          out_kind=0, blocking=False)


@pytest.mark.parametrize("stream", ["context", "caller"])
def test_decisions_enqueued_before_a_remap_keep_the_old_verdicts(stream):
    import kat
    rng = np.random.default_rng(21)
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
        P, G, src = _random_map(rng, m.P, m.G)
        src[:] = NONE                  # the new ring has no sample anywhere: the old verdicts cannot come from it
        eng.resident_remap(P, G, src)
        eng.sync()
        for (db, cb, smax), r in outs:
            assert np.array_equal(db, exp["decision_bits"]) and np.array_equal(cb, exp["candidate_bits"])
            assert (r.n_series, r.n_candidates) == (exp["n_series"], exp["n_candidates"])
            assert kat.smax_equal(smax, exp["series_max"])
        m = _remapped(m, P, G, src)
        _check_ring(eng, m, stream)
        assert same_verdict(decide(eng, m), expected(m)) is None
        if s is not None:
            s.synchronize()
    finally:
        eng.close()


def test_bad_maps_and_no_window_leave_everything_as_it_was():
    import kat
    import gpu_pruner_b200 as g
    rng = np.random.default_rng(5)
    eng = _engine()
    try:
        with pytest.raises(g.GprError) as ei:
            eng.resident_remap(2, 2, np.arange(4, dtype=np.uint32))
        assert ei.value.code == g.ffi.GPR_E_STATE
        m = _model_ring(rng, eng, 20, 3, 130, 3)
        n_old = m.rows
        before = _read_ring(eng, m.rows, m.T, 2)
        exp = expected(m)
        W = (m.P + 31) // 32
        bad_maps = [
            (n_old + 5, 1, np.r_[np.arange(n_old), [n_old], [NONE] * 4]),   # old row n_old: out of range
            (3, 2, [0, 1, NONE, 5, 0x7FFFFFFF, 2]),                          # out of range at 4
            (4, 1, [NONE, 7, 8, 7]),                                         # old row 7 twice: new row 1
            (n_old, 1, np.r_[np.arange(n_old - 1), [3]]),                    # old row 3 twice: new row 3
        ]
        for k, (P, G, src) in enumerate(bad_maps):
            src = np.asarray(src, np.uint64).astype(np.uint32)
            want_row = first_bad(src, n_old)
            assert want_row < src.size
            for dev in (False, True):
                o = (eng.host_array((W,), np.uint32), eng.host_array((W,), np.uint32),
                     eng.host_array((m.P, m.G), np.float32))
                r = _async_on_ring(eng, m, *o)
                with pytest.raises(g.GprError) as ei:
                    eng.resident_remap(P, G, torch.from_numpy(src.view(np.int32)).cuda() if dev else src)
                assert ei.value.code == g.ffi.GPR_E_INVALID, (k, dev)
                assert f"src_rows[{want_row}]" in str(ei.value), (k, dev, str(ei.value))
                eng.sync()           # the pending result retires with its verdict
                assert np.array_equal(o[0], exp["decision_bits"]) and r.n_candidates == exp["n_candidates"]
                assert kat.smax_equal(o[2], exp["series_max"])
                after = _read_ring(eng, m.rows, m.T, 2)
                assert all(np.array_equal(a, b) for a, b in zip(before, after)), (k, dev)
                assert eng.resident_head() == m.head
                assert same_verdict(decide(eng, m), exp) is None
        for P, G in ((0, 4), (4, 0)):
            with pytest.raises(g.GprError) as ei:
                eng.resident_remap(P, G, np.zeros(0, np.uint32))
            assert ei.value.code == g.ffi.GPR_E_INVALID
        # a stale index stays stale through a remap, and is refused until the reindex
        eng.samples_scatter([0, 1], [0], [1_700_000_000_000], [55.0], 1_700_000_000, 1, m.T, m.rows, resident=True,
                            window_seconds=1)
        P, G, src = _random_map(rng, m.P, m.G)
        eng.resident_remap(P, G, src)
        m = _remapped(m, P, G, src)
        with pytest.raises(g.GprError) as ei:
            decide(eng, m)
        assert ei.value.code == g.ffi.GPR_E_STATE
        eng.resident_reindex()
        m.planes = _read_ring(eng, m.rows, m.T, 2)
        assert same_verdict(decide(eng, m), expected(m)) is None
    finally:
        eng.close()


# ---- an integrator's timeline ------------------------------------------------------------------------------------
T_TL, STEP = 300, 1


class Store:
    """the series a Prometheus would hold: (pod, slot) -> sorted (ts_ms, value) arrays"""

    def __init__(self):
        self.s = {}

    def add(self, rng, pod, slot, t0, t1):
        _, _, smp = _series(rng, pod, slot, t0, t1, STEP, rng.choice(["idle", "busy"]))
        ts = np.array([int(round(t * 1000)) for t, _ in smp], np.int64)
        v = np.array([np.nan if x == "NaN" else float(x) for _, x in smp], np.float64)
        self.s[(pod, slot)] = (ts, v)

    def stop(self, pod, t):
        for k in [k for k in self.s if k[0] == pod]:
            ts, v = self.s[k]
            self.s[k] = (ts[ts <= t * 1000], v[ts <= t * 1000])

    def batch(self, rows_of, t_lo, t_hi):
        """the samples in (t_lo, t_hi] of every series with a row, as a CSR batch"""
        offsets, rows, ts, vals = [0], [], [], []
        for k, (a, b) in sorted(self.s.items()):
            if k not in rows_of:
                continue
            sel = (a > t_lo * 1000) & (a <= t_hi * 1000)
            rows.append(rows_of[k])
            ts.append(a[sel])
            vals.append(b[sel])
            offsets.append(offsets[-1] + int(sel.sum()))
        return (np.array(offsets, np.uint64), np.array(rows, np.uint32),
                np.concatenate(ts) if ts else np.zeros(0, np.int64), np.concatenate(vals) if vals else np.zeros(0))


class RowTable:
    """the integrator's pod -> pod slot table of a ring [P][G], with head-room"""

    def __init__(self, pods, P, G):
        self.pod_slot = {p: i for i, p in enumerate(pods)}
        self.P, self.G = P, G

    def rows(self, store):
        return {k: self.pod_slot[k[0]] * self.G + k[1] for k in store.s if k[0] in self.pod_slot and k[1] < self.G}

    def reshape(self, pods, P, G):
        """the map to a table holding `pods` (in this order; kept pods first) on [P][G]"""
        src = np.full(P * G, NONE, np.uint32)
        new = {p: i for i, p in enumerate(pods)}
        for p, i in new.items():
            if p in self.pod_slot:
                for g in range(min(G, self.G)):
                    src[i * G + g] = self.pod_slot[p] * self.G + g
        self.pod_slot, self.P, self.G = new, P, G
        return src


@pytest.mark.parametrize("block_index", [False, True])
def test_integrator_timeline_never_requeries_the_window(block_index):
    rng = random.Random(40 + block_index)
    t0 = 1_700_000_000
    store = Store()
    pods = [f"pod-{i}" for i in range(8)]
    for p in pods:
        for s in range(rng.choice([1, 2])):
            store.add(rng, p, s, t0 - T_TL - 40, t0 + 10_000)
    table = RowTable(pods, 10, 2)                 # two pods of head-room
    ring, ref = _engine(), _engine()
    into_ring = []                                # (tick, t_prev, timestamps) of every batch scattered into the ring
    try:
        ring.resident_init(table.P, table.G, T_TL, block_index=block_index)
        t = t0
        offsets, rows, ts, vals = store.batch(table.rows(store), t - T_TL * STEP, t)
        into_ring.append((0, None, ts))
        ring.samples_scatter(offsets, rows, ts, vals, t, STEP, T_TL, table.P * table.G, resident=True)
        remaps = []
        for tick in range(1, 11):
            t_prev, t = t, t + int(rng.choice([20, 45, 90, 150]))
            # what changed in the cluster since the last tick, and the map the integrator builds for it
            src = None
            if tick == 2:                          # four pods join: beyond the head-room
                joined = [f"pod-{i}" for i in range(8, 12)]
                for p in joined:
                    store.add(rng, p, 0, t_prev + 1, t0 + 10_000)
                pods = pods + joined
                src = table.reshape(pods, len(pods) + 2, table.G)
            elif tick == 4:                        # pod-3 gains a third slot
                store.add(rng, "pod-3", 2, t_prev + 1, t0 + 10_000)
                src = table.reshape(pods, table.P, 3)
            elif tick == 5:                        # three pods have left since the last tick
                for p in ("pod-1", "pod-5", "pod-9"):
                    store.stop(p, t_prev)
            elif tick == 7:                        # and are compacted away
                pods = [p for p in pods if p not in ("pod-1", "pod-5", "pod-9")]
                src = table.reshape(pods, len(pods) + 1, table.G)
            if src is not None:
                remaps.append(tick)
                dev = torch.from_numpy(src.view(np.int32)).cuda() if tick % 2 else src
                ring.resident_remap(table.P, table.G, dev)
            n_new = (t - t_prev) // STEP
            ring.resident_advance(n_new)
            offsets, rows, ts, vals = store.batch(table.rows(store), t_prev, t)
            into_ring.append((tick, t_prev, ts))
            ring.samples_scatter(offsets, rows, ts, vals, t, STEP, T_TL, table.P * table.G, resident=True,
                                 window_seconds=n_new * STEP)
            # a fresh query of the whole window, into a context plane of the same row layout
            n_rows = table.P * table.G
            offsets, rows, ts, vals = store.batch(table.rows(store), t - T_TL * STEP, t)
            # what went into the ring this tick is only the slice: exactly the samples of the whole window that are
            # newer than the last tick, and fewer than the window holds
            sl = into_ring[-1][2]
            assert sl.size and sl.min() > t_prev * 1000, tick
            assert sl.size == int((ts > t_prev * 1000).sum()) < ts.size, (tick, sl.size, ts.size)
            ref.samples_scatter(offsets, rows, ts, vals, t, STEP, T_TL, n_rows)
            fresh = np.empty((n_rows, T_TL), np.uint32)
            ref.memcpy(fresh, ref.text_planes()[0], fresh.nbytes, 0, 1)
            (got,) = _read_ring(ring, n_rows, T_TL, 1)
            unrolled = np.roll(got, -ring.resident_head(), axis=1)
            assert np.array_equal(unrolled, fresh), (tick, np.argwhere(unrolled != fresh)[:3])
            if block_index:
                ring.resident_reindex()
            m = RS.Ring(table.P, table.G, T_TL, 2 if block_index else 0)
            m.planes, m.head = [got], ring.resident_head()
            assert np.array_equal(m.window(0).reshape(n_rows, T_TL).view(np.uint32), fresh)
            bad = same_verdict(decide(ring, m), expected(m))     # the oracle on the fresh window
            assert bad is None, (tick, bad)
        assert remaps == [2, 4, 7]
        # only tick 0 brought the whole window into the ring: every later batch lies after the tick before it
        assert [k for k, _, _ in into_ring] == list(range(11))
        assert all(b.min() > tp * 1000 for k, tp, b in into_ring if k > 0)
        assert table.G == 3 and "pod-1" not in table.pod_slot
    finally:
        ring.close()
        ref.close()


def test_c2_shape_widened_and_grown():
    """10,000 pods x 4 slots x 1,800 samples with the power plane and the index (0.6 GB), remapped to G = 5 and
    12,500 pods (pods shuffled, the new slot and the new pods without a source): every plane equals the model, read
    on the device, and gpr_decide_resident equals the oracle on the model's unrolled window"""
    import kat
    P0, G0, T = 10_000, 4, 1800
    P, G = 12_500, 5
    rng = np.random.default_rng(8)
    eng = _engine()
    try:
        eng.resident_init(P0, G0, T, power_plane=True, block_index=True)
        u, p, _ = eng.resident_planes()
        eng.synth_fill(0x5EED0002, 0, u, 0, P0, G0, T)
        eng.synth_fill(0x5EED0002, 1, p, 0, P0, G0, T)
        eng.resident_reindex()
        eng.resident_advance(777)              # a head that is not 0
        old = [torch.empty(P0 * G0 * T, dtype=torch.int32, device="cuda:0") for _ in range(2)]
        for ptr, t in zip((u, p), old):
            eng.memcpy(t.data_ptr(), ptr, t.numel() * 4, 1, 1)
        src = np.full((P, G), NONE, np.uint32)
        order = rng.permutation(P0)
        src[order, :G0] = np.arange(P0 * G0, dtype=np.uint32).reshape(P0, G0)
        src = src.ravel()
        eng.resident_remap(P, G, torch.from_numpy(src.view(np.int32)).cuda())
        assert eng.resident_head() == 777
        u2, p2, ld = eng.resident_planes()
        assert ld == T
        idx = torch.from_numpy(src.astype(np.int64)).cuda()
        live = idx != NONE
        models = []
        for ptr, t in zip((u2, p2), old):
            got = torch.empty(P * G * T, dtype=torch.int32, device="cuda:0")
            eng.memcpy(got.data_ptr(), ptr, got.numel() * 4, 1, 1)
            want = torch.full((P * G, T), -1, dtype=torch.int32, device="cuda:0")
            want[live] = t.view(P0 * G0, T)[idx[live]]
            assert torch.equal(got.view(P * G, T), want)
            models.append(want)
        # the verdict (decided on the moved index) against the float64 oracle on the model's unrolled window
        from oracle import oracle_c
        win = [np.roll(t.cpu().numpy().view(np.float32), -777, axis=1).reshape(P, G, T) for t in models]
        del models
        want = oracle_c.decide(win[0], win[1], power_threshold=150.0, n_threads=os.cpu_count() or 1)
        W = (P + 31) // 32
        db, cb, smax = np.zeros(W, np.uint32), np.zeros(W, np.uint32), np.zeros((P, G), np.float32)
        r = eng.decide_ptr(None, P, G, T, db, candidate_bits=cb, series_max=smax, power_threshold=150.0, in_kind=1,
                           out_kind=0, resident=True)
        assert np.array_equal(db, want["decision_bits"]) and np.array_equal(cb, want["candidate_bits"])
        assert (r.n_series, r.n_candidates, r.n_decisions) == (want["n_series"], want["n_candidates"],
                                                               want["n_decisions"])
        assert kat.smax_equal(smax, want["series_max"])
        assert want["n_candidates"] > 0 and np.isnan(smax[:, G0:]).all() and np.isnan(smax[P0:]).all()
    finally:
        eng.close()


def test_engine_refuses_a_device_map_it_cannot_read_as_rows():
    """IdleEngine.resident_remap reads a device map as uint32 in place: a float tensor, a 64-bit one or a
    non-contiguous one is a ValueError before the C ABI is called, and the ring is untouched"""
    eng = _engine()
    try:
        eng.resident_init(4, 2, 16)
        before = _read_ring(eng, 8, 16, 1)
        rows = torch.arange(8, device="cuda:0")
        for bad in (rows.float(), rows, rows.to(torch.int32).view(2, 4).t()):
            with pytest.raises(ValueError):
                eng.resident_remap(4, 2, bad)
        assert all(np.array_equal(a, b) for a, b in zip(before, _read_ring(eng, 8, 16, 1)))
        eng.resident_remap(4, 2, rows.to(torch.int32).flip(0))
        assert eng.resident_head() == 0
    finally:
        eng.close()
