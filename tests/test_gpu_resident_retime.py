"""GPU: gpr_resident_retime on an H100 — the resident ring's newest n_keep buckets merged `factor` to a bucket.
  * rings filled by gpr_append at random heads (tests/ring_scripts.py's mixed cells: other NaNs, +-0, +-Inf, negatives),
    with and without the power plane and the block index, against the numpy model of tests/test_retime_emul.py; the
    head is 0 afterwards and gpr_decide_resident's verdicts on the retimed ring equal the oracle's;
  * an index that was stale before the call (a resident gpr_samples_scatter left it so) is current after it;
  * bit for bit against a fresh gpr_samples_scatter of the same samples on the new grid, +0 and -0 in both orders in one
    new bucket, on both planes;
  * every error (no ring, factor 0, n_keep 0 or above n_samples) leaves the ring, the head and the index as they were;
  * decisions enqueued before the call keep their verdicts, on the context's stream and on a torch.cuda.Stream;
  * one k_retime_rows per plane (the index is rebuilt by the same CTAs);
  * a C2-shaped ring (10,000 x 4 x 1,800 with the power plane and the index), factor 2."""
import numpy as np
import pytest

import ring_scripts as RS
from test_gpu_resident import decide, expected, same_verdict
from test_gpu_resident_remap import _async_on_ring, _engine, _model_ring, _read_ring
from test_retime_emul import _merge, retime_model

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")
T_END = 1_700_000_000


def _retimed(m, n_keep, factor):
    n = RS.Ring(m.P, m.G, -(-n_keep // factor), m.flags)
    n.planes = [retime_model(p, m.head, n_keep, factor) for p in m.planes]
    return n


def _check(eng, m, where):
    got = _read_ring(eng, m.rows, m.T, len(m.planes))
    for k, (g, w) in enumerate(zip(got, m.planes)):
        if not np.array_equal(g, w):
            r, c = map(int, np.argwhere(g != w)[0])
            raise AssertionError(f"{where}: plane {k} row {r} cell {c}: {g[r, c]:#010x} != {w[r, c]:#010x}")
    assert eng.resident_head() == m.head, where


@pytest.mark.parametrize("flags", [0, 1, 2, 3])
def test_retime_equals_the_model_and_decides_like_the_oracle(flags):
    rng = np.random.default_rng(100 + flags)
    eng = _engine()
    try:
        for T, n_keep, factor in ((1800, 1800, 2), (1800, 900, 1), (1800, 900, 2), (65, 64, 3), (64, 33, 7),
                                  (5, 5, 5), (63, 1, 1), (240, 240, 4)):
            m = _model_ring(rng, eng, 37, 3, T, flags)
            eng.resident_retime(n_keep, factor)
            n = _retimed(m, n_keep, factor)
            _check(eng, n, f"T={T} n_keep={n_keep} factor={factor} flags={flags}")
            assert eng.resident_head() == 0
            assert same_verdict(decide(eng, n), expected(n)) is None
            assert same_verdict(decide(eng, n, early=True), expected(n)) is None
    finally:
        eng.close()


def test_a_stale_index_is_current_after_the_call():
    rng = np.random.default_rng(7)
    eng = _engine()
    try:
        m = _model_ring(rng, eng, 40, 2, 128, 3)
        row, col = 5, (m.head + 127) % 128          # the newest bucket of row 5
        eng.samples_scatter([0, 1], [row], [T_END * 1000], [99.0], T_END, 1, m.T, m.rows, resident=True,
                            window_seconds=128)
        m.planes[0][row, col] = _merge(np.array([m.planes[0][row, col], np.float32(99.0).view(np.uint32)], np.uint32))
        with pytest.raises(RuntimeError):
            decide(eng, m)                           # the stale index is refused
        eng.resident_retime(128, 2)
        n = _retimed(m, 128, 2)
        _check(eng, n, "stale")
        assert same_verdict(decide(eng, n), expected(n)) is None
    finally:
        eng.close()


def _samples(rng, rows, t_end, N, step_ms_jitter=True):
    """per row, samples every second of (t_end - N, t_end] with some gaps; values with +-0 in both orders inside the
    buckets of a coarser step, negatives, NaN, +-Inf"""
    offsets, ts, vals, row_ids = [0], [], [], []
    for r in range(rows):
        t = np.arange(t_end - N + 1, t_end + 1, dtype=np.int64) * 1000
        if step_ms_jitter:
            t = t - rng.integers(0, 999, t.size)
        keep = rng.random(t.size) < 0.6
        t = np.sort(t[keep])
        v = rng.choice([0.0, -0.0, 37.5, 100.0, -3.0, np.nan, np.inf, -np.inf, 1e-3], t.size)
        if r % 3 == 0:
            v = np.where(np.arange(t.size) % 2 == (r // 3) % 2, 0.0, -0.0)
        ts.append(t)
        vals.append(v)
        row_ids.append(r)
        offsets.append(offsets[-1] + t.size)
    return (np.array(offsets, np.uint64), np.array(row_ids, np.uint32), np.concatenate(ts),
            np.concatenate(vals).astype(np.float64))


@pytest.mark.parametrize("N,s,N2,s2", [(120, 5, 120, 10), (120, 5, 60, 15), (100, 15, 100, 30), (120, 4, 40, 4)])
def test_bit_for_bit_against_a_fresh_scatter_on_the_new_grid(N, s, N2, s2):
    rng = np.random.default_rng(N + s + N2 + s2)
    P, G = 30, 2
    rows = P * G
    T, T2 = -(-N // s), -(-N2 // s2)
    n_keep, factor = (T if N2 == N else N2 // s), s2 // s
    off, rid, ts, v = _samples(rng, rows, T_END, N)
    poff, prid, pts, pv = _samples(rng, rows, T_END, N)
    pv = np.abs(pv) * 3
    eng = _engine()
    try:
        eng.resident_init(P, G, T, power_plane=True, block_index=True)
        for plane, a in ((0, (off, rid, ts, v)), (1, (poff, prid, pts, pv))):
            eng.samples_scatter(*a, T_END, s, T, rows, window_seconds=N, plane=plane, resident=True,
                                power_threshold=RS.THR if plane else 0.0)
        eng.resident_reindex()
        eng.resident_retime(n_keep, factor)
        got = _read_ring(eng, rows, T2, 2)
        eng.resident_init(P, G, T2, power_plane=True, block_index=True)
        for plane, a in ((0, (off, rid, ts, v)), (1, (poff, prid, pts, pv))):
            eng.samples_scatter(*a, T_END, s2, T2, rows, window_seconds=N2, plane=plane, resident=True,
                                power_threshold=RS.THR if plane else 0.0)
        want = _read_ring(eng, rows, T2, 2)
        for k in range(2):
            assert np.array_equal(got[k], want[k]), (k, np.argwhere(got[k] != want[k])[:3])
        assert (got[0] == 0).any()                    # +0 won over -0 somewhere
    finally:
        eng.close()


def test_errors_leave_the_ring_untouched():
    from gpu_pruner_b200 import ffi
    rng = np.random.default_rng(5)
    eng = _engine()
    try:
        assert eng._lib.gpr_resident_retime(eng._h, 10, 2) == ffi.GPR_E_STATE
        assert "no resident window" in eng._lib.gpr_last_error(eng._h).decode()
        m = _model_ring(rng, eng, 50, 2, 300, 3)
        exp = expected(m)
        before = _read_ring(eng, m.rows, m.T, 2)
        for n_keep, factor in ((10, 0), (0, 2), (301, 1), (0xFFFFFFFF, 3)):
            assert eng._lib.gpr_resident_retime(eng._h, n_keep, factor) == ffi.GPR_E_INVALID, (n_keep, factor)
            assert all(np.array_equal(a, b) for a, b in zip(_read_ring(eng, m.rows, m.T, 2), before))
            assert eng.resident_head() == m.head
            assert same_verdict(decide(eng, m), exp) is None      # the index is the old ring's
    finally:
        eng.close()


@pytest.mark.parametrize("stream", ["context", "caller"])
def test_decisions_enqueued_before_the_call_keep_their_verdicts(stream):
    import kat
    rng = np.random.default_rng(41)
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
        eng.resident_retime(1200, 2)
        eng.sync()
        for (db, cb, smax), r in outs:
            assert np.array_equal(db, exp["decision_bits"]) and np.array_equal(cb, exp["candidate_bits"])
            assert (r.n_series, r.n_candidates) == (exp["n_series"], exp["n_candidates"])
            assert kat.smax_equal(smax, exp["series_max"])
        n = _retimed(m, 1200, 2)
        _check(eng, n, "after pending")
        assert same_verdict(decide(eng, n), expected(n)) is None
        if s is not None:
            s.synchronize()
    finally:
        eng.close()


@pytest.mark.parametrize("flags,planes", [(0, 1), (1, 2), (2, 1), (3, 2)])
def test_launch_count(flags, planes):
    rng = np.random.default_rng(9)
    eng = _engine()
    try:
        _model_ring(rng, eng, 20, 2, 100, flags)
        n0 = eng.launch_count()
        eng.resident_retime(100, 3)
        assert eng.launch_count() - n0 == planes     # one k_retime_rows per plane; the index is rebuilt inside it
    finally:
        eng.close()


def test_c2_shaped_ring():
    """10,000 pods x 4 slots x 1,800 samples with the power plane and the index, step doubled"""
    rng = np.random.default_rng(2)
    P, G, T = 10_000, 4, 1800
    eng = _engine()
    try:
        m = RS.Ring(P, G, T, 3)
        eng.resident_init(P, G, T, power_plane=True, block_index=True)
        util = RS._mixed(rng, 0, m.rows, 1000)
        power = RS._mixed(rng, 1, m.rows, 1000)
        m.append(1000, util, power)
        eng.append(util.view(np.float32), power.view(np.float32))
        eng.resident_retime(1800, 2)
        n = _retimed(m, 1800, 2)
        _check(eng, n, "C2")
        assert same_verdict(decide(eng, n), expected(n)) is None
    finally:
        eng.close()
