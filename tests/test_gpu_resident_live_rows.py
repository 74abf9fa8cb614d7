"""GPU: gpr_resident_live_rows on an H100 — which rows of the resident ring hold a sample in the util or the power plane.
  * rings written through gpr_resident_planes (every position of one sample per row, other NaNs, +-0, +-Inf,
    denormals, row counts off a multiple of 32), with and without the power plane and the block index, against the numpy
    model of tests/test_live_rows_emul.py; host and device destinations between guard words;
  * a current index is read, a stale one (a resident gpr_samples_scatter left it so) is not, and not refused;
  * every error (no ring, NULL bits, bad mem_kind) leaves the destination untouched;
  * decisions enqueued before the call keep their verdicts, on the context's stream and on a torch.cuda.Stream;
  * a C2-shaped ring (10,000 x 4 x 1,800 with the power plane)."""
import ctypes as C

import numpy as np
import pytest

import ring_scripts as RS
from test_gpu_resident import decide, expected, same_verdict
from test_gpu_resident_remap import _async_on_ring, _engine, _model_ring
from test_live_rows_emul import Case, live_model, words_of

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")
GUARD = 0x5EC7AB1E


def _write_ring(eng, c, P, G):
    """the case's planes as the resident ring [P][G][T] (P * G == c.n_rows), the index rebuilt from them"""
    from gpu_pruner_b200 import ffi
    eng.resident_init(P, G, c.T, power_plane=bool(c.flags & 1), block_index=bool(c.flags & 2))
    u, p, ld = eng.resident_planes()
    assert ld == c.T
    for ptr, pl in zip((u, p), c.planes):
        eng.memcpy(ptr, np.ascontiguousarray(pl), pl.nbytes, ffi.GPR_MEM_DEVICE, ffi.GPR_MEM_HOST)
    eng.resident_reindex()


def _host_call(eng, n_words, kind=None):
    """the raw call into a host buffer between guard words: (rc, words, guards intact)"""
    from gpu_pruner_b200 import ffi
    buf = np.full(n_words + 2, GUARD, np.uint32)
    rc = eng._lib.gpr_resident_live_rows(eng._h, C.c_void_p(buf.ctypes.data + 4),
                                         ffi.GPR_MEM_HOST if kind is None else kind)
    return rc, buf[1:-1].copy(), buf[0] == GUARD and buf[-1] == GUARD


def _device_call(eng, n_words):
    from gpu_pruner_b200 import ffi
    t = torch.full((n_words + 2,), GUARD, dtype=torch.int32, device="cuda:0")
    rc = eng._lib.gpr_resident_live_rows(eng._h, C.c_void_p(t.data_ptr() + 4), ffi.GPR_MEM_DEVICE)
    torch.cuda.synchronize()
    a = t.cpu().numpy().view(np.uint32)
    return rc, a[1:-1].copy(), a[0] == GUARD and a[-1] == GUARD


def _shape(n_rows):
    """[P][G] with P * G == n_rows: G = 1 for an odd count, else 2"""
    return (n_rows, 1) if n_rows % 2 else (n_rows // 2, 2)


@pytest.mark.parametrize("T", [1, 3, 4, 63, 64, 65, 1800])
def test_live_rows_equal_the_model(T):
    eng = _engine()
    try:
        for flags in (0, 1, 2, 3):
            for head in sorted({0, T // 2, T - 1}):
                pos = None if T < 1800 else sorted(set(range(0, T, 11)) | {T - 1})
                c = Case(f"T={T} head={head} flags={flags}", T, flags, head, 1000 * T + 10 * flags + head, pos)
                _write_ring(eng, c, *_shape(c.n_rows))
                want = words_of(c.want)
                rc, got, guards = _host_call(eng, want.size)
                assert rc == 0 and guards and np.array_equal(got, want), c.name
                rc, got, guards = _device_call(eng, want.size)
                assert rc == 0 and guards and np.array_equal(got, want), c.name
                assert np.array_equal(eng.resident_live_rows(), c.want), c.name
    finally:
        eng.close()


def test_a_current_index_is_read_and_a_stale_one_is_not():
    from gpu_pruner_b200 import ffi
    eng = _engine()
    try:
        c = Case("index", 130, 3, 5, 77)
        P, G = _shape(c.n_rows)
        _write_ring(eng, c, P, G)
        dead = np.flatnonzero(~c.want)
        assert dead.size >= 2
        # planes written behind a current index's back (which only a writer of gpr_resident_planes can do): the index
        # answers, so the row reads dead
        row = int(dead[0])
        u, _, _ = eng.resident_planes()
        one = np.array([np.float32(42.0)]).view(np.uint32)
        eng.memcpy(u + (row * c.T + 7) * 4, one, 4, ffi.GPR_MEM_DEVICE, ffi.GPR_MEM_HOST)
        assert np.array_equal(eng.resident_live_rows(), c.want)
        # a resident merge makes the index stale: the planes answer, and the call is not refused
        row2 = int(dead[1])
        t_end = 1_700_000_000
        eng.samples_scatter([0, 1], [row2], [t_end * 1000], [55.0], t_end, 1, c.T, c.n_rows, resident=True,
                            window_seconds=1)
        want = c.want.copy()
        want[[row, row2]] = True
        assert np.array_equal(eng.resident_live_rows(), want)
        eng.resident_reindex()
        assert np.array_equal(eng.resident_live_rows(), want)
    finally:
        eng.close()


def test_errors_leave_the_destination_untouched():
    from gpu_pruner_b200 import ffi
    eng = _engine()
    try:
        rc, got, guards = _host_call(eng, 4)
        assert rc == ffi.GPR_E_STATE and guards and (got == GUARD).all()
        assert "no resident window" in eng._lib.gpr_last_error(eng._h).decode()
        rc, got, guards = _device_call(eng, 4)
        assert rc == ffi.GPR_E_STATE and guards and (got == GUARD).all()
        eng.resident_init(70, 2, 64, power_plane=True)
        assert eng._lib.gpr_resident_live_rows(eng._h, None, ffi.GPR_MEM_HOST) == ffi.GPR_E_INVALID
        for kind in (2, -1, 7):
            rc, got, guards = _host_call(eng, 5, kind)
            assert rc == ffi.GPR_E_INVALID and guards and (got == GUARD).all(), kind
        rc, got, guards = _host_call(eng, 5)
        assert rc == 0 and guards and (got == 0).all()   # a fresh ring: no sample anywhere
    finally:
        eng.close()


@pytest.mark.parametrize("stream", ["context", "caller"])
def test_decisions_enqueued_before_the_call_stay_pending(stream):
    import kat
    rng = np.random.default_rng(31)
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
        live = eng.resident_live_rows()
        assert np.array_equal(live, live_model(m.planes))
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


def test_c2_shaped_ring():
    """10,000 pods x 4 slots x 1,800 samples with the power plane: a fifth of the rows without a sample in either plane,
    a tenth with their only samples in the power plane"""
    from gpu_pruner_b200 import ffi
    rng = np.random.default_rng(2)
    P, G, T = 10_000, 4, 1800
    rows = P * G
    eng = _engine()
    try:
        eng.resident_init(P, G, T, power_plane=True)
        u, p, _ = eng.resident_planes()
        kind = rng.choice(3, rows, p=[0.7, 0.2, 0.1])     # 0: util samples, 1: none, 2: power only
        for ptr, plane in ((u, 0), (p, 1)):
            a = np.full((rows, T), RS.NO_SAMPLE, np.uint32)
            has = (kind == 0) if plane == 0 else (kind == 2)
            at = rng.integers(0, T, rows)
            a[has, at[has]] = np.float32(17.0).view(np.uint32)
            eng.memcpy(ptr, a, a.nbytes, ffi.GPR_MEM_DEVICE, ffi.GPR_MEM_HOST)
            del a
        want = kind != 1
        assert np.array_equal(eng.resident_live_rows(), want)
        rc, got, guards = _device_call(eng, (rows + 31) // 32)
        assert rc == 0 and guards and np.array_equal(got, words_of(want))
    finally:
        eng.close()
