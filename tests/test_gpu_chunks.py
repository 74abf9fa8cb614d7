"""gpr_chunks_scatter on the H100 against the paths it must equal (include/gpr.h): Prometheus XOR chunks of random
series, decoded on the GPU, leave the planes gpr_samples_scatter leaves for the same samples decoded by
tests/chunks_ref.py, and so those of gpr_text_scan + gpr_text_parse of the same samples as text — bit for bit, on the
util plane and on the power plane at the threshold's f32 neighbours, with equal counts.  Then: pageable, pinned and
device batches, data at odd addresses, a C2-sized batch of 120-sample chunks (600,000 chunks, more than two upload
pieces); a daemon timeline into the resident ring next to a samples-fed twin, with and without the block index; the
C2 window decided from chunks against deciding the synthetic planes directly; and malformed batches leaving the
destination and pending async results intact."""
import ctypes as C

import numpy as np
import pytest

import chunks_ref as R
import kat
from test_gpu_samples import (FILL, STEP, T_END, THR, _engine, _plane, _random_batch, _read, _render, _ring,
                              _text_parse, _torch_dev)

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    e = _engine()
    yield e
    e.close()


def _chunks_of(offsets, ts, vals, per_chunk=120):
    bits = np.ascontiguousarray(vals, np.float64).view(np.uint64)
    return R.encode_native(offsets, ts, bits, per_chunk)


def _decoded(sc, cb, data, n_series):
    """the chunks' samples by the reference decoder, in CSR form"""
    offsets, ts, vals = [0], [], []
    for s in range(n_series):
        for c in range(int(sc[s]), int(sc[s + 1])):
            t, v, fault = R.decode(data[int(cb[c]):int(cb[c + 1])].tobytes())
            assert fault is None
            ts += t
            vals += v
        offsets.append(len(ts))
    return (np.array(offsets, np.uint64), np.array(ts, np.int64),
            np.array(vals, np.uint64).view(np.float64))


@pytest.mark.parametrize("plane,thr", [(0, 0.0), (1, THR), (1, 149.99)])
def test_bit_identical_to_samples_and_text(eng, plane, thr):
    rng = np.random.default_rng(51 + plane + int(thr))
    T, n_rows = 120, 300
    offsets, rows, ts, vals = _random_batch(rng, 500, n_rows, T)
    if plane == 1:   # the threshold's f32 neighbours
        f = np.float32(thr)
        near = np.array([np.nextafter(f, np.float32(0)), f, np.nextafter(f, np.float32(1e9)), thr,
                         np.nextafter(thr, 0), np.nextafter(thr, 1e9)], np.float64)
        pick = rng.random(len(vals)) < 0.3
        vals[pick] = rng.choice(near, int(pick.sum()))
    stale = rng.random(len(vals)) < 0.03
    bits = vals.view(np.uint64).copy()
    bits[stale] = R.STALE_NAN_BITS
    vals = bits.view(np.float64)
    sc, cb, data = _chunks_of(offsets, ts, vals, int(rng.choice([7, 120])))
    st = eng.chunks_scatter(sc, rows, cb, data, T_END, STEP, T, n_rows, plane=plane, power_threshold=thr)
    got = _plane(eng, n_rows, T, plane)
    d_off, d_ts, d_vals = _decoded(sc, cb, data, len(rows))
    assert np.array_equal(d_ts, ts) and np.array_equal(d_vals.view(np.uint64), bits)
    want_st = eng.samples_scatter(d_off, rows, d_ts, d_vals, T_END, STEP, T, n_rows, plane=plane, power_threshold=thr)
    want = _plane(eng, n_rows, T, plane)
    assert np.array_equal(got, want), np.argwhere(got != want)[:8]
    assert st == want_st and st["n_in"] == len(ts) and st["n_oow"] > 0
    keep = ~stale                 # the text has no staleness marker: NaN there is dropped the same way
    k_off = np.concatenate([[0], np.cumsum([int(keep[int(offsets[s]):int(offsets[s + 1])].sum())
                                            for s in range(len(rows))])]).astype(np.uint64)
    text, order = _render(k_off, rows, ts[keep], vals[keep])
    _text_parse(eng, text, order, T, n_rows, plane, thr)
    assert np.array_equal(_plane(eng, n_rows, T, plane), got)
    assert (got != FILL).sum() > n_rows * T // 2


def test_every_source_gives_the_same_plane(eng):
    """6,000 series of ~1,800 samples as 120-sample chunks (about 90,000 chunks); a pageable, a pinned and a device
    batch, and the device data at 1 and 7 bytes past a 16-byte boundary; then a C2-sized batch (40,000 series,
    600,000 chunks, over two upload pieces) from pageable, pinned and device memory against gpr_samples_scatter"""
    import torch
    import gpu_pruner_b200 as g
    rng = np.random.default_rng(61)
    for n_rows, T, lo, hi in ((6000, 1800, 1500, 2100), (40000, 1800, 1790, 1810)):
        lengths = rng.integers(lo, hi, n_rows)
        lengths[rng.random(n_rows) < 0.02] = 0
        offsets = np.concatenate([[0], np.cumsum(lengths)]).astype(np.uint64)
        n = int(offsets[-1])
        rows = rng.permutation(n_rows).astype(np.uint32)
        base = T_END * 1000 - (T + 1) * 1000
        ts = (base + (np.arange(n) - np.repeat(offsets[:-1].astype(np.int64), lengths)) * 1000
              + rng.integers(-3, 4, n) * (rng.random(n) < 0.2)).astype(np.int64)
        vals = rng.integers(0, 101, n).astype(np.float64)
        vals[rng.random(n) < 0.1] = 0.0
        vals[rng.random(n) < 0.05] = np.nan
        sc, cb, data = _chunks_of(offsets, ts, vals)
        planes, stats = {}, {}
        stats["samples"] = eng.samples_scatter(offsets, rows, ts, vals, T_END, STEP, T, n_rows)
        planes["samples"] = _plane(eng, n_rows, T)
        stats["pageable"] = eng.chunks_scatter(sc, rows, cb, data, T_END, STEP, T, n_rows)
        planes["pageable"] = _plane(eng, n_rows, T)
        pdata = eng.host_array(len(data), np.uint8)
        pdata[:] = data
        stats["pinned"] = eng.chunks_scatter(sc, rows, cb, pdata, T_END, STEP, T, n_rows)
        planes["pinned"] = _plane(eng, n_rows, T)
        d_sc, d_rows, d_cb = _torch_dev(sc.view(np.int64)), _torch_dev(rows.view(np.int32)), _torch_dev(cb.view(np.int64))
        raw = torch.empty(len(data) + 16, dtype=torch.uint8, device="cuda")
        for shift in (0, 1, 7):
            raw[shift:shift + len(data)] = torch.from_numpy(data).cuda()
            torch.cuda.synchronize()
            assert raw[shift:].data_ptr() % 16 == shift
            k = f"device+{shift}"
            stats[k] = eng.chunks_scatter(d_sc, d_rows, d_cb, raw[shift:].data_ptr(), T_END, STEP, T, n_rows,
                                          mem_kind=g.ffi.GPR_MEM_DEVICE, n_series=n_rows)
            planes[k] = _plane(eng, n_rows, T)
        for k in planes:
            assert np.array_equal(planes[k], planes["samples"]), (n_rows, k)
            assert stats[k] == stats["samples"], (n_rows, k, stats[k], stats["samples"])
        if n_rows == 40000:
            assert len(cb) - 1 >= 600_000 and len(data) > 2 * (32 << 20), (len(cb), len(data))


@pytest.mark.parametrize("block_index", [False, True])
def test_daemon_timeline_matches_the_samples_fed_ring(block_index):
    """two contexts run the same ticks — advance + gpr_samples_scatter, advance + gpr_chunks_scatter of whole
    chunks that reach back before the slice (their older samples counted out of the window) — into rings with a power
    plane; the rings wrap and stay bit-identical; with the block index deciding before the reindex is GPR_E_STATE;
    after it gpr_decide_resident equals the oracle on the ring's samples"""
    import gpu_pruner_b200 as g
    from oracle import oracle_c
    rng = np.random.default_rng(71 + block_index)
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
                offsets, rows, ts, vals = _random_batch(rng, 60, P * G, n_new, max_len=3 * n_new, window=3 * n_new)
                ts += (t_end - T_END) * 1000
                if plane == 1:
                    vals = np.where(rng.random(len(vals)) < 0.5, rng.choice([149.999999, 150.0, 150.0000001, 80.0],
                                                                         len(vals)), vals)
                sc, cb, data = _chunks_of(offsets, ts, vals, 30)
                sa = a.samples_scatter(offsets, rows, ts, vals, t_end, STEP, T, P * G, plane=plane,
                                       power_threshold=thr, resident=True, window_seconds=n_new)
                sb = b.chunks_scatter(sc, rows, cb, data, t_end, STEP, T, P * G, plane=plane, power_threshold=thr,
                                      resident=True, window_seconds=n_new)
                assert sa == sb and sb["n_oow"] > 0
            ra, rb = _ring(a, P, G, T), _ring(b, P, G, T)
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
        assert advanced > T
    finally:
        a.close()
        b.close()


def test_c2_window_from_chunks_decides_like_the_window(eng):
    """the C2 synthetic window (10,000 pods x 4 GPUs x 1,800 samples), every present cell a sample at its bucket's
    timestamp, as 120-sample chunks from the device into the context planes, decided with the power veto and the
    gates: bitmaps, counts and series_max equal deciding the synthetic planes directly"""
    import torch
    import gpu_pruner_b200 as g
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
        offsets = np.zeros(rows + 1, np.uint64)
        offsets[1:] = np.cumsum(counts.cpu().numpy())
        r_idx, c_idx = present.nonzero(as_tuple=True)
        ts = (T_END * 1000 - (T - 1 - c_idx).to(torch.int64) * STEP * 1000).cpu().numpy()
        vals = src[r_idx, c_idx].to(torch.float64).cpu().numpy()
        sc, cb, data = _chunks_of(offsets, ts, vals)
        d = [_torch_dev(x) for x in (sc.view(np.int64), np.arange(rows, dtype=np.int32), cb.view(np.int64), data)]
        st = eng.chunks_scatter(*d, T_END, STEP, T, rows, plane=plane, power_threshold=THR if plane else 0.0,
                                mem_kind=g.ffi.GPR_MEM_DEVICE, n_series=rows)
        assert st["n_in"] == int(counts.sum()) and st["n_oow"] == 0
    tu, tw = eng.text_planes()
    got = decide(tu, tw)
    for k in range(3):
        assert np.array_equal(got[0][k].view(np.uint32), direct[0][k].view(np.uint32)), k
    assert got[1] == direct[1]


def _raw(eng, batch, n_rows, T, flags):
    import gpu_pruner_b200 as g
    grid = g.ffi.gpr_text_grid()
    grid.struct_size = C.sizeof(g.ffi.gpr_text_grid)
    grid.flags, grid.t_end, grid.window_seconds, grid.step = flags, T_END, T * STEP, STEP
    grid.n_samples, grid.n_rows = T, n_rows
    return eng._lib.gpr_chunks_scatter(eng.handle, C.byref(batch), C.byref(grid), 0, None)


def test_malformed_batches_leave_the_destination_untouched(eng):
    import torch
    import gpu_pruner_b200 as g
    from chunks_ref import BitWriter
    rng = np.random.default_rng(81)
    T, n_rows = 60, 20
    offsets, rows, ts, vals = _random_batch(rng, 30, n_rows, T, max_len=50)
    lengths = np.diff(offsets.astype(np.int64))
    offsets = np.concatenate([[0], np.cumsum(np.maximum(lengths, 1))]).astype(np.uint64)
    n = int(offsets[-1])
    ts = np.resize(ts, n).astype(np.int64)
    vals = np.resize(vals, n)
    sc, cb, data = _chunks_of(offsets, ts, vals, 9)
    eng.chunks_scatter(sc, rows, cb, data, T_END, STEP, T, n_rows)
    before = _plane(eng, n_rows, T)
    assert (before != FILL).any()
    # an async decision enqueued before the failing calls completes at gpr_sync
    P_d, G_d = 4, 5
    dbits = torch.zeros(1, dtype=torch.int32, device="cuda")
    r_async = eng.decide_ptr(eng.text_planes()[0], P_d, G_d, T, dbits, blocking=False)

    def with_chunk(k, chunk):
        """the batch with chunk k replaced"""
        parts = [data[int(cb[c]):int(cb[c + 1])].tobytes() for c in range(len(cb) - 1)]
        parts[k] = chunk
        return R.batch([parts[int(sc[s]):int(sc[s + 1])] for s in range(len(rows))])[1:]

    k = 5
    full = data[int(cb[k]):int(cb[k + 1])].tobytes()
    reuse = BitWriter().varint(0).put(0, 64).uvarint(1).string("10").put(0, 8).chunk(2)
    cases = {"ends mid-sample": with_chunk(k, full[:-1]),
             "shorter than its header": with_chunk(k, b"\x00"),
             "reuse before a window": with_chunk(k, reuse)}
    bad_row = rows.copy()
    bad_row[7] = n_rows
    dec = cb.copy()
    dec[6] = dec[5] - 1
    keep = []
    for kind in (g.ffi.GPR_MEM_HOST, g.ffi.GPR_MEM_DEVICE):
        def mk(s_=sc, r_=rows, c_=cb, d_=data, size=None):
            b = g.ffi.gpr_chunk_batch()
            b.struct_size = C.sizeof(g.ffi.gpr_chunk_batch) if size is None else size
            b.mem_kind = kind
            arrs = [s_, r_, c_, d_]
            if kind == g.ffi.GPR_MEM_DEVICE:
                arrs = [_torch_dev(a.view(np.int64) if a.dtype == np.uint64 else a.view(np.int32) if a.dtype == np.uint32
                                   else a) for a in arrs]
            else:
                arrs = [np.ascontiguousarray(a) for a in arrs]
            keep.append(arrs)
            ptr = [a.data_ptr() if hasattr(a, "data_ptr") else a.ctypes.data for a in arrs]
            b.series_chunks, b.rows, b.chunk_bytes, b.data = ptr
            b.n_series = len(rows)
            return b
        tried = {"struct_size": mk(size=8), "row >= n_rows": mk(r_=bad_row), "chunk_bytes decrease": mk(c_=dec),
                 "series_chunks[0] != 0": mk(s_=sc + np.uint64(1))}
        for name, (c2, d2) in cases.items():
            tried[name] = mk(c_=c2, d_=d2)
        for name, b in tried.items():
            rc = _raw(eng, b, n_rows, T, g.ffi.GPR_TEXT_FILL)
            msg = eng._lib.gpr_last_error(eng.handle)
            assert rc == g.ffi.GPR_E_INVALID, (name, kind, rc, msg)
            if name in cases:
                assert b"chunk 5 " in msg, (name, msg)
            assert np.array_equal(_plane(eng, n_rows, T), before), (name, kind)
    eng.sync()
    want = eng.decide_ptr(eng.text_planes()[0], P_d, G_d, T, torch.zeros(1, dtype=torch.int32, device="cuda"))
    assert (r_async.n_series, r_async.n_candidates) == (want.n_series, want.n_candidates)
