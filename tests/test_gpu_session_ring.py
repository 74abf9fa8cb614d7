"""One context through sequences that reshape, merge into, export and restore the resident ring, on an H100: the plans
of tests/ring_session_ops.py on every engine of tests/session_ops.py (own stream with PDL for auto, tma and ldg, own
stream without PDL, a caller-owned stream), checked against the plain model after every operation.

  * after every call that writes the ring (and after every failure) both planes are read back through
    gpr_resident_planes and compared with the model bit for bit, and gpr_resident_head with the model's head;
  * merges (text, decoded samples from pageable, pinned and device memory, XOR chunks from host and device memory) give
    the model's cells and its counts (n_in, n_oow, n_tiny);
  * there is no call that reads the block index, so it is read through gpr_resident_live_rows (which answers from a
    current index) and gpr_decide_resident in whole and early mode, after planted cells made every stale block
    maximum a wrong verdict or a wrong live row;
  * gpr_resident_export is byte-equal to tests/export_ref.py, and a second context restored from both planes' exports
    (maybe into another [P][G] through a pod table) holds the model's canonical window and decides like it;
  * decisions enqueued on the ring's planes retire, at the next gpr_sync or blocking decision, with the verdict of the
    ring when they were enqueued, whatever was appended, merged or remapped since, and gpr_step_stamps counts them;
  * every failure returns the ABI's code, writes none of its outputs, and leaves the ring, its head and the pending
    results as they were.
"""
import ctypes as C
import functools

import numpy as np
import pytest

import ring_scripts as RS
import ring_session_ops as RO
import session_ops as S
from test_gpu_geometry import DEV
from test_gpu_resident import decide, expected, same_verdict
from test_gpu_resident_export import _grid, _keep, _raw_export
from test_gpu_session import Call, Session, _engine, _span_array
from test_live_rows_emul import words_of

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")


@functools.lru_cache(maxsize=2)
def _replayed(seed):
    """(op, what it must give, the ring after it, stale, t_end) of every op of plan `seed` (shared by the engines)"""
    steps = []
    for op, out, md in RO.replay(RO.plan_ring(seed)):
        m = md.ring
        snap = None if m is None else ([p.copy() for p in m.planes], m.head, m.P, m.G, m.T, m.flags)
        steps.append((op, out, snap, md.stale, md.t_end))
    return steps


def _ring_of(snap):
    planes, head, P, G, T, flags = snap
    m = RS.Ring(P, G, T, flags)
    m.planes, m.head = [p.copy() for p in planes], head
    return m


def _guarded(n, kind):
    """n words of poison and GUARD guard words, host (numpy) or device (torch)"""
    if kind == "dev":
        return torch.full((n + S.GUARD,), S.POISON, dtype=torch.int32, device=DEV)
    return np.full(n + S.GUARD, S.POISON, np.uint32)


def _host_words(buf):
    return buf.cpu().numpy().view(np.uint32) if hasattr(buf, "cpu") else buf


class RingSession(Session):
    def __init__(self, eng, seed):
        super().__init__(eng, seed)
        self.twin = None

    # -- reading the device
    def read_ring(self, rows, T, n_planes):
        from gpu_pruner_b200 import ffi
        u, p, ld = self.eng.resident_planes()
        assert ld == T and (p is not None) == (n_planes > 1)
        out = []
        for ptr in (u, p)[:n_planes]:
            a = np.empty((rows, T), np.uint32)
            self.eng.memcpy(a, ptr, a.nbytes, ffi.GPR_MEM_HOST, ffi.GPR_MEM_DEVICE)
            out.append(a)
        return out

    def check_ring(self, snap, what):
        planes, head, P, G, T, _ = snap
        assert self.eng.resident_head() == head, (what, "head", self.eng.resident_head(), head)
        for pl, (got, want) in enumerate(zip(self.read_ring(P * G, T, len(planes)), planes)):
            if not np.array_equal(got, want):
                r, t = np.argwhere(got != want)[0]
                raise AssertionError(f"{what}: plane {pl} row {r} position {t}: {got[r, t]:#010x} != {want[r, t]:#010x}")

    # -- the ring calls
    def append(self, op, rows):
        from gpu_pruner_b200 import ffi
        u, p = RO.append_columns(op, rows)
        n = op["n_new"]
        ld = n + op["stride"] if op["stride"] else n

        def lay(a):
            x = np.full((rows, ld), np.float32(1e9), np.float32)
            x[:, :n] = a.view(np.float32)
            if op["src"] == "dev":
                t = torch.from_numpy(x).to(DEV)
                return t, t.data_ptr()
            return x, x.ctypes.data
        ku, pu = lay(u)
        kp, pp = lay(p) if p is not None else (None, None)
        torch.cuda.synchronize()
        rc = self.lib.gpr_append(self.h, pu, pp, n, ld if op["stride"] else 0,
                                 ffi.GPR_MEM_DEVICE if op["src"] == "dev" else ffi.GPR_MEM_HOST)
        self.expect_rc(rc, 0, "gpr_append")
        del ku, kp

    def merge(self, op, batch, n_rows, T, t_end, chunks=None):
        """one slice into the ring by op["src"] -> the counts (a GprError propagates)"""
        import gpu_pruner_b200 as g
        offsets, rows, ts, bits = batch
        src, pl = op["src"], op["plane"]
        thr = op["thr"] if pl == 1 else 0.0
        window = RO.merge_window(op, T)
        kw = dict(window_seconds=window, plane=pl, resident=True, power_threshold=thr)
        dev = g.ffi.GPR_MEM_DEVICE
        if src == "text":
            text, order = RO.text_of(offsets, rows, ts, bits)
            opens, closes = self.eng.text_scan(text, slot=1)
            assert len(opens) == len(order)
            sp = [(int(o) + 12, int(closes[np.searchsorted(closes, int(o) + 12)]) + 2, r) for o, r in zip(opens, order)]
            out = self.eng.text_parse(_span_array(sp), t_end, RO.STEP, T, n_rows, slot=1, **kw)
            assert not np.any(out["flags"] & 2), "a span went to the CPU parser"
            return {"n_in": int(out["n_in"].sum()), "n_oow": int(out["n_oow"].sum()), "n_tiny": int(out["n_tiny"].sum())}
        vals = bits.view(np.float64)
        if src == "samples_pageable":
            return self.eng.samples_scatter(offsets, rows, ts, vals, t_end, RO.STEP, T, n_rows, **kw)
        if src == "samples_pinned":
            pts, pvals = self.eng.host_array(ts.shape, np.int64), self.eng.host_array(vals.shape, np.float64)
            pts[:], pvals[:] = ts, vals
            return self.eng.samples_scatter(offsets, rows, pts, pvals, t_end, RO.STEP, T, n_rows, **kw)
        if src == "samples_dev":
            t = [torch.from_numpy(np.ascontiguousarray(a)).to(DEV) for a in
                 (offsets.view(np.int64), rows.view(np.int32), ts, vals)]
            torch.cuda.synchronize()
            return self.eng.samples_scatter(*t, t_end, RO.STEP, T, n_rows, mem_kind=dev, n_series=len(rows), **kw)
        sc, cb, data = chunks if chunks is not None else RO.slice_chunks(op, offsets, ts, bits)
        if src == "chunks_host":
            return self.eng.chunks_scatter(sc, rows, cb, data, t_end, RO.STEP, T, n_rows, **kw)
        t = [torch.from_numpy(np.ascontiguousarray(a)).to(DEV) for a in
             (sc.view(np.int64), rows.view(np.int32), cb.view(np.int64), data)]
        torch.cuda.synchronize()
        return self.eng.chunks_scatter(*t, t_end, RO.STEP, T, n_rows, mem_kind=dev, n_series=len(rows), **kw)

    def live_rows(self, rows, kind, mem_kind=None):
        """the raw call into a poisoned, guarded buffer -> (rc, words)"""
        from gpu_pruner_b200 import ffi
        n = (rows + 31) // 32
        buf = _guarded(n, kind)
        ptr = buf.data_ptr() if kind == "dev" else buf.ctypes.data
        if mem_kind is None:
            mem_kind = ffi.GPR_MEM_DEVICE if kind == "dev" else ffi.GPR_MEM_HOST
        rc = self.lib.gpr_resident_live_rows(self.h, C.c_void_p(ptr), mem_kind)
        torch.cuda.synchronize()
        w = _host_words(buf)
        assert np.all(w[n:] == np.uint32(S.POISON)), "guard words overwritten"
        return rc, w[:n]

    def remap_raw(self, op):
        from gpu_pruner_b200 import ffi
        src = np.asarray(op["src"], np.uint64).astype(np.uint32)
        if op.get("mem", "host") == "dev" or op.get("fail", "").endswith("_dev"):
            t = torch.from_numpy(src.view(np.int32)).to(DEV)
            torch.cuda.synchronize()
            return self.lib.gpr_resident_remap(self.h, op["P"], op["G"], C.c_void_p(t.data_ptr()), ffi.GPR_MEM_DEVICE)
        return self.lib.gpr_resident_remap(self.h, op["P"], op["G"], src.ctypes.data_as(C.c_void_p), ffi.GPR_MEM_HOST)

    def export(self, op, want, t_end):
        got = self.eng.resident_export(t_end, RO.STEP, plane=op["plane"], max_per_chunk=op["M"])
        sc, rows, cb, data, n = want
        for name, a, b in (("series_chunks", got["series_chunks"], sc), ("rows", got["rows"], rows),
                           ("chunk_bytes", got["chunk_bytes"], cb), ("data", got["data"], data)):
            assert np.array_equal(a, b), (name, "export differs from tests/export_ref.py")
        assert got["n_samples"] == n
        return got

    def restore(self, op, out, snap, t_end):
        import gpu_pruner_b200 as g
        planes, head, P, G, T, flags = snap
        m = _ring_of(snap)
        if self.twin is None:
            self.twin = g.IdleEngine(device=0)
        exports = [self.export(dict(plane=pl, M=120), out["exports"][pl], t_end) for pl in range(len(planes))]
        new_row = RO.twin_rows(op, m)
        tw = out["twin"]
        self.twin.resident_init(op["P"], op["G"], T, power_plane=bool(flags & 1), block_index=op["index"])
        for pl, ex in enumerate(exports):
            sc, rr, cb, data = _keep(ex, new_row[ex["rows"]])
            gr = ex["grid"]
            self.twin.chunks_scatter(sc, rr, cb, data, gr["t_end"], gr["step"], T, op["P"] * op["G"], plane=pl,
                                     resident=True, window_seconds=gr["window_seconds"])
        self.twin.resident_reindex()
        assert self.twin.resident_head() == 0
        u, p, _ = self.twin.resident_planes()
        for pl, ptr in enumerate((u, p)[:len(planes)]):
            a = np.empty((op["P"] * op["G"], T), np.uint32)
            self.twin.memcpy(a, ptr, a.nbytes, 0, 1)
            if not np.array_equal(a, tw.planes[pl]):
                r, t = np.argwhere(a != tw.planes[pl])[0]
                raise AssertionError(f"restored plane {pl} row {r} column {t}: {a[r, t]:#010x} != {tw.planes[pl][r, t]:#010x}")
        exp = expected(tw)
        for early in (False, True):
            bad = same_verdict(decide(self.twin, tw, early=early), exp)
            assert bad is None, ("the restored ring decides unlike the model", early, bad)

    def ring_async(self, op, out, snap):
        planes, head, P, G, T, _ = snap
        u, p, _ = self.eng.resident_planes()
        w0, w1 = out["window"]
        for spec in op["calls"]:
            rng = np.random.default_rng(spec["seed"])
            d = dict(util=w0, power=w1 if spec["thr"] else None, eligible=None, created_ts=None, cutoff_ts=0, table=None)
            if spec["gates"]:
                d["eligible"] = (rng.random(P) < 0.9).astype(np.uint8)
                d["created_ts"] = rng.integers(1000, 2000, P).astype(np.int64)
                d["cutoff_ts"] = 1500
            if spec["table"]:
                d["table"] = S.R.random_table(rng, P, G, share=0.7)
            w = dict(src="dev", P=P, G=G, T=T, thr=spec["thr"], gates=spec["gates"], table=spec["table"],
                     outs=spec["outs"], out_kind=spec["out_kind"], seed=0)
            c = Call(self.eng, w, data=d)
            c.win.util, c.win.power = u, (p if spec["thr"] else None)
            c.win.row_stride = 0
            self.enqueue(c)

    # -- failures
    def ring_fail(self, op, out, snap, t_end):
        import gpu_pruner_b200 as g
        f, code = op["fail"], op["code"]
        if f in ("remap_no_ring", "live_no_ring"):
            if f == "remap_no_ring":
                self.expect_rc(self.remap_raw(op), code, f)
            else:
                rc, w = self.live_rows(4, "host")
                self.expect_rc(rc, code, f)
                assert np.all(w == np.uint32(S.POISON)), (f, "bits written")
            return
        planes, head, P, G, T, _ = snap
        if f.startswith("remap_"):
            self.expect_rc(self.remap_raw(op), code, f)
            assert f"src_rows[{out['first_bad']}]" in self.err(), (f, self.err(), out["first_bad"])
        elif f == "live_bad_kind":
            rc, w = self.live_rows(P * G, "host", mem_kind=7)
            self.expect_rc(rc, code, f)
            assert np.all(w == np.uint32(S.POISON)), (f, "bits written")
        elif f.startswith("export_"):
            from gpu_pruner_b200 import ffi
            if f == "export_capacity":
                sc, rows, cb, data, n = out["export"]
                true = [len(rows), len(cb) - 1, len(data)]
                caps = list(true)
                caps[["series", "chunks", "bytes"].index(op["short"])] -= 1
            else:
                true, caps = [0, 0, 0], [4, 4, 64]
            arrays = [np.full(caps[0] + 1 + S.GUARD, 0x7BADBEEF7BADBEEF, np.uint64),
                      np.full(caps[0] + S.GUARD, S.POISON, np.uint32),
                      np.full(caps[1] + 1 + S.GUARD, 0x7BADBEEF7BADBEEF, np.uint64),
                      np.full(caps[2] + S.GUARD, 0xEF, np.uint8)]
            grid = _grid(op.get("T", T), t_end=t_end, step=RO.STEP, window_seconds=T * RO.STEP)
            rc, o = _raw_export(self.eng, grid, op["plane"], op["M"], arrays, ffi.GPR_MEM_HOST, caps=caps)
            self.expect_rc(rc, code, f)
            if f == "export_capacity":
                assert [o.n_series, o.n_chunks, o.n_bytes, o.n_samples] == true + [out["export"][4]], (f, "counts")
            for a, poison in zip(arrays, (0x7BADBEEF7BADBEEF, S.POISON, 0x7BADBEEF7BADBEEF, 0xEF)):
                assert np.all(a == poison), (f, "an array was written")
        elif f in ("merge_bad_row", "merge_truncated", "merge_no_power", "merge_rows_over"):
            if f != "merge_rows_over":      # (the slice of a merge whose grid is refused, without its advance)
                self.eng.resident_advance(op["n_new"])
            offsets, rows, ts, bits = RO.merge_slice(op, T, t_end)
            chunks = None
            n_rows = op["n_rows"]
            if f == "merge_bad_row":
                rows = rows.copy()
                rows[op["bad_series"]] = n_rows
            elif f == "merge_truncated":
                sc, rows, cb, data = out["batch"]
                chunks = (sc, cb, data)
            with pytest.raises(g.GprError) as ei:
                self.merge(op, (offsets, rows, ts, bits), n_rows, T, t_end, chunks=chunks)
            assert ei.value.code == code, (f, ei.value.code, str(ei.value))
            if f == "merge_truncated":
                assert f"chunk {op['chunk']} is the first malformed one" in str(ei.value), str(ei.value)
        elif f == "decide_stale":
            self.ring = _ring_of(snap)
            self.decide_resident(dict(mode="early"), fail=f)
        else:
            raise AssertionError(f)

    def step(self, op, out, snap, stale, t_end):
        from gpu_pruner_b200 import ffi
        k = op["kind"]
        if k == "async":
            self.enqueue(Call(self.eng, op["win"]))
        elif k == "init":
            r = op["ring"]
            self.eng.resident_init(r["P"], r["G"], r["T"], power_plane=r["power"], block_index=r["index"])
        elif k == "append":
            self.append(op, snap[2] * snap[3])
        elif k == "advance":
            self.eng.resident_advance(op["n_new"])
        elif k == "merge":
            planes, head, P, G, T, _ = snap
            self.eng.resident_advance(op["n_new"])
            got = self.merge(op, RO.merge_slice(op, T, t_end), op["n_rows"], T, t_end)
            want = dict(zip(("n_in", "n_oow", "n_tiny"), out["stats"]))
            assert got == want, ("merge counts", got, want)
        elif k == "plant":
            planes = snap[0]
            u, p, _ = self.eng.resident_planes()
            for ptr, cells in zip((u, p), planes):
                self.eng.memcpy(ptr, np.ascontiguousarray(cells), cells.nbytes, ffi.GPR_MEM_DEVICE, ffi.GPR_MEM_HOST)
            if snap[5] & 2:
                self.eng.resident_reindex()
        elif k == "live_rows":
            rc, w = self.live_rows(snap[2] * snap[3], op["out"])
            self.expect_rc(rc, 0, "gpr_resident_live_rows")
            want = words_of(out["live"])
            bad = np.flatnonzero(w != want)
            assert bad.size == 0, ("live rows", "stale index" if stale else "current index", int(bad[0]),
                                   hex(int(w[bad[0]])), hex(int(want[bad[0]])))
        elif k == "remap":
            self.expect_rc(self.remap_raw(op), 0, "gpr_resident_remap")
            self.eng._res_rows = op["P"] * op["G"]
        elif k == "export":
            self.export(op, out["export"], t_end)
        elif k == "restore":
            self.restore(op, out, snap, t_end)
        elif k == "ring_async":
            self.ring_async(op, out, snap)
        elif k == "sync":
            self.sync()
        elif k == "reindex":
            self.eng.resident_reindex()
        elif k == "decide_resident":
            self.ring = _ring_of(snap)
            self.decide_resident(op)
        elif k == "fail":
            self.ring_fail(op, out, snap, t_end)
        else:
            raise AssertionError(k)
        if snap is not None and (k in RO.WRITES_RING or k == "fail"):
            self.check_ring(snap, "the ring after the call")


def _describe(op):
    keys = ("fail", "src", "plane", "n_new", "n_rows", "how", "mem", "P", "G", "M", "out", "open")
    return op["kind"] + " " + " ".join(f"{k}={op[k]}" for k in keys if k in op)


@pytest.mark.parametrize("eid", [e[0] for e in S.ENGINES])
@pytest.mark.parametrize("seed", RO.SEEDS)
def test_ring_sequence(eid, seed):
    eng, stream = _engine(eid)
    s = RingSession(eng, seed)
    try:
        for i, (op, out, snap, stale, t_end) in enumerate(_replayed(seed)):
            try:
                s.step(op, out, snap, stale, t_end)
            except AssertionError as e:
                raise AssertionError(f"engine {eid}, seed {seed}, step {i}: {_describe(op)}: {e}") from None
        s.sync()
        assert s.retired > 0
    finally:
        eng.close()
        if s.twin is not None:
            s.twin.close()
        if stream is not None:
            stream.synchronize()
