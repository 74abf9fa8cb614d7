"""One context through whole sessions on an H100: the seeded call sequences of tests/session_ops.py, each on a fresh
IdleEngine, checked against plain references after every operation that completes work; and the caller-owned stream,
where stream order alone must put the library's work after the caller's.

Every engine stages host windows in 1 MB chunks (GPR_CHUNK_MB=1), so a host window spans many chunks.  Every output
buffer is its own allocation, filled with poison and followed by guard words; every gpr_result starts with sentinel
counters.  A result is checked when a gpr_sync or a successful blocking call retires it: counters, bitmaps (padding
bits included), series_max, veto_bits and idle_slots, and the number of gpr_step_stamps equals the number of
decisions retired.  A failing call must return the ABI's code, write none of its outputs and leave every earlier
result pending, to be retired right by the next gpr_sync or blocking call.
"""
import ctypes as C
import threading

import numpy as np
import pytest

import kat
import ring_scripts as RS
import session_ops as S
from test_gpu_geometry import DEV, _environ

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")


def _engine(eid):
    import gpu_pruner_b200 as g
    if not torch.cuda.is_available():
        pytest.fail("-m gpu tests need a CUDA device; the engine has no CPU fallback")
    _, stream, pdl, kernel = next(e for e in S.ENGINES if e[0] == eid)
    s = torch.cuda.Stream() if stream == "caller" else None
    with _environ({"GPR_PDL": str(pdl), "GPR_CHUNK_MB": "1"}):
        eng = g.IdleEngine(device=0, kernel=kernel, max_pods=S.MAX_CELLS, max_gpus=1, max_samples=1, power_plane=True,
                           stream=None if s is None else s.cuda_stream)
    return eng, s


# ---- buffers ---------------------------------------------------------------------------------------------------
def _poisoned(n, kind, f32=False):
    """n words of poison and GUARD guard words, on the device or in pinned host memory"""
    dtype = torch.float32 if f32 else torch.int32
    v = float(S.POISON_F32) if f32 else S.POISON
    if kind == "dev":
        return torch.full((n + S.GUARD,), v, dtype=dtype, device=DEV)
    return torch.empty((n + S.GUARD,), dtype=dtype, pin_memory=True).fill_(v)


def _words(t):
    return (t.cpu() if t.is_cuda else t).numpy().view(np.uint32)


POISON_BITS = {False: np.uint32(S.POISON), True: np.float32(S.POISON_F32).view(np.uint32)}


class Call:
    """one decision: its window and result structs, every buffer it references, and what it must return"""

    def __init__(self, eng, w, data=None, expected=None):
        from gpu_pruner_b200 import ffi
        import gpu_pruner_b200 as g
        self.w = w
        self.keep = []
        d = data if data is not None else S.window_data(w)
        self._d = d
        self._expected = expected
        P, G, T = w["P"], w["G"], w["T"]
        src = w["src"]
        u8 = S.is_u8(src)
        util = g.to_biased_u8(d["util"]) if u8 else d["util"]
        ld = T + 3 if src == "dev_strided" else T
        off = 1 if src == "dev_misaligned" else 0
        if src.startswith("dev"):
            def put(a, fill):
                return self._dev(a, fill, ld, off)
            in_kind = ffi.GPR_MEM_DEVICE
            up = put(util, 0x55 if u8 else 77.0)
            pp = put(d["power"], 1e9) if d["power"] is not None else None
            el = self._keep(torch.from_numpy(d["eligible"]).to(DEV)) if d["eligible"] is not None else None
            cr = self._keep(torch.from_numpy(d["created_ts"]).to(DEV)) if d["created_ts"] is not None else None
            tb = self._keep(torch.from_numpy(d["table"].astype(np.int32)).to(DEV)) if d["table"] is not None else None
        else:
            in_kind = ffi.GPR_MEM_HOST
            pin = src.startswith("pin")

            def host(a):
                if a is None:
                    return None
                a = np.ascontiguousarray(a)
                if a.dtype == np.uint32:
                    a = a.view(np.int32)
                if pin:
                    t = torch.from_numpy(a).pin_memory()
                    self.keep.append(t)
                    return t.data_ptr()
                self.keep.append(a)
                return a.ctypes.data
            up, pp = host(util), host(d["power"])
            el, cr, tb = host(d["eligible"]), host(d["created_ts"]), host(d["table"])
        self.win = eng._window(up, pp, el, cr, d["cutoff_ts"], P, G, T, ld if ld != T else 0, w["thr"], in_kind,
                               ffi.GPR_FMT_U8B if u8 else ffi.GPR_FMT_F32, tb)
        self.res = ffi.gpr_result()
        self.res.struct_size = C.sizeof(ffi.gpr_result)
        self.res.out_mem_kind = ffi.GPR_MEM_HOST if w["out_kind"] == "host" else ffi.GPR_MEM_DEVICE
        self.set_outputs(P, G, w["outs"], w["out_kind"])

    def _keep(self, t):
        self.keep.append(t)
        return t.data_ptr()

    def _dev(self, a, fill, ld, off):
        P, G, T = a.shape
        flat = np.full((P * G * ld + off + 4,), fill, a.dtype)
        flat[off:off + P * G * ld].reshape(P * G, ld)[:, :T] = a.reshape(P * G, T)
        t = torch.from_numpy(flat).to(DEV)
        self.keep.append(t)
        return t.data_ptr() + off * flat.itemsize

    def set_outputs(self, P, G, outs, kind):
        W, MW = (P + 31) // 32, (G + 31) // 32
        self.bufs = {"decision_bits": (_poisoned(W, kind), W, False)}
        if outs["cand"]:
            self.bufs["candidate_bits"] = (_poisoned(W, kind), W, False)
        if outs["smax"]:
            self.bufs["series_max"] = (_poisoned(P * G, kind, True), P * G, True)
        if outs["veto"]:
            self.bufs["veto_bits"] = (_poisoned(W, kind), W, False)
        if outs["islots"]:
            self.bufs["idle_slots"] = (_poisoned(P * MW, kind), P * MW, False)
        for name in ("decision_bits", "candidate_bits", "series_max", "veto_bits", "idle_slots"):
            setattr(self.res, name, self.bufs[name][0].data_ptr() if name in self.bufs else None)
        self.res.n_series = self.res.n_candidates = self.res.n_decisions = S.SENTINEL

    def expected(self):
        if self._expected is None:
            d = self._d
            self._expected = S.expected(d["util"], d["power"], self.w["thr"], d["eligible"], d["created_ts"],
                                        d["cutoff_ts"], d["table"])
        return self._expected

    def check_done(self, what):
        e = self.expected()
        r = self.res
        assert (r.n_series, r.n_candidates, r.n_decisions) == (e["n_series"], e["n_candidates"], e["n_decisions"]), \
            (what, "counters", (r.n_series, r.n_candidates, r.n_decisions))
        for name, (t, n, f32) in self.bufs.items():
            got = _words(t)
            assert np.all(got[n:] == POISON_BITS[f32]), (what, name, "guard words overwritten")
            want = e[name]
            if name == "series_max":
                assert kat.smax_equal(got[:n].view(np.float32), want.ravel()), (what, name)
            else:
                bad = np.flatnonzero(got[:n] != np.asarray(want, np.uint32).ravel())
                assert bad.size == 0, (what, name, int(bad[0]), hex(int(got[bad[0]])),
                                       hex(int(np.asarray(want).ravel()[bad[0]])))

    def check_untouched(self, what, counters=True):
        if counters:
            r = self.res
            assert (r.n_series, r.n_candidates, r.n_decisions) == (S.SENTINEL,) * 3, (what, "counters written")
        for name, (t, n, f32) in self.bufs.items():
            assert np.all(_words(t) == POISON_BITS[f32]), (what, name, "written by a call that failed")

    def check_guards(self, what):
        for name, (t, n, f32) in self.bufs.items():
            assert np.all(_words(t)[n:] == POISON_BITS[f32]), (what, name, "guard words overwritten")


# ---- one sequence ----------------------------------------------------------------------------------------------
class Session:
    def __init__(self, eng, seed):
        self.eng, self.lib, self.h = eng, eng._lib, eng.handle
        self.seed = seed
        self.pending = []       # Calls enqueued and not yet retired
        self.untouched = []     # Calls a failure must never write
        self.ring = None
        self.t_end = S.T_END
        self.retired = 0

    def err(self):
        return (self.lib.gpr_last_error(self.h) or b"").decode()

    def call(self, fn, *args):
        return fn(self.h, *args)

    def expect_rc(self, rc, want, what):
        assert rc == want, (what, rc, want, self.err())

    def retire(self, calls, what):
        """calls were retired by a gpr_sync / blocking call: check each, and the number of stamps"""
        _, stamps = self.eng.step_stamps()
        assert len(stamps) == len(calls), (what, "stamps", len(stamps), len(calls))
        torch.cuda.synchronize()
        for k, c in enumerate(calls):
            if c.w.get("table") == "bad":
                c.check_guards((what, k))
            else:
                c.check_done((what, "retired result", k))
        for c in self.untouched:
            c.check_untouched((what, "a failed call's outputs"))
        self.untouched = []
        self.retired += len(calls)

    def decide(self, w):
        c = Call(self.eng, w)
        torch.cuda.synchronize()
        self.expect_rc(self.call(self.lib.gpr_decide, C.byref(c.win), C.byref(c.res)), 0, "gpr_decide")
        done, self.pending = self.pending + [c], []
        self.retire(done, "blocking decision")

    def enqueue(self, c):
        torch.cuda.synchronize()
        self.expect_rc(self.call(self.lib.gpr_decide_async, C.byref(c.win), C.byref(c.res)), 0, "gpr_decide_async")
        self.pending.append(c)

    def batch(self, calls, fail_at=None, how=None):
        from gpu_pruner_b200 import ffi
        n = len(calls)
        wins, ress = (ffi.gpr_window * n)(), (ffi.gpr_result * n)()
        for i, c in enumerate(calls):
            if i == fail_at:
                if how == "row_stride":
                    c.win.row_stride = c.w["T"] - 1
                else:
                    c.win.struct_size = 12
            C.memmove(C.byref(wins, i * C.sizeof(ffi.gpr_window)), C.byref(c.win), C.sizeof(ffi.gpr_window))
            C.memmove(C.byref(ress, i * C.sizeof(ffi.gpr_result)), C.byref(c.res), C.sizeof(ffi.gpr_result))
            c.res = ress[i]             # the library writes the array's element
            c.keep.append((wins, ress))
        torch.cuda.synchronize()
        rc = self.lib.gpr_decide_batch_async(self.h, wins, ress, n)
        if fail_at is None:
            self.expect_rc(rc, 0, "gpr_decide_batch_async")
            self.pending += calls
        else:
            self.expect_rc(rc, S.E_INVALID, ("batch failing at", fail_at))
            self.pending += calls[:fail_at]
            self.untouched += calls[fail_at:]

    def sync(self, want=0):
        rc = self.lib.gpr_sync(self.h)
        self.expect_rc(rc, want, "gpr_sync")
        done, self.pending = self.pending, []
        self.retire(done, "gpr_sync")

    # -- the resident ring
    def resident_init(self, r):
        self.eng.resident_init(r["P"], r["G"], r["T"], power_plane=r["power"], block_index=r["index"])
        self.ring = RS.Ring(r["P"], r["G"], r["T"], (1 if r["power"] else 0) | (2 if r["index"] else 0))

    def append(self, op):
        m = self.ring
        n, ld = op["n_new"], op["stride"] or op["n_new"]
        u, p = S.ring_columns(op["seed"], m.rows, n, op["power_cols"])

        def lay(a):
            x = np.full((m.rows, ld), 1e9, np.float32)
            x[:, :n] = a
            if op["src"] == "dev":
                t = torch.from_numpy(x).to(DEV)
                return t, t.data_ptr()
            return x, x.ctypes.data
        ku, pu = lay(u)
        kp, pp = lay(p) if p is not None else (None, None)
        torch.cuda.synchronize()
        rc = self.lib.gpr_append(self.h, pu, pp, n, op["stride"], 1 if op["src"] == "dev" else 0)
        self.expect_rc(rc, 0, "gpr_append")
        del ku, kp
        m.append(n, u.view(np.uint32), None if p is None else p.view(np.uint32))

    def text_resident(self, op):
        m = self.ring
        self.t_end += op["n_new"] * S.STEP
        spans, window = S.ring_after_slice(m, op, self.t_end)
        self.eng.resident_advance(op["n_new"])
        if not spans:
            return
        text, sp = S.text_bytes(spans)
        self.eng.text_scan(text, slot=1)
        out = self.eng.text_parse(_span_array(sp), self.t_end, S.STEP, m.T, m.rows, slot=1, resident=True,
                                  window_seconds=window)
        assert not np.any(out["flags"] & 2), "a plain sample was declined"
        assert self.eng.resident_head() == m.head

    def decide_resident(self, op, fail=None):
        from gpu_pruner_b200 import ffi
        m = self.ring
        P, G, T = (m.P, m.G, m.T) if m is not None else (3, 4, 4)
        rng = np.random.default_rng(op.get("seed", 0))
        util = m.window(0) if m is not None else np.zeros((P, G, T), np.float32)
        power = m.window(1) if m is not None and len(m.planes) > 1 and op.get("thr") else None
        d = dict(util=util, power=power, eligible=None, created_ts=None, cutoff_ts=0, table=None)
        if op.get("gates"):
            d["eligible"] = (rng.random(P) < 0.9).astype(np.uint8)
            d["created_ts"] = rng.integers(1000, 2000, P).astype(np.int64)
            d["cutoff_ts"] = 1500
        if op.get("table"):
            d["table"] = S.R.random_table(rng, P, G, share=0.7)
        whole = op.get("mode") == "whole"
        kind = "host" if rng.random() < 0.5 else "dev"
        w = dict(src="dev" if op.get("gates_kind", "dev") == "dev" else "pageable", P=P, G=G, T=T, thr=op.get("thr"),
                 gates=bool(op.get("gates")), table=bool(op.get("table")), out_kind=kind, seed=0,
                 outs=dict(cand=True, smax=whole, veto=bool(rng.random() < 0.5), islots=not whole or rng.random() < .5))
        c = Call(self.eng, w, data=d)
        c.win.util = c.win.power = None
        torch.cuda.synchronize()
        rc = self.lib.gpr_decide_resident(self.h, C.byref(c.win), C.byref(c.res))
        if fail:
            self.expect_rc(rc, S.E_STATE, fail)
            self.untouched.append(c)
            return
        self.expect_rc(rc, 0, "gpr_decide_resident")
        done, self.pending = self.pending + [c], []
        self.retire(done, "resident decision")

    # -- the text planes
    def text_planes(self, op):
        P, G, T, thr = op["P"], op["G"], op["T"], op["thr"]
        us, ws, u, wc = S.plane_text(op["seed"], P, G, T, thr)
        for slot, plane, spans in ((0, 0, us), (2, 1, ws)):
            if spans is None:
                continue
            text, sp = S.text_bytes(spans)
            self.eng.text_scan(text, slot=slot)
            out = self.eng.text_parse(_span_array(sp), S.T_END, S.STEP, T, P * G, slot=slot, plane=plane,
                                      power_threshold=thr if plane else 0.0)
            assert not np.any(out["flags"] & 2) and int(out["n_in"].sum()) == sum(len(s) for _, s in spans)
        pu, pw = self.eng.text_planes()
        exp = S.expected(u, wc, thr)
        for dspec in op["decisions"]:
            w = dict(src="dev", P=P, G=G, T=T, thr=thr, gates=False, table=False, seed=0, outs=dspec["outs"],
                     out_kind=dspec["out_kind"])
            c = Call(self.eng, w, data=dict(util=u, power=wc, eligible=None, created_ts=None, cutoff_ts=0, table=None),
                     expected=exp)
            c.win.util, c.win.power = pu, (pw if thr else None)
            c.win.row_stride = 0
            self.enqueue(c)

    # -- failures
    def fail(self, op):
        f, code = op["fail"], op["code"]
        import gpu_pruner_b200 as g
        if f in ("struct_size", "row_stride", "bad_host_table"):
            w = dict(op["win"])
            d = S.window_data(w)
            if f == "bad_host_table":
                d["table"] = d["table"].copy()
                d["table"][int(d["table"].shape[0]) // 2, 2] = 3
            c = Call(self.eng, w, data=d)
            if f == "struct_size":
                c.win.struct_size = 12
            elif f == "row_stride":
                c.win.row_stride = w["T"] - 1
            torch.cuda.synchronize()
            self.expect_rc(self.lib.gpr_decide(self.h, C.byref(c.win), C.byref(c.res)), code, f)
            self.untouched.append(c)
        elif f in ("g257", "over_capacity"):
            P, G, T = (1, 257, 4) if f == "g257" else (1, 1, S.MAX_CELLS + 1)
            w = dict(src="pageable", P=P, G=G, T=T, thr=None, gates=False, table=False, seed=0, out_kind="host",
                     outs=dict(cand=True, smax=True, veto=True, islots=True))
            d = dict(util=np.zeros((P, G, T), np.float32), power=None, eligible=None, created_ts=None, cutoff_ts=0,
                     table=None)
            c = Call(self.eng, w, data=d)
            self.expect_rc(self.lib.gpr_decide(self.h, C.byref(c.win), C.byref(c.res)), code, f)
            self.untouched.append(c)
        elif f == "resident_no_ring":
            assert self.ring is None
            self.decide_resident({}, fail=f)
        elif f == "resident_stale":
            self.decide_resident(dict(op, mode="early"), fail=f)
        elif f == "batch_fail":
            self.batch([Call(self.eng, w) for w in op["wins"]], fail_at=op["k"], how=op["how"])
        elif f == "async_bad_device_table":
            for w in op["before"]:
                self.enqueue(Call(self.eng, w))
            self.enqueue(Call(self.eng, op["win"]))
            for w in op["after"]:
                self.enqueue(Call(self.eng, w))
            self.sync(want=code)
        elif f == "slots_full":
            data = [(w, S.window_data(w)) for w in op["wins"]]
            exps = [S.expected(d["util"], d["power"], w["thr"], d["eligible"], d["created_ts"], d["cutoff_ts"], None)
                    for w, d in data]
            k = 0
            while len(self.pending) < S.MAX_PENDING:
                w, d = data[k % len(data)]
                self.enqueue(Call(self.eng, w, data=d, expected=exps[k % len(data)]))
                k += 1
            w, d = data[0]
            extra = Call(self.eng, w, data=d)
            torch.cuda.synchronize()
            self.expect_rc(self.lib.gpr_decide_async(self.h, C.byref(extra.win), C.byref(extra.res)), code,
                           "257th async result")
            blocking = Call(self.eng, w, data=d)
            self.expect_rc(self.lib.gpr_decide(self.h, C.byref(blocking.win), C.byref(blocking.res)), code,
                           "blocking call with 256 results pending")
            self.untouched += [extra, blocking]
            self.sync()
        else:
            raise AssertionError(f)

    def run(self, op):
        k = op["kind"]
        if k == "decide":
            self.decide(op["win"])
        elif k == "async":
            self.enqueue(Call(self.eng, op["win"]))
        elif k == "batch":
            self.batch([Call(self.eng, w) for w in op["wins"]])
        elif k == "sync":
            self.sync()
        elif k == "resident_init":
            self.resident_init(op["ring"])
        elif k == "append":
            self.append(op)
        elif k == "advance":
            self.eng.resident_advance(op["n_new"])
            self.ring.advance(op["n_new"])
        elif k == "text_resident":
            self.text_resident(op)
        elif k == "reindex":
            self.eng.resident_reindex()
        elif k == "decide_resident":
            self.decide_resident(op)
        elif k == "text_planes":
            self.text_planes(op)
        elif k == "fail":
            self.fail(op)
        else:
            raise AssertionError(k)


def _span_array(sp):
    import gpu_pruner_b200 as g
    out = np.zeros(len(sp), g.IdleEngine.SPAN_DTYPE)
    for i, (b, e, r) in enumerate(sp):
        out[i]["begin"], out[i]["end"], out[i]["row"] = b, e, r
    return out


def _describe(op):
    k = op["kind"]
    if "win" in op:
        w = op["win"]
        return f"{k} {op.get('fail', '')} {w['src']} {w['P']}x{w['G']}x{w['T']} thr={w['thr']} table={w['table']}"
    return f"{k} {op.get('fail', '')}".strip()


@pytest.mark.parametrize("seed", S.SEEDS)
@pytest.mark.parametrize("eid", [e[0] for e in S.ENGINES])
def test_call_sequence(eid, seed):
    eng, stream = _engine(eid)
    try:
        s = Session(eng, seed)
        ops = S.plan(seed)
        for i, op in enumerate(ops):
            try:
                s.run(op)
            except AssertionError as e:
                raise AssertionError(f"engine {eid}, seed {seed}, step {i}: {_describe(op)}: {e}") from None
        s.sync()
        assert s.retired > 0
    finally:
        eng.close()
        if stream is not None:
            stream.synchronize()


# ---- the caller-owned stream, deterministically ----------------------------------------------------------------
SLEEP_CYCLES = 100_000_000      # about 50 ms at the H100's clocks


def test_caller_stream_orders_the_library_after_the_callers_work():
    """on the caller's stream s, with no host synchronisation between the steps: a 50 ms sleep kernel, a torch write
    of the input, the library call on it, a torch copy of the output.  A library that ran on a stream of its own would
    read the input before the write.  The steps run from two Python threads in turn (the context is thread-agnostic);
    after gpr_destroy, s must still work."""
    import gpu_pruner_b200 as g
    from gpu_pruner_b200 import ffi
    s = torch.cuda.Stream()
    with _environ({"GPR_CHUNK_MB": "1"}):
        eng = g.IdleEngine(device=0, stream=s.cuda_stream)
    P, G, T = 1000, 4, 180
    W = (P + 31) // 32
    rng = np.random.default_rng(1)
    new = np.zeros((P, G, T), np.float32)
    new[rng.random(P) < 0.5, 0, 7] = 5.0
    want = S.expected(new)
    lock = threading.Lock()
    results = {}

    def decide_step():
        u = torch.full((P, G, T), 9.0, device=DEV)                 # the old window: every pod busy
        new_t = torch.from_numpy(new).to(DEV)
        db = torch.full((W,), S.POISON, dtype=torch.int32, device=DEV)
        torch.cuda.synchronize()
        with torch.cuda.stream(s):
            torch.cuda._sleep(SLEEP_CYCLES)
            u.copy_(new_t)
            eng.decide_ptr(u, P, G, T, db, blocking=False)
            results["bits"] = db.clone()
        eng.sync()
        results["keep"] = (u, new_t, db)

    rows, T_r = 6, 64

    def append_step():
        eng.resident_init(rows, 1, T_r)
        cols = torch.full((rows, T_r), 3.0, device=DEV)            # busy columns, overwritten on s
        torch.cuda.synchronize()
        with torch.cuda.stream(s):
            torch.cuda._sleep(SLEEP_CYCLES)
            cols[::2].zero_()
            eng.append(cols.data_ptr(), None, n_new=T_r, mem_kind=ffi.GPR_MEM_DEVICE)
        db = np.zeros(1, np.uint32)
        r = eng.decide_ptr(None, rows, 1, T_r, db, in_kind=0, out_kind=0, resident=True)
        results["append"] = (int(db[0]), r.n_decisions)

    decoy = b" " * 4096
    real = bytearray(decoy)
    marks = [100, 1000, 3000]
    for m in marks:
        real[m:m + 12] = b'},"values":['

    def scan_step():
        t = torch.from_numpy(np.frombuffer(decoy, np.uint8).copy()).to(DEV)
        real_t = torch.from_numpy(np.frombuffer(bytes(real), np.uint8).copy()).to(DEV)
        torch.cuda.synchronize()
        with torch.cuda.stream(s):
            torch.cuda._sleep(SLEEP_CYCLES)
            t.copy_(real_t)
            opens, _ = eng.text_scan(t.data_ptr(), slot=0, n_bytes=len(real), mem_kind=ffi.GPR_MEM_DEVICE)
        results["scan"] = opens.tolist()

    errors = []

    def run(step):
        with lock:
            try:
                step()
            except BaseException as e:     # reported by the main thread
                errors.append(e)
    for step in (decide_step, append_step, scan_step):
        th = threading.Thread(target=run, args=(step,))
        th.start()
        th.join()
    assert not errors, errors
    got = results["bits"].cpu().numpy().view(np.uint32)
    assert np.array_equal(got, want["decision_bits"]), "the decision read the window before the caller's write"
    assert results["append"] == (0b010101, 3), results["append"]
    assert results["scan"] == [m + 0 for m in marks], results["scan"]
    eng.close()
    with torch.cuda.stream(s):               # the library did not destroy the caller's stream
        x = torch.ones(1024, device=DEV) * 2
    s.synchronize()
    assert float(x.sum()) == 2048.0
