"""GPU: whole context lifetimes (gpr_create .. gpr_destroy, gpu-pruner_b200/csrc/gpr_api.cu).  Every buffer, event and
stream a context makes is a member that releases itself, and gpr_destroy first stops whatever could still use them:
  * cycles: ten contexts in turn, each through a host decision with gates, groups, series_max and idle_slots, an async
    batch and gpr_sync, gpr_resident_init twice with the block index, append, advance and a resident decision, a text
    scan from pageable and from pinned memory and its parse, gpr_samples_scatter from host and from device memory,
    gpr_flush_l2 and the timer.  Every result equals the references the other suites use (the C oracle, groups_ref,
    the ring model, the regex's markers), and the device memory NVML charges to this process after the last cycle
    equals that after the first;
  * a context destroyed while its scan of a 160 MB pageable text is still uploading on 8 threads: a new context scans
    and parses the same text to the same markers and cells, and the device still works;
  * gpr_create failing after its first allocations (a bad kernel_variant), ten times: each returns GPR_E_INVALID and a
    good create afterwards decides right."""
import ctypes as C
import os
import re
import warnings

import numpy as np
import pytest

import kat
import ring_scripts as RS
import session_ops as S
from test_gpu_geometry import DEV, _environ
from test_gpu_text_scan import PRE, REC, STEP as SCAN_STEP, T_END as SCAN_T_END, _big_template, _digits

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

MB = 1 << 20
OPEN, CLOSE = b'},"values":[', b'"]]'
CYCLES = 10
MEM_TOL = 8 * MB                 # a per-cycle leak of 1 MB adds up to 9 MB over the cycles after the first


def _engine(env=None, **kw):
    import gpu_pruner_b200 as g
    if not torch.cuda.is_available():
        pytest.fail("-m gpu tests need a CUDA device; the engine has no CPU fallback")
    with _environ(env or {}):
        return g.IdleEngine(device=0, **kw)


# ---- the device memory NVML charges to this process -------------------------------------------------------------
class _ProcInfo(C.Structure):
    _fields_ = [("pid", C.c_uint), ("usedGpuMemory", C.c_ulonglong), ("gpuInstanceId", C.c_uint),
                ("computeInstanceId", C.c_uint)]


def _process_bytes():
    """-> (bytes of device memory NVML lists for this process over all devices, None) or (None, why not)"""
    try:
        nv = C.CDLL("libnvidia-ml.so.1")
    except OSError as e:
        return None, f"NVML is not loadable ({e})"
    if nv.nvmlInit_v2() != 0:
        return None, "nvmlInit_v2 failed"
    try:
        n = C.c_uint(0)
        if nv.nvmlDeviceGetCount_v2(C.byref(n)) != 0:
            return None, "nvmlDeviceGetCount_v2 failed"
        total, seen = 0, False
        for i in range(n.value):
            h = C.c_void_p()
            if nv.nvmlDeviceGetHandleByIndex_v2(i, C.byref(h)) != 0:
                continue
            infos = (_ProcInfo * 256)()
            k = C.c_uint(len(infos))
            if nv.nvmlDeviceGetComputeRunningProcesses_v3(h, C.byref(k), infos) != 0:
                continue
            for p in infos[:k.value]:
                if p.pid == os.getpid():
                    if p.usedGpuMemory == 2**64 - 1:
                        return None, "NVML lists this process without its memory (NVML_VALUE_NOT_AVAILABLE)"
                    total, seen = total + p.usedGpuMemory, True
        return (total, None) if seen else (None, f"NVML lists no compute process with this pid ({os.getpid()})")
    finally:
        nv.nvmlShutdown()


# ---- the work of one cycle, with its references ---------------------------------------------------------------
HP, HG, HT, THR = 1000, 4, 181, 150.0


def _host_window():
    w = dict(src="pageable", P=HP, G=HG, T=HT, seed=7, thr=THR, gates=True, table=True, outs={}, out_kind="host")
    d = S.window_data(w)
    assert d["table"] is not None and d["eligible"] is not None
    return d, S.expected(d["util"], d["power"], THR, d["eligible"], d["created_ts"], d["cutoff_ts"], d["table"])


BATCH = [(33, 4, 180, 101), (1000, 4, 181, 102), (9000, 1, 180, 103)]     # growing: the scratch grows in the batch


def _batch_windows():
    out = []
    for P, G, T, seed in BATCH:
        w = dict(src="dev", P=P, G=G, T=T, seed=seed, thr=THR, gates=True, table=False, outs={}, out_kind="dev")
        d = S.window_data(w)
        out.append((w, d, S.expected(d["util"], d["power"], THR, d["eligible"], d["created_ts"], d["cutoff_ts"])))
    return out


RP, RG, RT = 33, 4, 200                         # a ring of four index blocks


def _ring_ops():
    """(append columns and the ring model after append, advance, append)"""
    rows = RP * RG
    m = RS.Ring(RP, RG, RT, 3)
    u1, p1 = S.ring_columns(201, rows, RT + 5, True)
    u2, p2 = S.ring_columns(202, rows, 3, True)
    m.append(RT + 5, u1.view(np.uint32), p1.view(np.uint32))
    m.advance(7)
    m.append(3, u2.view(np.uint32), p2.view(np.uint32))
    return (u1, p1, u2, p2), S.expected(m.window(0), m.window(1), RS.THR)


TP, TG, TT = 1000, 4, 90                        # about 6 MB of text: three pageable chunks
T_END = 1_700_000_000


def _response():
    """a matrix response with a sample of every series at every second of the window but a few; -> (text, util
    [P, G, T] with NaN where a sample is absent, markers, spans, CSR samples)"""
    rng = np.random.default_rng(301)
    rows = TP * TG
    u = rng.choice(np.array([0, 0, 0, 2, np.nan], np.float32), size=(rows, TT))
    u[rng.random(rows) < 0.5] = 0.0
    u[:, -1] = np.where(np.isnan(u[:, -1]), 0.0, u[:, -1])          # no empty series
    ts = T_END - TT + 1 + np.arange(TT)
    parts = []
    for r in range(rows):
        body = ",".join('[%d,"%d"]' % (ts[c], u[r, c]) for c in range(TT) if not np.isnan(u[r, c]))
        parts.append('{"metric":{"pod":"p%d","gpu":"%d"},"values":[%s]}' % (r // TG, r % TG, body))
    text = ('{"status":"success","data":{"resultType":"matrix","result":[' + ",".join(parts) + "]}}").encode()
    opens = np.array([m.start() for m in re.finditer(re.escape(OPEN), text)], np.uint64)
    closes = np.array([m.start() for m in re.finditer(re.escape(CLOSE), text)], np.uint64)
    import gpu_pruner_b200 as g
    spans = np.zeros(rows, g.IdleEngine.SPAN_DTYPE)
    spans["begin"] = opens + 12
    spans["end"] = closes[np.searchsorted(closes, opens + 12)] + 2
    spans["row"] = np.arange(rows)
    present = ~np.isnan(u)
    offsets = np.concatenate([[0], np.cumsum(present.sum(1))]).astype(np.uint64)
    csr = (offsets, np.arange(rows, dtype=np.uint32), (np.broadcast_to(ts, u.shape)[present] * 1000).astype(np.int64),
           u[present].astype(np.float64))
    return text, u.reshape(TP, TG, TT), opens, closes, spans, csr


@pytest.fixture(scope="module")
def refs():
    return dict(host=_host_window(), batch=_batch_windows(), ring=_ring_ops(), text=_response())


def _counts(r):
    return (r.n_series, r.n_candidates, r.n_decisions)


def _want_counts(e):
    return (e["n_series"], e["n_candidates"], e["n_decisions"])


def _words(a):
    return np.asarray(a.cpu() if hasattr(a, "cpu") else a).view(np.uint32).ravel()


def _same_bits(got, want, what):
    assert np.array_equal(_words(got), np.asarray(want, np.uint32).ravel()), what


def _host_decision(eng, refs, what):
    d, want = refs["host"]
    r = eng.decide(d["util"], d["power"], d["eligible"], d["created_ts"], d["cutoff_ts"], power_threshold=THR,
                   want_series_max=True, want_veto=True, groups=d["table"], want_idle_slots=True)
    assert _counts(r) == _want_counts(want), what
    for name in ("decision_bits", "candidate_bits", "veto_bits", "idle_slots"):
        _same_bits(getattr(r, name), want[name], (what, name))
    assert kat.smax_equal(r.series_max.ravel(), want["series_max"].ravel()), what


def _async_batch(eng, refs, what):
    def dev(a):
        return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)
    calls, keep = [], []
    for w, d, _ in refs["batch"]:
        P, G, T = w["P"], w["G"], w["T"]
        W = (P + 31) // 32
        out = dict(decision_bits=torch.zeros(W, dtype=torch.int32, device=DEV),
                   candidate_bits=torch.zeros(W, dtype=torch.int32, device=DEV),
                   veto_bits=torch.zeros(W, dtype=torch.int32, device=DEV),
                   series_max=torch.zeros(P * G, dtype=torch.float32, device=DEV))
        ins = dict(util=dev(d["util"]), power=dev(d["power"]), eligible=dev(d["eligible"]),
                   created_ts=dev(d["created_ts"]))
        keep.append((ins, out))
        calls.append(dict(ins, **out, cutoff_ts=d["cutoff_ts"], P=P, G=G, T=T, power_threshold=w["thr"]))
    torch.cuda.synchronize()                    # the context's stream is not ordered with torch's
    ress = eng.decide_batch_async(eng.make_batch(calls))
    eng.sync()
    for (w, _, want), r, (_, out) in zip(refs["batch"], ress, keep):
        assert _counts(r) == _want_counts(want), (what, w["P"])
        for name in ("decision_bits", "candidate_bits", "veto_bits"):
            _same_bits(out[name], want[name], (what, w["P"], name))
        assert kat.smax_equal(out["series_max"].cpu().numpy(), want["series_max"].ravel()), (what, w["P"])


def _resident(eng, refs, what):
    (u1, p1, u2, p2), want = refs["ring"]
    eng.resident_init(RP, RG, 64, power_plane=True, block_index=True)
    eng.resident_init(RP, RG, RT, power_plane=True, block_index=True)     # the planes and the index reallocated
    eng.append(u1, p1)
    eng.resident_advance(7)
    eng.append(u2, p2)
    W = (RP + 31) // 32
    db, cb, vb = (np.zeros(W, np.uint32) for _ in range(3))
    r = eng.decide_ptr(None, RP, RG, RT, db, candidate_bits=cb, veto_bits=vb, power_threshold=RS.THR, in_kind=0,
                       out_kind=0, resident=True)
    assert _counts(r) == _want_counts(want), what
    for name, got in (("decision_bits", db), ("candidate_bits", cb), ("veto_bits", vb)):
        _same_bits(got, want[name], (what, name))


def _read_plane(eng):
    got = np.empty((TP, TG, TT), np.float32)
    eng.memcpy(got, eng.text_planes()[0], got.nbytes, 0, 1)
    return got


def _same_plane(got, u, what):
    assert np.array_equal(np.isnan(got), np.isnan(u)) and np.array_equal(np.nan_to_num(got), np.nan_to_num(u)), what


def _text(eng, refs, what):
    import gpu_pruner_b200 as g
    text, u, opens, closes, spans, _ = refs["text"]
    o, c = eng.text_scan(text, slot=0)                                   # pageable: staged, several threads
    assert np.array_equal(o, opens) and np.array_equal(c, closes), (what, "pageable scan")
    pinned = eng.host_array((len(text),), np.uint8)
    pinned[:] = np.frombuffer(text, np.uint8)
    o, c = eng.text_scan(pinned, slot=1, n_bytes=len(text))
    assert np.array_equal(o, opens) and np.array_equal(c, closes), (what, "pinned scan")
    out = eng.text_parse(spans.copy(), T_END, 1, TT, TP * TG, slot=1)
    assert int(out["n_in"].sum()) == int((~np.isnan(u)).sum()) and not np.any(out["flags"] & 2), what
    _same_plane(_read_plane(eng), u, (what, "parsed plane"))
    want = S.expected(u)
    db = np.zeros((TP + 31) // 32, np.uint32)
    r = eng.decide_ptr(eng.text_planes()[0], TP, TG, TT, db, in_kind=g.ffi.GPR_MEM_DEVICE, out_kind=g.ffi.GPR_MEM_HOST)
    assert r.n_decisions == want["n_decisions"], what
    _same_bits(db, want["decision_bits"], (what, "decision on the parsed plane"))


def _scatter(eng, refs, what):
    import gpu_pruner_b200 as g
    _, u, _, _, _, (offsets, rows, ts, vals) = refs["text"]
    n = len(ts)
    st = eng.samples_scatter(offsets, rows, ts, vals, T_END, 1, TT, TP * TG)
    assert st == {"n_in": n, "n_oow": 0, "n_tiny": 0}, (what, "host batch", st)
    _same_plane(_read_plane(eng), u, (what, "host batch"))
    dev = [torch.from_numpy(np.ascontiguousarray(a)).to(DEV) for a in (offsets.view(np.int64), rows.view(np.int32),
                                                                       ts, vals)]
    torch.cuda.synchronize()
    st = eng.samples_scatter(*dev, T_END, 1, TT, TP * TG, mem_kind=g.ffi.GPR_MEM_DEVICE, n_series=len(rows))
    assert st == {"n_in": n, "n_oow": 0, "n_tiny": 0}, (what, "device batch", st)
    _same_plane(_read_plane(eng), u, (what, "device batch"))


def _cycle(refs, what):
    eng = _engine(max_pods=HP, max_gpus=HG, max_samples=HT, power_plane=True)
    try:
        _host_decision(eng, refs, what)
        _async_batch(eng, refs, what)
        _resident(eng, refs, what)
        _text(eng, refs, what)
        _scatter(eng, refs, what)
        eng.timer_begin()
        eng.flush_l2()
        assert eng.timer_end() > 0, what
    finally:
        eng.close()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


def test_cycles_give_the_references_and_release_their_memory(refs):
    used = []
    for k in range(CYCLES):
        _cycle(refs, f"cycle {k}")
        used.append(_process_bytes())
    first, why = used[0]
    if first is None:
        warnings.warn(f"device memory per cycle not checked: {why}")
        print(f"\n[cycles] device memory per cycle not checked: {why}")
        return
    mb = [round(b / MB, 1) for b, _ in used]
    print(f"\n[cycles] device memory of this process after each cycle (MB, NVML): {mb}")
    assert abs(used[-1][0] - first) <= MEM_TOL, mb


# ---- a context destroyed while its scan is in flight ---------------------------------------------------------------
N_REC = 320_000                                   # 164 MB: 79 chunks of 2 MB, far more than the marker ring holds


def _big_text():
    """fixed-width records (tests/test_gpu_text_scan.py): row i holds 5, 10 + i % 90 and 1,000,000 + i"""
    rec, lab, mid, last, o_off, c_off = _big_template()
    n = len(PRE) + N_REC * REC + 3
    text = np.empty(n, np.uint8)
    text[:len(PRE)] = np.frombuffer(PRE, np.uint8)
    body = text[len(PRE):len(PRE) + N_REC * REC].reshape(N_REC, REC)
    body[:] = np.frombuffer(rec, np.uint8)
    idx = np.arange(N_REC, dtype=np.int64)
    _digits(body, lab, idx, 7)
    _digits(body, mid, 10 + idx % 90, 2)
    _digits(body, last, 1_000_000 + idx, 7)
    body[-1, -1] = ord(" ")
    text[-3:] = np.frombuffer(b"]}}", np.uint8)
    opens = (len(PRE) + idx * REC + o_off).astype(np.uint64)
    closes = (len(PRE) + idx * REC + c_off).astype(np.uint64)
    cells = np.stack([np.full(N_REC, 5.0), 10 + idx % 90, 1_000_000 + idx], 1).astype(np.float32)
    return text, opens, closes, cells


def test_destroy_during_a_scan_leaves_the_device_usable():
    text, opens, closes, cells = _big_text()
    eng = _engine({"GPR_TEXT_UPLOAD_THREADS": "8", "GPR_TEXT_CHUNK_MB": "2"})
    chunks = eng.text_scan_chunks(text)
    o, c, done = next(chunks)
    assert 0 < done <= 2 * MB and np.array_equal(o, opens[opens < done]) and np.array_equal(c, closes[closes < done])
    chunks.close()                                 # (the generator makes no call when closed)
    eng.close()                                    # gpr_destroy with the scan of the other 77 chunks unfinished
    eng = _engine()
    try:
        o, c = eng.text_scan(text)
        assert np.array_equal(o, opens) and np.array_equal(c, closes)
        spans = np.zeros(N_REC, eng.SPAN_DTYPE)
        spans["begin"], spans["end"], spans["row"] = opens + 12, closes + 2, np.arange(N_REC)
        out = eng.text_parse(spans, SCAN_T_END, SCAN_STEP, 3, N_REC, window_seconds=45)
        assert np.all(out["n_in"] == 3) and np.all(out["n_oow"] == 0) and not np.any(out["flags"] & 2)
        got = np.empty((N_REC, 3), np.float32)
        eng.memcpy(got, eng.text_planes()[0], got.nbytes, 0, 1)
        bad = np.flatnonzero((got != cells).any(1))
        assert len(bad) == 0, [(int(b), got[b].tolist(), cells[b].tolist()) for b in bad[:8]]
    finally:
        eng.close()
    x = torch.arange(1 << 20, device=DEV, dtype=torch.float64) * 2
    assert float(x.sum()) == float((1 << 20) * ((1 << 20) - 1))


# ---- gpr_create failing after its allocations ------------------------------------------------------------------
def test_failed_creates_release_and_a_good_one_follows(oracle_c):
    import gpu_pruner_b200 as g
    from gpu_pruner_b200 import ffi
    if not torch.cuda.is_available():
        pytest.fail("-m gpu tests need a CUDA device; the engine has no CPU fallback")
    lib = ffi.load()
    P, G, T, seed = 100, 4, 1800, 0x5EED0001
    with _environ({}):                              # no GPR_KERNEL to override the variant
        for _ in range(10):
            cfg = ffi.gpr_config(struct_size=C.sizeof(ffi.gpr_config), device=0, max_pods=P, max_gpus=G,
                                 max_samples=T, flags=ffi.GPR_F_POWER_PLANE, kernel_variant=7)
            h = C.c_void_p()
            assert lib.gpr_create(C.byref(cfg), C.byref(h)) == ffi.GPR_E_INVALID
            assert h.value is None and b"bad kernel_variant 7" in lib.gpr_last_error(None)
    u = oracle_c.synth_fill(seed, 0, 0, P, G, T)
    w = oracle_c.synth_fill(seed, 1, 0, P, G, T)
    e = oracle_c.synth_eligible(seed, 0, P)
    want = oracle_c.decide(u, w, e, power_threshold=THR)
    eng = _engine(max_pods=P, max_gpus=G, max_samples=T, power_plane=True)
    try:
        d = eng.decide(u, w, e, power_threshold=THR)
        assert np.array_equal(d.decision_bits, want["decision_bits"])
        assert (d.n_series, d.n_candidates, d.n_decisions) == (want["n_series"], want["n_candidates"],
                                                               want["n_decisions"])
    finally:
        eng.close()
