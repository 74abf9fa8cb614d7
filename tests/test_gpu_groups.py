"""`sum by` groups (gpr_window.groups) on the H100, through libgpr.so: the windows of tests/test_groups_emul.py with
both f32 kernels and the byte format, from device memory (dense, strided, 4 bytes off alignment) and host memory, with
the power plane and series_max on and off; the resident ring with and without its block index; an async batch that
mixes grouped and ungrouped windows under PDL; a C2-scale window with 15 % grouped pods; malformed device tables; and
the float64 PromQL scenarios of test_promql_semantics.py decided on device planes with the table, no host fix-up.
Everything is compared with the restatement in tests/groups_ref.py."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

import groups_ref as R
import hostlib as H
import test_groups_emul as GE
from test_gpu_geometry import DEV, _u32

pytestmark = pytest.mark.gpu
THR = GE.THR


CHUNK_PODS = 24   # pods per 1 MB staging chunk of a 3 x 1800 window with power (48 without)


def _chunked_window():
    """150 x 3 x 1800: 7 staging chunks with power and 4 without at GPR_CHUNK_MB=1, and a table that changes from
    chunk to chunk (no groups; all three slots one group; slots 1-2 one group), so a chunk that read another chunk's
    grouped rows or wrote its row maxima over another chunk's would decide differently"""
    rng = np.random.default_rng(77)
    P, G, T = 150, 3, 1800
    layouts = [[0, 1, 2], [0, 0, 0], [0, 1, 1]]
    table = np.array([layouts[(p // CHUNK_PODS) % 3] for p in range(P)], np.uint32)
    table |= np.where(rng.random((P, G)) < 0.5, R.UTIL, 0).astype(np.uint32)
    m = np.array(R.PALETTE, np.float32)[rng.integers(0, len(R.PALETTE), (P, G))]
    util = R.window_for(rng, m, T)
    power = np.full((P, G, T), 100.0, np.float32)
    power[rng.random(P) < 0.2, 0, T // 3] = THR
    return util, power, table


def _cases():
    out = []
    for i, (P, G, T, size) in enumerate(GE.SHAPES):
        out.append((f"gen{i}", *GE._generated(100 + i, P, G, T, max_size=size)))
    u, table, _ = GE._host_window()
    out.append(("ingested", u, None, table))
    out.append(("chunked", *_chunked_window()))
    return out


def _want(util, power, table, use_power):
    return R.decide(util, power if use_power else None, THR if use_power else 0.0, table)


def _check(got, want, tag):
    dbits, cbits, counts, islots = got
    assert np.array_equal(dbits, want["decision_bits"]), tag
    assert np.array_equal(cbits, want["candidate_bits"]), tag
    assert tuple(counts) == (want["n_series"], want["n_candidates"], want["n_candidates"]), (tag, counts)
    assert np.array_equal(islots.reshape(want["idle_slots"].shape), want["idle_slots"]), tag


def _smax_equal(a, b):
    return np.array_equal(np.asarray(a, np.float32).view(np.uint32), np.asarray(b, np.float32).view(np.uint32))


def _device(eng, util, power, table, use_power, smax, stride=0, offset=0, u8=False):
    import gpu_pruner_b200 as g
    P, G, T = util.shape
    ld = stride or T
    if u8:
        flat = np.zeros((P * G * ld + 16,), np.uint8)
        flat[offset:offset + P * G * ld].reshape(P * G, ld)[:, :T] = g.to_biased_u8(util).reshape(P * G, T)
    else:
        flat = np.full((P * G * ld + 4,), 77.0, np.float32)
        flat[offset:offset + P * G * ld].reshape(P * G, ld)[:, :T] = util.reshape(P * G, T)
    u_t = torch.from_numpy(flat).to(DEV)
    u_ptr = u_t.data_ptr() + offset * flat.itemsize
    w_t = None
    if use_power:
        pw = np.full((P * G * ld + 4,), 1e9, np.float32)
        pw[offset:offset + P * G * ld].reshape(P * G, ld)[:, :T] = power.reshape(P * G, T)
        w_t = torch.from_numpy(pw).to(DEV)
    W, MW = max((P + 31) // 32, 1), (G + 31) // 32
    db = torch.full((W,), 0x7BADBEEF, dtype=torch.int32, device=DEV)
    cb = torch.full((W,), 0x7BADBEEF, dtype=torch.int32, device=DEV)
    isl = torch.full((P * MW,), 0x5A5A5A5A, dtype=torch.int32, device=DEV)
    sm = torch.full((P * G,), -777.0, dtype=torch.float32, device=DEV) if smax else None
    g_t = None if table is None else torch.from_numpy(table.astype(np.int32)).to(DEV)
    torch.cuda.synchronize()
    r = eng.decide_ptr(u_ptr, P, G, T, db, power=None if w_t is None else w_t.data_ptr() + offset * 4,
                       power_threshold=THR if use_power else 0.0, candidate_bits=cb, series_max=sm, row_stride=stride,
                       groups=g_t, idle_slots=isl, util_format=1 if u8 else 0)
    W = (P + 31) // 32
    return (_u32(db)[:W], _u32(cb)[:W], (r.n_series, r.n_candidates, r.n_decisions), _u32(isl)), \
        (sm.cpu().numpy().reshape(P, G) if smax else None)


@pytest.mark.parametrize("kernel", ["ldg", "tma"])
def test_windows_from_every_source(kernel):
    """device windows (dense, strided, misaligned) and host windows, the host ones also staged in 1 MB chunks
    (GPR_CHUNK_MB=1), where the windows of 1800 samples span several chunks and the table follows them"""
    import gpu_pruner_b200 as g
    from test_gpu_geometry import _environ
    caps = dict(device=0, kernel=kernel, max_pods=256, max_gpus=256, max_samples=2048, power_plane=True)
    with _environ({"GPR_CHUNK_MB": "1"}):
        chunked = g.IdleEngine(**caps)
    with g.IdleEngine(**caps) as eng, chunked:
        assert 150 * 3 * 1800 * 8 > 6 << 20      # the chunked case: more than six 1 MB chunks with power
        for name, util, power, table in _cases():
            P, G, T = util.shape
            for use_power in (False, True) if power is not None else (False,):
                want = _want(util, power, table, use_power)
                for smax in (False, True):
                    smax_by_table = {}
                    for t in (table, None):
                        w = want if t is not None else _want(util, power, None, use_power)
                        for stride, offset in ((0, 0), (T + 4, 0), (0, 1)):
                            tag = (kernel, name, use_power, smax, t is not None, stride, offset)
                            got, sm = _device(eng, util, power, t, use_power, smax, stride, offset)
                            _check(got, w, tag)
                            if smax:
                                m = R.row_max(util)
                                assert np.array_equal(np.isnan(sm), np.isnan(m)) and np.array_equal(
                                    np.nan_to_num(sm), np.nan_to_num(m)), tag
                                smax_by_table.setdefault(t is not None, sm)
                        for e, leg in ((eng, "host"), (chunked, "host, 1 MB chunks")):
                            d = e.decide(util, power if use_power else None, power_threshold=THR if use_power else 0.0,
                                         want_series_max=smax, groups=t, want_idle_slots=True)
                            _check((d.decision_bits, d.candidate_bits, (d.n_series, d.n_candidates, d.n_decisions),
                                    d.idle_slots), w, (kernel, name, leg, use_power, smax, t is not None))
                            if smax:
                                m = R.row_max(util)
                                assert np.array_equal(np.isnan(d.series_max), np.isnan(m)) and np.array_equal(
                                    np.nan_to_num(d.series_max), np.nan_to_num(m)), (kernel, name, leg)
                    if smax:   # series_max does not depend on the table
                        assert _smax_equal(smax_by_table[True], smax_by_table[False]), (kernel, name)


def test_byte_windows():
    import gpu_pruner_b200 as g
    with g.IdleEngine(device=0, max_pods=128, max_gpus=256, max_samples=2048, power_plane=True) as eng:
        for i, (P, G, T, size) in enumerate(GE.SHAPES):
            util, power, table = GE._generated(200 + i, P, G, T, u8=True, max_size=size)
            for use_power in (False, True):
                want = _want(util, power, table, use_power)
                for smax in (False, True):
                    for offset in (0, 3):
                        got, _ = _device(eng, util, power, table, use_power, smax, 0, offset, u8=True)
                        _check(got, want, ("u8", i, use_power, smax, offset))
                d = eng.decide(g.to_biased_u8(util), power if use_power else None,
                               power_threshold=THR if use_power else 0.0, groups=table, want_idle_slots=True)
                _check((d.decision_bits, d.candidate_bits, (d.n_series, d.n_candidates, d.n_decisions), d.idle_slots),
                       want, ("u8 host", i, use_power))


def test_previous_struct_sizes_decide_as_before():
    """without a table, and with the struct sizes of a caller built before the table existed, every output is
    bit-identical to the new sizes without a table"""
    import gpu_pruner_b200 as g
    from gpu_pruner_b200 import ffi
    util, power, _ = GE._generated(7, 37, 4, 256)
    P, G, T = util.shape
    with g.IdleEngine(device=0, max_pods=64, max_gpus=4, max_samples=256, power_plane=True) as eng:
        outs = []
        for old in (False, True):
            w = eng._window(util, power, None, None, 0, P, G, T, 0, THR, ffi.GPR_MEM_HOST)
            r = ffi.gpr_result()
            r.struct_size = ffi.gpr_result.idle_slots.offset if old else C.sizeof(ffi.gpr_result)
            if old:
                w.struct_size = ffi.gpr_window.groups.offset
            db, cb, vb = (np.zeros(2, np.uint32) for _ in range(3))
            sm = np.zeros((P, G), np.float32)
            r.out_mem_kind = ffi.GPR_MEM_HOST
            r.decision_bits, r.candidate_bits, r.veto_bits, r.series_max = (x.ctypes.data for x in (db, cb, vb, sm))
            assert eng._lib.gpr_decide(eng.handle, C.byref(w), C.byref(r)) == 0
            outs.append((db, cb, vb, sm.view(np.uint32), (r.n_series, r.n_candidates, r.n_decisions)))
        for a, b in zip(*outs):
            assert np.array_equal(a, b) if isinstance(a, np.ndarray) else a == b
        w.struct_size = 12
        assert eng._lib.gpr_decide(eng.handle, C.byref(w), C.byref(r)) == ffi.GPR_E_INVALID


@pytest.mark.parametrize("block_index", [False, True])
def test_resident_ring(block_index):
    import gpu_pruner_b200 as g
    util, power, table = GE._generated(31, 37, 40, 192)
    P, G, T = util.shape
    with g.IdleEngine(device=0) as eng:
        eng.resident_init(P, G, T, power_plane=True, block_index=block_index)
        eng.append(util.reshape(P * G, T), power.reshape(P * G, T))
        for t in (table, None):
            want = _want(util, power, t, True)
            W, MW = (P + 31) // 32, (G + 31) // 32
            db, cb, isl = np.zeros(W, np.uint32), np.zeros(W, np.uint32), np.zeros(P * MW, np.uint32)
            r = eng.decide_ptr(None, P, G, T, db, candidate_bits=cb, power_threshold=THR, groups=t, idle_slots=isl,
                               in_kind=0, out_kind=0, resident=True)
            _check((db, cb, (r.n_series, r.n_candidates, r.n_decisions), isl), want, ("resident", block_index, t is None))


@pytest.mark.parametrize("pdl", ["1", "0"])
def test_async_batch_mixing_grouped_and_ungrouped(pdl, monkeypatch):
    import gpu_pruner_b200 as g
    monkeypatch.setenv("GPR_PDL", pdl)
    cases = [GE._generated(300 + i, P, G, T, max_size=s) for i, (P, G, T, s) in enumerate(GE.SHAPES[:3])]
    with g.IdleEngine(device=0, kernel="tma") as eng:
        calls, wants, keep = [], [], []
        for rep in range(3):
            for k, (util, power, table) in enumerate(cases):
                t = table if (rep + k) % 2 == 0 else None
                P, G, T = util.shape
                u_t = torch.from_numpy(util).to(DEV)
                w_t = torch.from_numpy(power).to(DEV)
                g_t = None if t is None else torch.from_numpy(t.astype(np.int32)).to(DEV)
                W, MW = max((P + 31) // 32, 1), (G + 31) // 32
                db = torch.zeros(W, dtype=torch.int32, device=DEV)
                cb = torch.zeros(W, dtype=torch.int32, device=DEV)
                isl = torch.zeros(P * MW, dtype=torch.int32, device=DEV)
                keep += [u_t, w_t, g_t]
                calls.append(dict(util=u_t, power=w_t, P=P, G=G, T=T, power_threshold=THR, decision_bits=db,
                                  candidate_bits=cb, groups=g_t, idle_slots=isl))
                wants.append(_want(util, power, t, True))
        torch.cuda.synchronize()
        batch = eng.make_batch(calls)
        ress = eng.decide_batch_async(batch)
        eng.sync()
        for i, (kw, want) in enumerate(zip(calls, wants)):
            r = ress[i]
            W = (kw["P"] + 31) // 32
            _check((_u32(kw["decision_bits"])[:W], _u32(kw["candidate_bits"])[:W],
                    (r.n_series, r.n_candidates, r.n_decisions), _u32(kw["idle_slots"])), want, ("batch", pdl, i))


def test_c2_scale_window_with_grouped_pods():
    """a C2-shaped synthetic window (10,000 pods x 4 x 1800), 15 % of the pods with groups of 2-3 series"""
    import gpu_pruner_b200 as g
    P, G, T = 10000, 4, 1800
    rng = np.random.default_rng(5)
    table = np.tile(np.arange(G, dtype=np.uint32), (P, 1))
    for p in np.flatnonzero(rng.random(P) < 0.15):
        size = int(rng.integers(2, 4))
        table[p, 1:size] = 0
        table[p] |= np.where(rng.random(G) < 0.5, R.UTIL, 0).astype(np.uint32)
    with g.IdleEngine(device=0) as eng:
        u = torch.full((P, G, T), float("nan"), dtype=torch.float32, device=DEV)
        eng.synth_fill(0x5EED0002, 0, u, 0, P, G, T)
        torch.cuda.synchronize()
        m = R.row_max(u.cpu().numpy())
        want = R.decide(None, table=table, m=m)
        for kernel_table in (table, None):
            W = (P + 31) // 32
            db = torch.zeros(W, dtype=torch.int32, device=DEV)
            cb = torch.zeros(W, dtype=torch.int32, device=DEV)
            isl = torch.zeros(P, dtype=torch.int32, device=DEV)
            g_t = None if kernel_table is None else torch.from_numpy(kernel_table.astype(np.int32)).to(DEV)
            r = eng.decide_ptr(u, P, G, T, db, candidate_bits=cb, groups=g_t, idle_slots=isl)
            w = want if kernel_table is not None else R.decide(None, m=m)
            _check((_u32(db), _u32(cb), (r.n_series, r.n_candidates, r.n_decisions), _u32(isl)), w,
                   ("c2", kernel_table is None))
        assert len(want["values"]) > 1000            # groups of two or more that the kernels summed


def test_malformed_device_table_fails_and_the_next_decision_is_right():
    import gpu_pruner_b200 as g
    from gpu_pruner_b200 import ffi
    util, power, table = GE._generated(41, 37, 4, 256)
    P, G, T = util.shape
    bad = table.copy()
    bad[17, 2] = 3                                         # leader above its slot
    with g.IdleEngine(device=0) as eng:
        with pytest.raises(g.GprError) as ei:
            _device(eng, util, power, bad, True, False)
        assert ei.value.code == ffi.GPR_E_INVALID and "pod 17" in str(ei.value)
        got, _ = _device(eng, util, power, table, True, False)
        _check(got, _want(util, power, table, True), "after the failure")
        with pytest.raises(g.GprError) as ei:                # a host table is checked before anything is enqueued
            eng.decide(util, groups=bad)
        assert ei.value.code == ffi.GPR_E_INVALID and "pod 17" in str(ei.value)
        got, _ = _device(eng, util, power, None, True, True)
        _check(got, _want(util, power, None, True), "after the host failure")


@pytest.mark.parametrize("seed", range(40))
def test_promql_scenarios_on_device_planes_without_host_fixup(seed):
    """float64 PromQL (tests/promql_mini.py) picks the pods; the engine, given the group table, must return the same
    pods and num_series by itself"""
    import gpu_pruner_b200 as g
    import test_promql_semantics as PS
    sc = PS.scenario(seed)
    if not sc["util"]["data"]["result"] and not sc["prof"]["data"]["result"]:
        return
    u, w, meta = H.ingest(sc["util"], sc["prof"], sc["power"], duration_min=sc["dur"], step=sc["step"],
                          t_end=sc["t_eval"], power_threshold=sc["thr"])
    P, G, T = u.shape
    table = np.zeros((P, G), np.uint32)
    H.lib().gph_group_table(C.c_uint(P), table.ctypes.data_as(C.c_void_p))
    names = [(p["name"], p["namespace"]) for p in meta["pods"]]
    thr = sc["thr"]
    use_power = w is not None and bool(thr) and not np.isnan(thr)
    with g.IdleEngine(device=0) as eng:
        u_t = torch.from_numpy(u).to(DEV)
        w_t = torch.from_numpy(w).to(DEV) if use_power else None
        g_t = torch.from_numpy(table.astype(np.int32)).to(DEV)
        W = max((P + 31) // 32, 1)
        db = torch.zeros(W, dtype=torch.int32, device=DEV)
        cb = torch.zeros(W, dtype=torch.int32, device=DEV)
        isl = torch.zeros(P * ((G + 31) // 32), dtype=torch.int32, device=DEV)
        r = eng.decide_ptr(u_t, P, G, T, db, power=w_t, power_threshold=thr if use_power else 0.0, candidate_bits=cb,
                           groups=g_t, idle_slots=isl)
        cand = np.unpackbits(_u32(cb).view(np.uint8), bitorder="little")[:P]
        assert {names[i] for i in np.flatnonzero(cand)} == set(sc["pods"]), seed
        assert r.n_series == sc["n_series"], seed


@pytest.mark.parametrize("kernel", ["tma", "ldg"])
def test_pipelined_decisions_into_one_idle_slots_buffer(kernel, monkeypatch):
    """ungrouped decisions under PDL, a large window and a small one in turn, all writing one device idle_slots
    buffer: each decision's words land after its predecessor's (the fold waits for the previous fold before it writes
    the caller's buffer), so the buffer ends as the small window's words over the large one's"""
    import gpu_pruner_b200 as g
    monkeypatch.setenv("GPR_PDL", "1")
    rng = np.random.default_rng(9)
    shapes = [(4000, 4, 1800), (37, 4, 256)]
    wins = []
    for P, G, T in shapes:
        u = np.zeros((P, G, T), np.float32)
        u[rng.random((P, G)) < 0.6, T // 2] = 3.0
        wins.append((u, R.decide(u)["idle_slots"].ravel()))
    with g.IdleEngine(device=0, kernel=kernel) as eng:
        isl = torch.full((4000,), 0x5A5A5A5A, dtype=torch.int32, device=DEV)
        ts = [torch.from_numpy(u).to(DEV) for u, _ in wins]
        dbs = []
        torch.cuda.synchronize()
        for rep in range(8):
            for k, (P, G, T) in enumerate(shapes):
                db = torch.zeros((P + 31) // 32, dtype=torch.int32, device=DEV)
                dbs.append(db)
                eng.decide_ptr(ts[k], P, G, T, db, idle_slots=isl, blocking=False)
        eng.sync()
        want = wins[0][1].copy()
        want[:wins[1][1].size] = wins[1][1]
        assert np.array_equal(_u32(isl), want)


def test_binary_decides_sum_by_groups_and_reports_the_first_idle_element(tmp_path):
    """the `test_exact_sum_by_of_duplicate_series` cluster and a pod whose first group is busy and second idle, through
    the gpu-pruner binary (verdict, num_series, scale-downs) and through the same tick in a driver that prints the
    PodMetricData rows (tests/cpp/tick_driver.cpp)"""
    import json
    import subprocess
    import test_gpu_promql as GP
    NOW = GP.NOW

    def lab(pod, gpu, ctr="main", model="NVIDIA A100", **kw):
        d = {"Hostname": "node1", "modelName": model, "UUID": "GPU-x", "gpu": str(gpu), "exported_pod": pod,
             "exported_namespace": "ml", "exported_container": ctr}
        d.update(kw)
        return d

    def ser(labels, v):
        return {"metric": labels, "values": [[NOW - 30, str(v)], [NOW, str(v)]]}
    util = [ser(lab("mixed", 0, UUID="a"), 5), ser(lab("mixed", 0, UUID="b"), -5),
            ser(lab("halfbusy", 0, UUID="a"), 0), ser(lab("halfbusy", 0, UUID="b"), 7),
            ser(lab("allidle", 0, UUID="a"), 0), ser(lab("allidle", 0, UUID="b"), 0),
            ser(lab("single", 0), 0),
            ser(lab("second", 0, ctr="c0", UUID="a"), 0), ser(lab("second", 0, ctr="c0", UUID="b"), 7),
            ser(lab("second", 1, ctr="c1", model="NVIDIA H100", UUID="a"), 5),
            ser(lab("second", 1, ctr="c1", model="NVIDIA H100", UUID="b"), -5)]
    resp = lambda ss: {"status": "success", "data": {"resultType": "matrix", "result": ss}}
    prom, kube = tmp_path / "prom", tmp_path / "kube"
    prom.mkdir()
    (prom / "util.json").write_bytes(GP._dump(resp(util)))
    (prom / "prof.json").write_bytes(GP._dump(resp([])))
    (prom / "query.json").write_text(json.dumps({"end": NOW, "step": 1}))
    pods = ["mixed", "halfbusy", "allidle", "single", "second"]
    GP._kube(kube, [(p, "ml") for p in pods])
    idle = {"mixed", "allidle", "single", "second"}
    for kernel in ("ldg", "tma"):
        msgs = GP._run_bin(prom, kube, None, kernel)
        assert "Query returned 4 series across 4 unique pods" in msgs, [m for m in msgs if m.startswith("Query")]
        sent = {m.split("dep-")[1].split()[0] for m in msgs if m.startswith("Dry-run: Would have sent")}
        assert sent == idle, (kernel, sent)
    exe = tmp_path / "tick_driver"
    host = os.path.join(GE.ROOT, "gpu-pruner_b200", "host")
    lib = os.path.join(GE.ROOT, "gpu-pruner_b200")
    srcs = [os.path.join(host, f) for f in ("cli.cpp", "promql.cpp", "json.cpp", "kube.cpp", "ingest.cpp",
                                             "ingest_device.cpp", "controller.cpp", "gpr_engine.cpp")]
    subprocess.run(["g++", "-std=c++17", "-O1", "-I", host, os.path.join(GE.ROOT, "tests", "cpp", "tick_driver.cpp")]
                   + srcs + ["-L", lib, "-lgpr", "-Wl,-rpath," + lib, "-lpthread", "-o", str(exe)],
                   check=True, capture_output=True, text=True)
    r = subprocess.run([str(exe), "--prometheus-url", f"file://{prom}", "--kube-fixture", str(kube), "-t", "2", "-g",
                        "300", "--now", str(NOW), "-l", "json"], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr[-3000:]
    out = json.loads(r.stdout)
    assert out["ok"] and out["num_pods"] == 4, out
    rows = {u["name"]: u for u in out["unique_pods"]}
    assert set(rows) == idle
    for name, u in rows.items():
        ctr, model = ("c1", "NVIDIA H100") if name == "second" else ("main", "NVIDIA A100")
        assert (u["namespace"], u["container"], u["gpu_model"], u["node_type"], u["value"]) == \
            ("ml", ctr, model, "unknown", 0.0), u
