"""The decision kernels on an H100 in the launch geometries away from the defaults, and at scale.

* Knob sets: a fresh IdleEngine per set of tuning knobs (GPR_TMA_WARPS / _CHUNK / _DEPTH, GPR_LDG_CTAS,
  GPR_FOLD_THREADS, GPR_PDL, GPR_CHUNK_MB), read by gpr_create from the environment.  Together the sets take every
  value of every knob.  Each runs test_gpu_parity's random windows, strided and misaligned rows, a host window staged
  in many chunks and a batch of unlike decisions, all against the C oracle; the geometry header
  (gpu-pruner_b200/csrc/gpr_launch.h, through tests/cpp/launch_plan.cpp) says which kernel ran, and the test asserts
  it was the one the set is about, not a fallback.  The AUTO sets decide their windows twice: with series_max (every
  row read whole, k_reduce_tma) and with idle_slots alone (rows stop early, the probe kernel), every row checked.
* Scale: device windows from gpr_synth_fill against the streaming oracle, every row checked (series_max or
  idle_slots, veto bits), where the fold loops (more than 4 * (fold_threads / 32) * sm_count bitmap words).
* Limit (slow): a window of 2^31 - 32 series with a power plane, 2^32 - 64 rows in one reduce launch.

Large allocations check the free device memory first and skip when it is not there: the GPU may be shared.
"""
import contextlib
import dataclasses
import os
import time

import numpy as np
import pytest

import geometry
import kat
from test_gpu_parity import SHAPES, _random_window, check_idle_slots

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")
DEV = "cuda:0"
GB = 1 << 30

K = geometry.Knobs
# (knobs, kernel, GPR_PDL): together every value of every knob; sm_count is the device's
KNOB_SETS = [
    (K(tma_warps=16, tma_chunk=8192, tma_depth=3, ldg_ctas=2, fold_threads=256), "tma", 1),
    (K(tma_warps=4, tma_chunk=512, tma_depth=1, ldg_ctas=2, fold_threads=64), "tma", 0),
    (K(tma_warps=8, tma_chunk=2048, tma_depth=2, ldg_ctas=1, fold_threads=128), "tma", 1),
    (K(tma_warps=32, tma_chunk=2048, tma_depth=3, ldg_ctas=1, fold_threads=256), "tma", 0),
    (K(tma_warps=32, tma_chunk=512, tma_depth=1, ldg_ctas=2, fold_threads=64), "auto", 1),
    (K(tma_warps=8, tma_chunk=16384, tma_depth=2, ldg_ctas=2, fold_threads=128), "tma", 1),
    (K(tma_warps=4, tma_chunk=65536, tma_depth=3, ldg_ctas=2, fold_threads=256), "tma", 1),
    (K(tma_warps=16, tma_chunk=4096, tma_depth=1, ldg_ctas=1, fold_threads=64), "auto", 0),
    (K(ldg_ctas=1, fold_threads=64), "ldg", 1),
    (K(ldg_ctas=2, fold_threads=128), "ldg", 0),
    (K(ldg_ctas=4, fold_threads=256), "ldg", 1),
]
SET_IDS = [f"{v}-w{k.tma_warps}-c{k.tma_chunk}-d{k.tma_depth}-l{k.ldg_ctas}-f{k.fold_threads}-pdl{p}"
           for k, v, p in KNOB_SETS]


@pytest.fixture(scope="module")
def plan_exe(tmp_path_factory):
    return geometry.build(tmp_path_factory.mktemp("launch_plan"))


@pytest.fixture(scope="module")
def sm_count():
    import gpu_pruner_b200 as g
    if not torch.cuda.is_available():
        pytest.fail("-m gpu tests need a CUDA device; the engine has no CPU fallback")
    with g.IdleEngine(device=0) as e:
        return e.device_info()["sm_count"]


@contextlib.contextmanager
def _environ(env):
    keys = set(env) | {"GPR_KERNEL"}
    saved = {k: os.environ.get(k) for k in keys}
    os.environ.pop("GPR_KERNEL", None)          # would override the kernel the engine asks for
    os.environ.update(env)
    try:
        yield
    finally:
        for k, v in saved.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def _engine(knobs, kernel, pdl=1, chunk_mb=None, **caps):
    import gpu_pruner_b200 as g
    env = dict(knobs.env(), GPR_PDL=str(pdl))
    if chunk_mb is not None:
        env["GPR_CHUNK_MB"] = str(chunk_mb)
    with _environ(env):
        return g.IdleEngine(device=0, kernel=kernel, **caps)


def _need(nbytes, what):
    free, _ = torch.cuda.mem_get_info()
    if free < nbytes + 2 * GB:
        pytest.skip(f"{what} needs {nbytes / GB:.1f} GB of device memory, {free / GB:.1f} GB free")


def _u32(t):
    return t.cpu().numpy().view(np.uint32)


def _check(bits, cbits, counts, exp, smax=None, vbits=None, islots=None):
    assert np.array_equal(bits, exp["decision_bits"]), "decision bitmap differs from oracle"
    assert np.array_equal(cbits, exp["candidate_bits"]), "candidate bitmap differs from oracle"
    assert tuple(counts) == (exp["n_series"], exp["n_candidates"], exp["n_decisions"])
    if smax is not None:
        assert kat.smax_equal(smax, exp["series_max"]), "series_max differs from oracle"
    if vbits is not None:
        assert np.array_equal(vbits, exp["veto_bits"]), "veto bitmap differs from oracle"
    if islots is not None:
        check_idle_slots(islots, exp["series_max"])


def _assert_intended(plan_exe, knobs, kernel, T, rows, P, tma_ok=True, util_u8=False, may_stop=False):
    """the geometry header's verdict for this call: the set's own kernel, with the set's own shape.  may_stop: the
    call passes no series_max (and no group table), so AUTO runs the probe kernel, whose layout ignores the tma knobs"""
    p = geometry.plan(plan_exe, knobs, kernel, T, rows, tma_ok, util_u8, P, may_stop)
    if util_u8:
        assert p.kernel == "u8", p
    elif kernel == "ldg" or not tma_ok:
        assert p.kernel == "ldg" and p.fallback == (None if kernel == "ldg" else "alignment"), p
        assert p.grid == max(1, min(knobs.sm_count * knobs.ldg_ctas, (rows + 15) // 16)), p
    elif kernel == "auto" and may_stop:
        assert p.kernel == "probe" and p.fallback is None and p.block == 1024, p
        assert p.grid == max(1, min(knobs.sm_count, (rows + 31) // 32)), p
        base = geometry.plan(plan_exe, K(sm_count=knobs.sm_count), kernel, T, rows, tma_ok, util_u8, P, may_stop)
        assert (p.depth, p.stage_bytes, p.chunk_elems, p.n_chunks, p.head_elems, p.smem) == \
            (base.depth, base.stage_bytes, base.chunk_elems, base.n_chunks, base.head_elems, base.smem), (p, base)
    else:
        assert p.kernel == "tma" and p.fallback is None and p.block == 32 * knobs.tma_warps, p
        assert p.depth <= knobs.tma_depth and 4 * p.chunk_elems <= max(knobs.tma_chunk, 16), p
    assert p.fold_grid <= knobs.sm_count
    return p


def _device_decide(eng, u_t, P, G, T, w_t=None, kw=None, thr=0.0, stride=0, util_format=0, want_smax=True,
                   want_veto=False, want_slots=False):
    """-> bits, candidate bits, counts, series_max, veto bits, idle_slots ([P, ceil(G / 32)]); the last three None
    unless asked for"""
    kw = kw or {}
    e_t = torch.from_numpy(np.ascontiguousarray(kw["eligible"], np.uint8)).to(DEV) if "eligible" in kw else None
    c_t = torch.from_numpy(np.ascontiguousarray(kw["created_ts"], np.int64)).to(DEV) if "created_ts" in kw else None
    W = max((P + 31) // 32, 1)
    db = torch.full((W,), 0x7BADBEEF, dtype=torch.int32, device=DEV)
    cb = torch.full((W,), 0x7BADBEEF, dtype=torch.int32, device=DEV)
    vb = torch.full((W,), 0x5A5A5A5A, dtype=torch.int32, device=DEV) if want_veto else None
    sm = torch.full((max(P * G, 1),), -777.0, dtype=torch.float32, device=DEV) if want_smax else None
    MW = (G + 31) // 32
    isl = torch.full((max(P, 1) * MW,), 0x7BADBEEF, dtype=torch.int32, device=DEV) if want_slots else None
    torch.cuda.synchronize()
    r = eng.decide_ptr(u_t, P, G, T, db, power=w_t, eligible=e_t, created_ts=c_t, cutoff_ts=kw.get("cutoff_ts", 0),
                       power_threshold=thr, candidate_bits=cb, series_max=sm, veto_bits=vb, row_stride=stride,
                       util_format=util_format, idle_slots=isl)
    W = (P + 31) // 32
    return (_u32(db)[:W], _u32(cb)[:W], (r.n_series, r.n_candidates, r.n_decisions),
            sm.cpu().numpy()[:P * G].reshape(P, G) if want_smax else None, _u32(vb)[:W] if want_veto else None,
            _u32(isl)[:P * MW].reshape(P, MW) if want_slots else None)


# ---------------------------------------------------------------------------------------------
# knob sets
# ---------------------------------------------------------------------------------------------
def test_knob_sets_cover_every_value():
    ks = [k for k, _, _ in KNOB_SETS]
    assert {k.tma_warps for k, v, _ in KNOB_SETS if v != "ldg"} == {4, 8, 16, 32}
    assert {512, 2048, 8192, 16384, 65536} <= {k.tma_chunk for k, v, _ in KNOB_SETS if v != "ldg"}
    assert {k.tma_depth for k, v, _ in KNOB_SETS if v != "ldg"} == {1, 2, 3}
    assert {k.ldg_ctas for k in ks} >= {1, 2, 4} and {k.fold_threads for k in ks} == {64, 128, 256}
    assert {p for _, _, p in KNOB_SETS} == {0, 1} and {v for _, v, _ in KNOB_SETS} == {"tma", "ldg", "auto"}


def _modes(kernel):
    """read modes a knob set decides in: whole (series_max) always; early (idle_slots, no series_max) for AUTO, whose
    kernel it changes"""
    return (False, True) if kernel == "auto" else (False,)


@pytest.mark.parametrize("ks", KNOB_SETS, ids=SET_IDS)
def test_knob_set_random_and_strided_windows(ks, sm_count, plan_exe, oracle_c):
    knobs, kernel, pdl = ks
    knobs = dataclasses.replace(knobs, sm_count=sm_count)
    eng = _engine(knobs, kernel, pdl)
    try:
        for early in _modes(kernel):
            for P, G, T in SHAPES:
                for opts in ((False, False), (True, True)):
                    rng = np.random.default_rng(P * 31 + G * 7 + T)
                    u, kw = _random_window(rng, P, G, T, *opts)
                    exp = oracle_c.decide(u, **kw)
                    _assert_intended(plan_exe, knobs, kernel, T, P * G * (2 if opts[0] else 1), P, tma_ok=T % 4 == 0,
                                     may_stop=early)
                    u_t = torch.from_numpy(u).to(DEV)
                    w_t = torch.from_numpy(kw["power"]).to(DEV) if opts[0] else None
                    bits, cbits, counts, smax, _, isl = _device_decide(eng, u_t, P, G, T, w_t, kw,
                                                                       kw.get("power_threshold", 0.0),
                                                                       want_smax=not early, want_slots=early)
                    _check(bits, cbits, counts, exp, smax, islots=isl)
            for T, stride, offset in [(100, 104, 0), (100, 101, 0), (97, 97, 1), (64, 64, 3), (1800, 1800, 2),
                                      (1800, 1816, 0), (33, 40, 1)]:
                P, G = 130, 4
                rng = np.random.default_rng(T * 7 + stride + offset)
                u, _ = _random_window(rng, P, G, T, False, False)
                buf = np.full(offset + P * G * stride + 8, 99.0, np.float32)    # poisoned padding and slack
                buf[offset: offset + P * G * stride].reshape(P * G, stride)[:, :T] = u.reshape(P * G, T)
                t = torch.from_numpy(buf).to(DEV)
                _assert_intended(plan_exe, knobs, kernel, T, P * G, P,
                                 tma_ok=T % 4 == 0 and stride % 4 == 0 and offset == 0, may_stop=early)
                bits, cbits, counts, smax, _, isl = _device_decide(eng, t[offset:].data_ptr(), P, G, T, stride=stride,
                                                                   want_smax=not early, want_slots=early)
                _check(bits, cbits, counts, oracle_c.decide(u), smax, islots=isl)
    finally:
        eng.close()


@pytest.mark.parametrize("ks", KNOB_SETS, ids=SET_IDS)
def test_knob_set_host_window_in_many_chunks(ks, sm_count, plan_exe, oracle_c):
    """GPR_CHUNK_MB=1: the host window goes up in 1 MB pod chunks, one reduce launch per chunk into one fold"""
    knobs, kernel, pdl = ks
    knobs = dataclasses.replace(knobs, sm_count=sm_count)
    P, G, T = 3001, 4, 180
    eng = _engine(knobs, kernel, pdl, chunk_mb=1, max_pods=P, max_gpus=G, max_samples=T, power_plane=True)
    try:
        rng = np.random.default_rng(3001)
        u, kw = _random_window(rng, P, G, T, True, True)
        chunk_pods = (1 << 20) // (G * T * 8)
        assert (P + chunk_pods - 1) // chunk_pods >= 15
        exp = oracle_c.decide(u, **kw)
        from oracle import oracle_np
        exp["veto_bits"] = oracle_np.decide(u, kw["power"], kw["eligible"], kw["created_ts"], kw["cutoff_ts"],
                                            kw["power_threshold"])["veto_bits"]
        for early in _modes(kernel):
            _assert_intended(plan_exe, knobs, kernel, T, chunk_pods * G * 2, P, may_stop=early)
            d = eng.decide(u, kw["power"], kw["eligible"], kw["created_ts"], kw["cutoff_ts"], kw["power_threshold"],
                           want_series_max=not early, want_veto=True, want_idle_slots=early)
            _check(d.decision_bits, d.candidate_bits, (d.n_series, d.n_candidates, d.n_decisions), exp, d.series_max,
                   d.veto_bits, d.idle_slots)
    finally:
        eng.close()


@pytest.mark.parametrize("ks", KNOB_SETS, ids=SET_IDS)
def test_knob_set_batch_of_unlike_decisions(ks, sm_count, plan_exe, oracle_c):
    """one gpr_decide_batch_async of decisions that differ in every dimension: tiny and large P alternating, G from
    1 to 40, power on and off, f32 and biased-byte util, series_max on some; enqueued three times"""
    from gpu_pruner_b200 import ffi, to_biased_u8
    knobs, kernel, pdl = ks
    knobs = dataclasses.replace(knobs, sm_count=sm_count)
    eng = _engine(knobs, kernel, pdl)
    try:
        rng = np.random.default_rng(4242)
        calls, keep = [], []
        for i in range(12):
            P = int(rng.integers(1, 40)) if i % 2 == 0 else int(rng.integers(9000, 21000))
            G = [1, 40, 3, 33, 8, 2, 17, 1, 32, 5, 40, 4][i]
            T = int(rng.choice([1, 7, 64, 100, 181, 360])) if P > 1000 else int(rng.choice([4, 33, 600, 1800]))
            if P > 1000 and G > 8:
                P = 2000 + i
            power, u8, smax = i % 3 != 1, i % 4 == 3, i % 5 < 2
            u, kw = _random_window(rng, P, G, T, power, i % 2 == 1)
            if u8:
                u[np.isin(u, np.float32(-3)) | (np.signbit(u) & (u == 0))] = 0.0     # integers 0..254 or NaN
                ut = torch.from_numpy(to_biased_u8(u)).to(DEV)
            else:
                ut = torch.from_numpy(u).to(DEV)
            W = (P + 31) // 32
            c = dict(util=ut, P=P, G=G, T=T, util_format=ffi.GPR_FMT_U8B if u8 else ffi.GPR_FMT_F32,
                     decision_bits=torch.full((W,), -1, dtype=torch.int32, device=DEV),
                     candidate_bits=torch.full((W,), -1, dtype=torch.int32, device=DEV))
            if power:
                c["power"], c["power_threshold"] = torch.from_numpy(kw["power"]).to(DEV), kw["power_threshold"]
            if "eligible" in kw:
                c["eligible"] = torch.from_numpy(kw["eligible"]).to(DEV)
                c["created_ts"] = torch.from_numpy(kw["created_ts"]).to(DEV)
                c["cutoff_ts"] = kw["cutoff_ts"]
            if smax:
                c["series_max"] = torch.full((P * G,), -777.0, dtype=torch.float32, device=DEV)
            rows = P * G * (2 if power else 1)
            _assert_intended(plan_exe, knobs, kernel, T, rows, P, tma_ok=T % 4 == 0, util_u8=u8, may_stop=not smax)
            calls.append(c)
            keep.append((u, kw))
        batch = eng.make_batch(calls)
        torch.cuda.synchronize()
        for rep in range(3):
            ress = eng.decide_batch_async(batch)
            eng.sync()
            for c, (u, kw), r in zip(calls, keep, ress):
                exp = oracle_c.decide(u, **kw)
                sm = c["series_max"].cpu().numpy().reshape(c["P"], c["G"]) if "series_max" in c else None
                _check(_u32(c["decision_bits"]), _u32(c["candidate_bits"]),
                       (r.n_series, r.n_candidates, r.n_decisions), exp, sm)
    finally:
        eng.close()


# ---------------------------------------------------------------------------------------------
# scale: synthetic device windows where the fold loops
# ---------------------------------------------------------------------------------------------
_ORACLE = {}


def _oracle_synth(oracle_c, seed, P, G, T, power, smax=True):
    key = (seed, P, G, T, power, smax)
    if key not in _ORACLE:
        _ORACLE.clear()
        _ORACLE[key] = oracle_c.decide_synth(seed, 0, P, G, T, use_power=power, power_threshold=150.0 if power else 0.0,
                                             use_elig=True, want_series_max=smax, want_veto=power)
    return _ORACLE[key]


def _synth(eng, seed, P, G, T, power):
    u = torch.empty((P, G, T), dtype=torch.float32, device=DEV)
    eng.synth_fill(seed, 0, u, 0, P, G, T)
    w = None
    if power:
        w = torch.empty((P, G, T), dtype=torch.float32, device=DEV)
        eng.synth_fill(seed, 1, w, 0, P, G, T)
    e = torch.empty(P, dtype=torch.uint8, device=DEV)
    eng.synth_eligible(seed, e, 0, P)
    return u, w, e


@pytest.mark.parametrize("P,fold_threads", [(140_000, 256), (250_000, 256), (40_000, 64)])
def test_scale_fold_loops(P, fold_threads, sm_count, plan_exe, oracle_c):
    """fold rounds > 1 at the default tilings (and 64-thread fold CTAs), power and eligibility: tma and ldg reading
    every row whole, every row checked through series_max; the probe kernel (auto, rows stop early) with every row
    checked through idle_slots, which the fold (k_fold<false, true>) writes; the veto bits always"""
    G, T, seed = 4, 1800, 0x5EED0004 + P
    _need(2 * P * G * T * 4, f"{P} x {G} x {T} with power")
    knobs = K(sm_count=sm_count, fold_threads=fold_threads)
    exp = _oracle_synth(oracle_c, seed, P, G, T, True)
    for kernel, early in (("tma", False), ("ldg", False), ("auto", True)):
        eng = _engine(knobs, kernel)
        try:
            p = _assert_intended(plan_exe, knobs, kernel, T, 2 * P * G, P, may_stop=early)
            assert p.fold_rounds >= 2, p
            u, w, e = _synth(eng, seed, P, G, T, True)
            out = _device_decide(eng, u, P, G, T, w, {"eligible": e.cpu().numpy()}, 150.0, want_veto=True,
                                 want_smax=not early, want_slots=early)
            _check(*out[:3], exp, out[3], out[4], out[5])
            assert 0 < out[2][2] < P
            del u, w, e
        finally:
            eng.close()


def _u8_plane(eng, seed, P, G, T, pods_per_fill=20_000):
    """the synthetic util plane in GPR_FMT_U8B, generated in slices (the f32 plane would need 4x the memory)"""
    b = torch.empty((P, G, T), dtype=torch.uint8, device=DEV)
    tmp = torch.empty((min(P, pods_per_fill), G, T), dtype=torch.float32, device=DEV)
    for p0 in range(0, P, pods_per_fill):
        n = min(pods_per_fill, P - p0)
        eng.synth_fill(seed, 0, tmp[:n], p0, n, G, T)   # (on the engine's stream, which it synchronises)
        b[p0:p0 + n] = torch.where(torch.isnan(tmp[:n]), torch.zeros_like(tmp[:n]), tmp[:n] + 1).to(torch.uint8)
        torch.cuda.synchronize()                           # torch's stream: done with tmp before the next fill
    del tmp
    return b


@pytest.mark.slow
@pytest.mark.parametrize("fmt", ["f32", "u8"])
def test_scale_config_5_shard(fmt, sm_count, plan_exe, oracle_c):
    """BASELINE config 5 per GPU: 312,500 x 4 x 7,200 = 9.0e9 cells, more than 2^32; the fold takes 3 rounds.  As f32
    also with rows that stop early (AUTO: the probe kernel), every row checked through idle_slots"""
    P, G, T, seed = 312_500, 4, 7200, 0x5EED0005
    cells = P * G * T
    _need(cells * (4 if fmt == "f32" else 1) + 3 * GB, f"config 5 shard as {fmt}")
    knobs = K(sm_count=sm_count)
    exp = _oracle_synth(oracle_c, seed, P, G, T, False)
    legs = (("tma", False), ("ldg", False), ("auto", True)) if fmt == "f32" else (("auto", False),)
    eng = _engine(knobs, "auto")
    try:
        if fmt == "f32":
            u = torch.empty((P, G, T), dtype=torch.float32, device=DEV)
            eng.synth_fill(seed, 0, u, 0, P, G, T)
        else:
            u = _u8_plane(eng, seed, P, G, T)
        e = torch.empty(P, dtype=torch.uint8, device=DEV)
        eng.synth_eligible(seed, e, 0, P)
        torch.cuda.synchronize()
        for kernel, early in legs:
            k_eng = eng if kernel == "auto" else _engine(knobs, kernel)
            try:
                p = _assert_intended(plan_exe, knobs, kernel, T, P * G, P, util_u8=fmt == "u8", may_stop=early)
                assert p.fold_rounds >= 3, p
                out = _device_decide(k_eng, u, P, G, T, None, {"eligible": e.cpu().numpy()},
                                     util_format=1 if fmt == "u8" else 0, want_smax=not early, want_slots=early)
                _check(*out[:3], exp, out[3], None, out[5])
            finally:
                if k_eng is not eng:
                    k_eng.close()
        del u, e
    finally:
        eng.close()


# ---------------------------------------------------------------------------------------------
# the series limit: 2^31 - 32 series with a power plane = 2^32 - 64 rows in one reduce launch
# ---------------------------------------------------------------------------------------------
def _check_idle_slots_synth(oracle_c, islots, seed, P, G, T, pods_per_slice=1 << 21):
    """idle_slots of a synthetic window against the oracle's row maxima, one slice of pods at a time (the maxima of
    every series at the series limit would take 8 GB of host memory)"""
    for p0 in range(0, P, pods_per_slice):
        n = min(pods_per_slice, P - p0)
        smax = oracle_c.decide_synth(seed, p0, n, G, T, want_series_max=True)["series_max"]
        check_idle_slots(islots[p0:p0 + n], smax)


@pytest.mark.slow
@pytest.mark.parametrize("kernel,T", [("ldg", 1), ("tma", 4), ("auto", 4)])
def test_series_limit_with_power(kernel, T, sm_count, plan_exe, oracle_c):
    """ldg and tma ask for no series_max and stop rows early; auto does the same with the probe kernel, on sm_count
    CTAs, every row checked through idle_slots"""
    P, G, seed = 67_108_863, 32, 0x5EED0006
    S = P * G
    assert S == 2**31 - 32
    early_slots = kernel == "auto"
    _need(2 * S * T * 4 + (P * 4 if early_slots else 0), f"the series limit at T = {T}")
    knobs = K(sm_count=sm_count)
    p = _assert_intended(plan_exe, knobs, kernel, T, 2 * S, P, may_stop=True)
    assert p.grid == (2 * sm_count if kernel == "ldg" else sm_count), p
    exp = _oracle_synth(oracle_c, seed, P, G, T, True, smax=False)
    eng = _engine(knobs, kernel)
    try:
        u, w, e = _synth(eng, seed, P, G, T, True)
        out = _device_decide(eng, u, P, G, T, w, {"eligible": e.cpu().numpy()}, 150.0, want_smax=False,
                             want_veto=True, want_slots=early_slots)
        _check(*out[:3], exp, None, out[4])
        if early_slots:
            _check_idle_slots_synth(oracle_c, out[5], seed, P, G, T)
        del u, w, e
    finally:
        eng.close()


@pytest.fixture(autouse=True)
def _release_device_memory():
    """hand the large planes back to the device after each test: the next test's free-memory check is then honest,
    and the GPU may be shared"""
    yield
    import gc
    gc.collect()
    torch.cuda.empty_cache()


@pytest.fixture(autouse=True)
def _report(request):
    """GPR_GEOMETRY_REPORT=<file>: append each test's wall time and peak device memory in use (whole device, from
    cudaMemGetInfo sampled every 50 ms) as one JSON line"""
    path = os.environ.get("GPR_GEOMETRY_REPORT")
    if not path:
        yield
        return
    import json
    import threading
    free0, total = torch.cuda.mem_get_info()
    peak = [total - free0]
    stop = threading.Event()

    def sample():
        while not stop.wait(0.05):
            f, _ = torch.cuda.mem_get_info()
            peak[0] = max(peak[0], total - f)

    th = threading.Thread(target=sample, daemon=True)
    t0 = time.time()
    th.start()
    try:
        yield
    finally:
        stop.set()
        th.join()
        with open(path, "a") as f:
            f.write(json.dumps({"test": request.node.nodeid, "seconds": round(time.time() - t0, 2),
                                "used_gb_at_start": round((total - free0) / GB, 2),
                                "peak_used_gb": round(peak[0] / GB, 2)}) + "\n")
