"""GPU parity: the CUDA path, called through the C ABI (libgpr.so), against the CPU oracles.

Bit-exact on the decision / candidate bitmaps and the three counts; series_max numerically
exact (tolerance 0; -0.0 == +0.0, NaN matches NaN — the fmax tree does not preserve which
signed zero came first, Prometheus' sequential fold does; the verdict is unaffected).

Most windows are decided in two read modes.  "whole" asks for series_max, so every kernel reads
every row to its end.  "early" asks for idle_slots and no series_max, the call the gpu-pruner
binary makes: rows stop at their first settling sample, and AUTO runs the probe kernel
(k_reduce_probe) when the rows can be bulk-copied, else the early-exit LDG kernel.  idle_slots
is the per-row output that keeps early exit on, so every row's verdict is checked word for word,
not only the per-pod bitmaps where another row of the same pod could hide a wrong one.
"""
import ctypes as C
import os

import numpy as np
import pytest

import geometry
import kat

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")
KATS = kat.all_kats()
VARIANTS = ["ldg", "tma", "auto"]
MODES = ["whole", "early"]
# (kernel variant, read mode); a whole-row call is named by its variant alone
VARIANT_MODES = [(v, m) for v in VARIANTS for m in MODES]
VM_IDS = [v if m == "whole" else f"{v}-{m}" for v, m in VARIANT_MODES]


@pytest.fixture(scope="module")
def engines():
    import gpu_pruner_b200 as g
    if not torch.cuda.is_available():
        pytest.fail("-m gpu tests need a CUDA device; the engine has no CPU fallback")
    e = {v: g.IdleEngine(device=0, max_pods=12000, max_gpus=8, max_samples=2048, power_plane=True,
                         kernel=v) for v in VARIANTS}
    yield e
    for x in e.values():
        x.close()


@pytest.fixture(scope="module")
def plan_exe(tmp_path_factory):
    return geometry.build(tmp_path_factory.mktemp("launch_plan"))


def expected_idle_slots(series_max):
    """gpr_result.idle_slots without a group table (include/gpr.h): bit g of pod p's ceil(G / 32) words is set iff
    row g's window max is == 0 (-0.0 counts, NaN — no sample — does not); the bits above G are 0"""
    smax = np.asarray(series_max, np.float32)
    P, G = smax.shape
    MW = (G + 31) // 32
    idle = np.zeros((P, MW * 32), bool)
    idle[:, :G] = smax == 0
    return np.packbits(idle.reshape(P, MW, 32), axis=-1, bitorder="little").view("<u4").reshape(P, MW)


def check_idle_slots(islots, series_max):
    want = expected_idle_slots(series_max)
    got = np.asarray(islots).view(np.uint32).reshape(want.shape)
    bad = np.argwhere(got != want)
    assert bad.size == 0, (f"idle_slots differ from the oracle at pod {bad[0][0]} word {bad[0][1]}: "
                           f"{int(got[tuple(bad[0])]):#010x} != {int(want[tuple(bad[0])]):#010x}")


def _check(res_bits, res_cbits, counts, exp, smax=None, islots=None):
    assert np.array_equal(res_bits, exp["decision_bits"]), "decision bitmap differs from oracle"
    assert np.array_equal(res_cbits, exp["candidate_bits"]), "candidate bitmap differs from oracle"
    assert counts == (exp["n_series"], exp["n_candidates"], exp["n_decisions"])
    if smax is not None:
        assert kat.smax_equal(smax, exp["series_max"])
    if islots is not None:
        check_idle_slots(islots, exp["series_max"])


def _outputs(mode):
    """the outputs a call asks for in the given read mode"""
    assert mode in MODES
    return {"want_smax": mode == "whole", "want_slots": mode == "early"}


def assert_ran(plan_exe, sm_count, variant, mode, T, rows, tma_ok=True, P=1):
    """the geometry header's verdict for this call (gpu-pruner_b200/csrc/gpr_launch.h, which gpr_api.cu launches):
    rows that cannot be bulk-copied take LDG; an early AUTO call the probe kernel, a whole one k_reduce_tma"""
    p = geometry.plan(plan_exe, geometry.Knobs(sm_count=sm_count), variant, T, rows, tma_ok, False, P,
                      mode == "early")
    if variant == "ldg" or not tma_ok:
        want = "ldg"
    else:
        want = "probe" if variant == "auto" and mode == "early" else "tma"
    assert p.kernel == want, (variant, mode, p)
    return p


@pytest.fixture(scope="module")
def sm_count(engines):
    return engines["ldg"].device_info()["sm_count"]


def _device_decide(eng, u, power=None, eligible=None, created=None, cutoff=0, thr=0.0, stride=0,
                   want_smax=True, u_t=None, w_t=None, want_slots=False):
    """window already on the device (torch tensors) -> numpy results (idle_slots last, [P, ceil(G / 32)])"""
    dev = "cuda:0"
    P, G, T = u.shape if u_t is None else (u_t.shape[0], u_t.shape[1], u_t.shape[2])
    if u_t is None:
        u_t = torch.from_numpy(np.ascontiguousarray(u)).to(dev)
    if power is not None and w_t is None:
        w_t = torch.from_numpy(np.ascontiguousarray(power)).to(dev)
    e_t = torch.from_numpy(np.ascontiguousarray(eligible, dtype=np.uint8)).to(dev) if eligible is not None else None
    c_t = torch.from_numpy(np.ascontiguousarray(created, dtype=np.int64)).to(dev) if created is not None else None
    W = max((P + 31) // 32, 1)
    db = torch.full((W,), 0x7BADBEEF, dtype=torch.int32, device=dev)
    cb = torch.full((W,), 0x7BADBEEF, dtype=torch.int32, device=dev)
    sm = torch.full((max(P * G, 1),), -777.0, dtype=torch.float32, device=dev) if want_smax else None
    MW = (G + 31) // 32
    isl = torch.full((max(P, 1) * MW,), 0x7BADBEEF, dtype=torch.int32, device=dev) if want_slots else None
    torch.cuda.synchronize()
    r = eng.decide_ptr(u_t, P, G, T, db, power=w_t, eligible=e_t, created_ts=c_t, cutoff_ts=cutoff,
                       power_threshold=thr, candidate_bits=cb, series_max=sm, row_stride=stride, idle_slots=isl)
    W = (P + 31) // 32
    bits = db.cpu().numpy().view(np.uint32)[:W]
    cbits = cb.cpu().numpy().view(np.uint32)[:W]
    smax = sm.cpu().numpy()[: P * G].reshape(P, G) if want_smax else None
    islots = isl.cpu().numpy().view(np.uint32)[: P * MW].reshape(P, MW) if want_slots else None
    return bits, cbits, (r.n_series, r.n_candidates, r.n_decisions), smax, r, islots


# ---------------------------------------------------------------------------------------------
# known-answer vectors, both kernels, host and device windows
# ---------------------------------------------------------------------------------------------
def _kat_smax(k, oracle_c):
    """the row maxima the KAT writes out, else the oracle's"""
    if k.series_max is not None:
        return k.series_max
    return oracle_c.decide(k.util, k.power, k.eligible, k.created_ts, k.cutoff_ts, k.power_threshold)["series_max"]


def _kat_rows(k):
    P, G, _ = k.util.shape
    return P * G * (2 if k.power is not None and k.power_threshold else 1)


@pytest.mark.parametrize("variant,mode", VARIANT_MODES, ids=VM_IDS)
@pytest.mark.parametrize("k", KATS, ids=[k.name for k in KATS])
def test_kat_host_window(k, variant, mode, engines, oracle_c, plan_exe, sm_count):
    assert_ran(plan_exe, sm_count, variant, mode, k.util.shape[2], _kat_rows(k), k.util.shape[2] % 4 == 0)
    d = engines[variant].decide(k.util, k.power, k.eligible, k.created_ts, k.cutoff_ts,
                                k.power_threshold, want_series_max=mode == "whole",
                                want_idle_slots=mode == "early")
    assert np.array_equal(d.candidate_bits, kat.expected_bits(k.candidate)), k.why
    assert np.array_equal(d.decision_bits, kat.expected_bits(k.decision)), k.why
    assert (d.n_candidates, d.n_decisions) == (sum(k.candidate), sum(k.decision))
    if mode == "early":
        check_idle_slots(d.idle_slots, _kat_smax(k, oracle_c))
    elif k.series_max is not None:
        assert kat.smax_equal(d.series_max, k.series_max)
    if k.n_series is not None:
        assert d.n_series == k.n_series


@pytest.mark.parametrize("variant,mode", VARIANT_MODES, ids=VM_IDS)
@pytest.mark.parametrize("k", KATS, ids=[k.name for k in KATS])
def test_kat_device_window(k, variant, mode, engines, oracle_c, plan_exe, sm_count):
    assert_ran(plan_exe, sm_count, variant, mode, k.util.shape[2], _kat_rows(k), k.util.shape[2] % 4 == 0)
    bits, cbits, counts, smax, _, islots = _device_decide(engines[variant], k.util, k.power, k.eligible,
                                                          k.created_ts, k.cutoff_ts, k.power_threshold,
                                                          **_outputs(mode))
    assert np.array_equal(cbits, kat.expected_bits(k.candidate)), k.why
    assert np.array_equal(bits, kat.expected_bits(k.decision)), k.why
    if mode == "early":
        check_idle_slots(islots, _kat_smax(k, oracle_c))
    elif k.series_max is not None:
        assert kat.smax_equal(smax, k.series_max)


# ---------------------------------------------------------------------------------------------
# random windows vs both oracles: ragged shapes, strides, misaligned bases
# ---------------------------------------------------------------------------------------------
def _random_window(rng, P, G, T, with_power, with_gates):
    u = rng.choice(np.array([0, 1, 50, 100, np.nan, -0.0, -3], np.float32), size=(P, G, T),
                   p=[.85, .02, .01, .01, .09, .01, .01])
    idle_rows = rng.random((P, G)) < 0.5
    u[idle_rows] = np.where(rng.random((int(idle_rows.sum()), T)) < 0.05, np.nan, 0).astype(np.float32)
    burst = np.flatnonzero(rng.random(P) < 0.2)
    u[burst, rng.integers(0, G, burst.size), rng.integers(0, T, burst.size)] = 1.0
    kw = {}
    if with_power:
        w = rng.choice(np.array([40, 60, 149.99, np.nan], np.float32), size=(P, G, T), p=[.5, .44, .02, .04])
        hot = np.flatnonzero(rng.random(P) < 0.4)
        w[hot, rng.integers(0, G, hot.size), rng.integers(0, T, hot.size)] = rng.choice(
            np.array([150, 150.01, 400], np.float32), size=hot.size)
        kw["power"], kw["power_threshold"] = w, 150.0
    if with_gates:
        kw["eligible"] = (rng.random(P) < 0.9).astype(np.uint8)
        kw["created_ts"] = rng.integers(1000, 2000, P).astype(np.int64)
        kw["cutoff_ts"] = 1500
    return u, kw


SHAPES = [(1, 1, 1), (3, 2, 5), (31, 4, 33), (64, 1, 450), (257, 8, 100), (1000, 4, 180),
          (999, 3, 1801), (4097, 4, 64), (50, 4, 7200), (20, 2, 9000), (6, 1, 20000)]


@pytest.mark.parametrize("variant,mode", VARIANT_MODES, ids=VM_IDS)
@pytest.mark.parametrize("P,G,T", SHAPES)
@pytest.mark.parametrize("opts", [(False, False), (True, True)])
def test_random_device_window(P, G, T, opts, variant, mode, engines, oracle_c, oracle_np, plan_exe, sm_count):
    rng = np.random.default_rng(P * 31 + G * 7 + T)
    u, kw = _random_window(rng, P, G, T, *opts)
    exp = oracle_c.decide(u, **kw)
    exp2 = oracle_np.decide(u, **kw)
    assert np.array_equal(exp["decision_bits"], exp2["decision_bits"])
    assert_ran(plan_exe, sm_count, variant, mode, T, P * G * (2 if opts[0] else 1), T % 4 == 0)
    bits, cbits, counts, smax, _, islots = _device_decide(
        engines[variant], u, kw.get("power"), kw.get("eligible"), kw.get("created_ts"),
        kw.get("cutoff_ts", 0), kw.get("power_threshold", 0.0), **_outputs(mode))
    _check(bits, cbits, counts, exp, smax, islots)


@pytest.mark.parametrize("variant,mode", VARIANT_MODES, ids=VM_IDS)
@pytest.mark.parametrize("P,G,T", [(3, 2, 5), (257, 8, 100), (1000, 4, 180), (999, 3, 1801), (300, 4, 2048)])
def test_random_host_window(P, G, T, variant, mode, engines, oracle_c, plan_exe, sm_count):
    rng = np.random.default_rng(P + T)
    u, kw = _random_window(rng, P, G, T, True, True)
    exp = oracle_c.decide(u, **kw)
    assert_ran(plan_exe, sm_count, variant, mode, T, 2 * P * G, T % 4 == 0)
    d = engines[variant].decide(u, kw["power"], kw["eligible"], kw["created_ts"], kw["cutoff_ts"],
                                kw["power_threshold"], want_series_max=mode == "whole",
                                want_idle_slots=mode == "early")
    _check(d.decision_bits, d.candidate_bits, (d.n_series, d.n_candidates, d.n_decisions), exp,
           d.series_max, d.idle_slots)
    assert d.kernel_ms > 0


@pytest.mark.parametrize("variant,mode", VARIANT_MODES, ids=VM_IDS)
@pytest.mark.parametrize("T,stride,offset", [(100, 104, 0), (100, 101, 0), (97, 97, 1), (64, 64, 3),
                                             (1800, 1800, 2), (1800, 1816, 0), (33, 40, 1)])
def test_strided_and_misaligned_rows(T, stride, offset, variant, mode, engines, oracle_c, plan_exe, sm_count):
    """row_stride > T and bases that are only 4-byte aligned: the head/tail peel must read every
    sample exactly once and never a neighbour's"""
    P, G = 130, 4
    rng = np.random.default_rng(T * 7 + stride + offset)
    u, _ = _random_window(rng, P, G, T, False, False)
    # poison the padding and the slack before the first row: reading it would flip verdicts
    buf = np.full(offset + P * G * stride + 8, 99.0, np.float32)
    view = buf[offset: offset + P * G * stride].reshape(P * G, stride)
    view[:, :T] = u.reshape(P * G, T)
    t = torch.from_numpy(buf).to("cuda:0")
    u_t = t[offset:]
    exp = oracle_c.decide(u)
    assert_ran(plan_exe, sm_count, variant, mode, T, P * G, T % 4 == 0 and stride % 4 == 0 and offset == 0)
    W = (P + 31) // 32
    db = torch.zeros(W, dtype=torch.int32, device="cuda:0")
    cb = torch.zeros(W, dtype=torch.int32, device="cuda:0")
    sm = torch.zeros(P * G, dtype=torch.float32, device="cuda:0") if mode == "whole" else None
    isl = torch.full((P,), 0x7BADBEEF, dtype=torch.int32, device="cuda:0") if mode == "early" else None
    torch.cuda.synchronize()   # the engine's stream is not ordered with torch's: buffers must be ready
    r = engines[variant].decide_ptr(u_t.data_ptr(), P, G, T, db, candidate_bits=cb, series_max=sm,
                                    row_stride=stride, idle_slots=isl)
    _check(db.cpu().numpy().view(np.uint32), cb.cpu().numpy().view(np.uint32),
           (r.n_series, r.n_candidates, r.n_decisions), exp,
           None if sm is None else sm.cpu().numpy().reshape(P, G), None if isl is None else isl.cpu().numpy())


# ---------------------------------------------------------------------------------------------
# synthetic universe: CUDA generator == C oracle generator; full-size parity by regeneration
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("plane", [0, 1])
@pytest.mark.parametrize("P,G,T,off", [(64, 4, 180, 0), (33, 8, 77, 12345), (10, 4, 1800, 7)])
def test_cuda_generator_matches_oracle(plane, P, G, T, off, engines, oracle_c):
    eng = engines["ldg"]
    t = torch.empty((P, G, T), dtype=torch.float32, device="cuda:0")
    eng.synth_fill(0x5EED0002, plane, t, off, P, G, T)
    a = t.cpu().numpy()
    b = oracle_c.synth_fill(0x5EED0002, plane, off, P, G, T)
    assert np.all((a == b) | (np.isnan(a) & np.isnan(b)))
    e = torch.empty(P, dtype=torch.uint8, device="cuda:0")
    eng.synth_eligible(0x5EED0002, e, off, P)
    assert np.array_equal(e.cpu().numpy(), oracle_c.synth_eligible(0x5EED0002, off, P))


def _synth_device(eng, seed, P, G, T, power, off=0):
    u = torch.empty((P, G, T), dtype=torch.float32, device="cuda:0")
    eng.synth_fill(seed, 0, u, off, P, G, T)
    w = None
    if power:
        w = torch.empty((P, G, T), dtype=torch.float32, device="cuda:0")
        eng.synth_fill(seed, 1, w, off, P, G, T)
    e = torch.empty(P, dtype=torch.uint8, device="cuda:0")
    eng.synth_eligible(seed, e, off, P)
    return u, w, e


@pytest.mark.parametrize("variant,mode", VARIANT_MODES, ids=VM_IDS)
@pytest.mark.parametrize("power", [False, True])
def test_config_c2_full_parity(variant, power, mode, engines, oracle_c, plan_exe, sm_count):
    """BASELINE config #2: 10k pods x 4 GPUs x 1800 samples, every bit (and every row's max or idle slot) against
    the oracle"""
    seed, P, G, T = 0x5EED0002, 10000, 4, 1800
    eng = engines[variant]
    u, w, e = _synth_device(eng, seed, P, G, T, power)
    exp = oracle_c.decide_synth(seed, 0, P, G, T, use_power=power, power_threshold=150.0, use_elig=True,
                                want_series_max=True)
    assert_ran(plan_exe, sm_count, variant, mode, T, P * G * (2 if power else 1))
    bits, cbits, counts, smax, r, islots = _device_decide(eng, None, u_t=u, w_t=w, eligible=e.cpu().numpy(),
                                                          thr=150.0 if power else 0.0, **_outputs(mode))
    _check(bits, cbits, counts, exp, smax, islots)
    assert 0 < counts[2] < P
    # and through the host-window path (pinned staging, chunked H2D overlapped with the reduce)
    d = eng.decide(u.cpu().numpy(), None if w is None else w.cpu().numpy(), e.cpu().numpy(),
                   power_threshold=150.0 if power else 0.0, want_series_max=mode == "whole",
                   want_idle_slots=mode == "early")
    _check(d.decision_bits, d.candidate_bits, (d.n_series, d.n_candidates, d.n_decisions), exp, d.series_max,
           d.idle_slots)


def test_config_c1_golden_fixture(engines):
    """BASELINE config #1 (100 x 4 x 1800): the checked-in idle set"""
    gold = np.load(os.path.join(os.path.dirname(__file__), "golden", "c1_idle_set.npz"))
    seed, P, G, T = int(gold["seed"]), int(gold["P"]), int(gold["G"]), int(gold["T"])
    for v in VARIANTS:
        u, w, e = _synth_device(engines[v], seed, P, G, T, True)
        bits, cbits, counts, _, _, _ = _device_decide(engines[v], None, u_t=u, eligible=e.cpu().numpy(),
                                                      want_smax=False)
        assert np.array_equal(bits, gold["decision_bits"]) and np.array_equal(cbits, gold["candidate_bits"])
        bits, cbits, counts, _, _, _ = _device_decide(engines[v], None, u_t=u, w_t=w, thr=150.0,
                                                      eligible=e.cpu().numpy(), want_smax=False)
        assert np.array_equal(bits, gold["decision_bits_power"])
        assert list(np.flatnonzero(np.unpackbits(bits.view(np.uint8), bitorder="little"))) == \
            list(gold["idle_pods_power"])


@pytest.mark.slow
@pytest.mark.parametrize("variant,mode", VARIANT_MODES, ids=VM_IDS)
def test_config_c3_full_parity_and_properties(variant, mode, engines, oracle_c, plan_exe, sm_count):
    """BASELINE config #3: 100k x 8 x 3600 (11.5 GB).  Full parity by streaming regeneration on the
    host, every row through series_max or idle_slots, plus size-independent properties: idempotence,
    shard consistency, time-reversal invariance (max is order independent), monotonicity, counts ==
    popcounts."""
    seed, P, G, T = 0x5EED0003, 100000, 8, 3600
    eng = engines[variant]
    u, _, e = _synth_device(eng, seed, P, G, T, False)
    en = e.cpu().numpy()
    assert_ran(plan_exe, sm_count, variant, mode, T, P * G)
    bits, cbits, counts, smax, _, islots = _device_decide(eng, None, u_t=u, eligible=en, **_outputs(mode))
    exp = oracle_c.decide_synth(seed, 0, P, G, T, use_elig=True, want_series_max=True)
    _check(bits, cbits, counts, exp, smax, islots)
    pop = lambda b: int(np.unpackbits(b.view(np.uint8)).sum())
    assert counts[1] == pop(cbits) and counts[2] == pop(bits)
    assert np.all(bits & ~cbits == 0)                       # decision implies candidate
    # idempotence
    bits2, cbits2, counts2, _, _, _ = _device_decide(eng, None, u_t=u, eligible=en, want_smax=False)
    assert np.array_equal(bits, bits2) and counts == counts2
    # shard consistency: a 32-aligned slice of the window gives the same words
    p0, p1 = 32 * 1000, 32 * 2200
    sb, scb, _, _, _, _ = _device_decide(eng, None, u_t=u[p0:p1], eligible=en[p0:p1], want_smax=False)
    assert np.array_equal(sb, bits[p0 // 32: p1 // 32]) and np.array_equal(scb, cbits[p0 // 32: p1 // 32])
    # time reversal
    sub = u[:20000].flip(2).contiguous()
    rb, rcb, _, _, _, _ = _device_decide(eng, None, u_t=sub, eligible=en[:20000], want_smax=False)
    assert np.array_equal(rb, bits[:625]) and np.array_equal(rcb, cbits[:625])
    # monotonicity: poke one positive sample into 1000 random series -> bits can only clear
    g = torch.Generator(device="cpu").manual_seed(1)
    pods = torch.randint(0, P, (1000,), generator=g)
    u[pods, torch.randint(0, G, (1000,), generator=g), torch.randint(0, T, (1000,), generator=g)] = 9.0
    mb, mcb, _, _, _, _ = _device_decide(eng, None, u_t=u, eligible=en, want_smax=False)
    assert np.all(mcb & ~cbits == 0) and not np.array_equal(mcb, cbits)


# ---------------------------------------------------------------------------------------------
# async entry point, resident window, error paths
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("variant", VARIANTS)
def test_async_back_to_back(variant, engines, oracle_c):
    eng = engines[variant]
    seed, P, G, T = 77, 2048, 4, 600
    outs = []
    for i in range(5):
        u, _, e = _synth_device(eng, seed + i, P, G, T, False)
        db = torch.zeros(P // 32, dtype=torch.int32, device="cuda:0")
        torch.cuda.synchronize()
        r = eng.decide_ptr(u, P, G, T, db, eligible=e, blocking=False)
        outs.append((u, e, db, r, seed + i))
    eng.sync()
    for u, e, db, r, s in outs:
        exp = oracle_c.decide_synth(s, 0, P, G, T, use_elig=True)
        assert np.array_equal(db.cpu().numpy().view(np.uint32), exp["decision_bits"])
        assert (r.n_series, r.n_candidates, r.n_decisions) == (exp["n_series"], exp["n_candidates"], exp["n_decisions"])


@pytest.mark.parametrize("variant", VARIANTS)
def test_batch_entry_point(variant, engines, oracle_c):
    """gpr_decide_batch_async == n calls of gpr_decide_async, including overlapped launches"""
    eng = engines[variant]
    P, G, T = 4096, 4, 360
    calls, keep = [], []
    for i in range(12):
        u, w, e = _synth_device(eng, 900 + i, P, G, T, i % 3 == 0)
        db = torch.zeros(P // 32, dtype=torch.int32, device="cuda:0")
        cb = torch.zeros(P // 32, dtype=torch.int32, device="cuda:0")
        calls.append(dict(util=u, power=w, power_threshold=150.0 if w is not None else 0.0, eligible=e,
                          P=P, G=G, T=T, decision_bits=db, candidate_bits=cb))
        keep.append((900 + i, w is not None, db, cb))
    batch = eng.make_batch(calls)
    torch.cuda.synchronize()
    for rep in range(3):
        ress = eng.decide_batch_async(batch)
        eng.sync()
    for (seed, power, db, cb), r in zip(keep, ress):
        exp = oracle_c.decide_synth(seed, 0, P, G, T, use_power=power, power_threshold=150.0, use_elig=True)
        _check(db.cpu().numpy().view(np.uint32), cb.cpu().numpy().view(np.uint32),
               (r.n_series, r.n_candidates, r.n_decisions), exp)


def resident_ld(T, block_index):
    """the row length gpr_decide_resident decides on: the ring's T, or the block index's idx_ld = ceil(T / 64)
    rounded up to a multiple of 4"""
    return (-(-T // 64) + 3) // 4 * 4 if block_index else T


@pytest.mark.parametrize("block_index", [False, True], ids=["rescan", "block-index"])
@pytest.mark.parametrize("variant,mode", VARIANT_MODES, ids=VM_IDS)
def test_resident_window_ring(variant, block_index, mode, engines, oracle_c, plan_exe, sm_count):
    """daemon mode: append columns tick by tick into the HBM ring, rescan, compare with the
    oracle on the window a fresh range query would have returned"""
    eng = engines[variant]
    seed, P, G, T = 0x5EED0005, 777, 4, 240
    total = 900
    full = oracle_c.synth_fill(seed, 0, 0, P, G, total)       # one long history
    fullw = oracle_c.synth_fill(seed, 1, 0, P, G, total)
    eng.resident_init(P, G, T, power_plane=True, block_index=block_index)
    assert_ran(plan_exe, sm_count, variant, mode, resident_ld(T, block_index), 2 * P * G)
    W = (P + 31) // 32
    db = np.zeros(W, np.uint32)
    cb = np.zeros(W, np.uint32)
    sm = np.zeros((P, G), np.float32) if mode == "whole" else None
    isl = np.full(P, 0xDEADBEEF, np.uint32) if mode == "early" else None
    t = 0
    for n_new in (60, 1, 179, 240, 37, 300, 83):              # 300 > T: only the newest T survive
        eng.append(full[:, :, t:t + n_new], fullw[:, :, t:t + n_new])
        t += n_new
        r = eng.decide_ptr(None, 0, 0, 0, db, candidate_bits=cb, series_max=sm, power_threshold=150.0,
                           in_kind=0, out_kind=0, resident=True, idle_slots=isl)
        lo = max(0, t - T)
        win = np.full((P, G, T), np.nan, np.float32)
        win[:, :, : t - lo] = full[:, :, lo:t]
        winw = np.full((P, G, T), np.nan, np.float32)
        winw[:, :, : t - lo] = fullw[:, :, lo:t]
        exp = oracle_c.decide(win, winw, power_threshold=150.0)
        _check(db, cb, (r.n_series, r.n_candidates, r.n_decisions), exp, sm, isl)


@pytest.mark.parametrize("T", [64, 100, 240, 7200])
def test_block_index_rebuild_after_direct_writes(T, engines, oracle_c):
    """GPR_F_BLOCK_INDEX: the index follows gpr_append by itself and gpr_resident_reindex after the
    caller filled the planes directly; deciding on it equals deciding on the full rows"""
    eng = engines["tma"]
    seed, P, G = 0x5EED0005, 300, 4
    eng.resident_init(P, G, T, block_index=True)
    u_ptr, _, ld = eng.resident_planes()
    assert ld == T
    eng.synth_fill(seed, 0, u_ptr, 0, P, G, T)            # written behind the library's back ...
    eng.resident_reindex()                                # ... so the index must be rebuilt
    W = (P + 31) // 32
    db, cb, sm = np.zeros(W, np.uint32), np.zeros(W, np.uint32), np.zeros((P, G), np.float32)
    r = eng.decide_ptr(None, 0, 0, 0, db, candidate_bits=cb, series_max=sm, in_kind=0, out_kind=0, resident=True)
    full = oracle_c.synth_fill(seed, 0, 0, P, G, T)
    _check(db, cb, (r.n_series, r.n_candidates, r.n_decisions), oracle_c.decide(full), sm)
    # overwrite the burst of a few series through gpr_append: their block maxima must drop again
    n_new = min(T, 70)
    cols = np.zeros((P, G, n_new), np.float32)
    eng.append(cols)
    full = np.concatenate([full[:, :, n_new:], cols], axis=2) if n_new < T else cols
    r = eng.decide_ptr(None, 0, 0, 0, db, candidate_bits=cb, series_max=sm, in_kind=0, out_kind=0, resident=True)
    _check(db, cb, (r.n_series, r.n_candidates, r.n_decisions), oracle_c.decide(full), sm)


def test_error_paths(engines):
    import gpu_pruner_b200 as g
    eng = engines["ldg"]
    with pytest.raises(g.GprError) as ei:          # over capacity: more cells than the staging planes hold
        eng.decide(np.zeros((12001, 8, 2048), np.float32))
    assert ei.value.code == g.ffi.GPR_E_CAPACITY
    # only the number of cells counts (staging is dense): more pods / samples than the shape given at create
    # is fine as long as the product fits (ADVICE r1: a window that grows by one GPU slot must not fail)
    d = eng.decide(np.zeros((12001, 1, 8), np.float32))
    assert d.n_decisions == 12001
    d = eng.decide(np.zeros((3, 9, 2052), np.float32))
    assert d.n_decisions == 3
    torch.cuda.synchronize()
    with pytest.raises(g.GprError) as ei:          # missing required output
        eng.decide_ptr(torch.zeros(8, device="cuda:0"), 1, 1, 8, None)
    assert ei.value.code == g.ffi.GPR_E_INVALID
    with pytest.raises(g.GprError) as ei:          # stride smaller than the row
        eng.decide_ptr(torch.zeros(64, device="cuda:0"), 2, 1, 8, torch.zeros(1, dtype=torch.int32, device="cuda:0"),
                       row_stride=4)
    assert ei.value.code == g.ffi.GPR_E_INVALID
    fresh = g.IdleEngine(device=0)
    with pytest.raises(g.GprError) as ei:          # no resident window
        fresh.decide_ptr(None, 0, 0, 0, np.zeros(1, np.uint32), in_kind=0, out_kind=0, resident=True)
    assert ei.value.code == g.ffi.GPR_E_STATE
    with pytest.raises(g.GprError):                # bad device ordinal
        g.IdleEngine(device=99)
    fresh.close()
    # the context is still usable after errors
    d = eng.decide(np.zeros((5, 2, 8), np.float32))
    assert d.n_decisions == 5


def test_empty_window(engines):
    d = engines["ldg"].decide(np.zeros((0, 4, 16), np.float32))
    assert d.n_decisions == 0 and d.decision_bits.size == 0


def test_native_library_is_what_ran(engines):
    """the .so loaded is the in-tree libgpr.so and kernels were actually launched"""
    from gpu_pruner_b200 import ffi
    assert os.path.samefile(ffi.lib_path(), os.path.join(os.path.dirname(os.path.dirname(
        os.path.abspath(__file__))), "gpu-pruner_b200", "libgpr.so"))
    maps = open("/proc/self/maps").read()
    assert "libgpr.so" in maps
    assert engines["ldg"].launch_count() > 0 and engines["tma"].launch_count() > 0
    info = engines["ldg"].device_info()
    assert info["cc"] == (9, 0) and info["sm_count"] > 0


# ---------------------------------------------------------------------------------------------
# seeded fuzz over shape / stride / alignment / clause combinations, G up to the 32-slot limit
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("variant,mode", VARIANT_MODES, ids=VM_IDS)
@pytest.mark.parametrize("seed", range(24))
def test_fuzz_shapes(seed, variant, mode, engines, oracle_c, plan_exe, sm_count):
    rng = np.random.default_rng(10_000 + seed)
    P = int(rng.choice([1, 2, 31, 32, 33, 63, 100, 257, 1000, 3000]))
    G = int(rng.choice([1, 2, 3, 4, 5, 7, 8, 16, 31, 32]))
    T = int(rng.choice([1, 3, 4, 7, 16, 60, 179, 180, 181, 900, 1800, 2047, 2052]))
    if P * G * T > 6_000_000:
        P = max(1, 6_000_000 // (G * T))
    pad = int(rng.choice([0, 0, 1, 3, 4, 12]))
    off = int(rng.choice([0, 0, 1, 2, 3]))
    with_power, with_gates = bool(rng.integers(2)), bool(rng.integers(2))
    u, kw = _random_window(rng, P, G, T, with_power, with_gates)
    exp = oracle_c.decide(u, **kw)
    stride = T + pad

    def plane(x):
        buf = np.full(off + P * G * stride + 8, 77.0, np.float32)      # poison: never part of a window
        buf[off: off + P * G * stride].reshape(P * G, stride)[:, :T] = x.reshape(P * G, T)
        return torch.from_numpy(buf).to("cuda:0")

    ut = plane(u)
    wt = plane(kw["power"]) if with_power else None
    et = torch.from_numpy(kw["eligible"]).to("cuda:0") if with_gates else None
    ct = torch.from_numpy(kw["created_ts"]).to("cuda:0") if with_gates else None
    assert_ran(plan_exe, sm_count, variant, mode, T, P * G * (2 if with_power else 1),
               T % 4 == 0 and stride % 4 == 0 and off == 0)
    W = (P + 31) // 32
    db = torch.full((W,), -1, dtype=torch.int32, device="cuda:0")
    cb = torch.full((W,), -1, dtype=torch.int32, device="cuda:0")
    sm = torch.zeros(P * G, dtype=torch.float32, device="cuda:0") if mode == "whole" else None
    isl = torch.full((P,), -1, dtype=torch.int32, device="cuda:0") if mode == "early" else None
    torch.cuda.synchronize()
    r = engines[variant].decide_ptr(ut[off:].data_ptr(), P, G, T, db,
                                    power=None if wt is None else wt[off:].data_ptr(), eligible=et,
                                    created_ts=ct, cutoff_ts=kw.get("cutoff_ts", 0),
                                    power_threshold=kw.get("power_threshold", 0.0), candidate_bits=cb,
                                    series_max=sm, row_stride=stride, idle_slots=isl)
    _check(db.cpu().numpy().view(np.uint32), cb.cpu().numpy().view(np.uint32),
           (r.n_series, r.n_candidates, r.n_decisions), exp,
           None if sm is None else sm.cpu().numpy().reshape(P, G), None if isl is None else isl.cpu().numpy())


def test_gpu_slot_limit(engines):
    import gpu_pruner_b200 as g
    eng = engines["tma"]
    # all 32 slots usable: only the last GPU of each pod is idle
    P, G, T = 40, 32, 16
    u = np.full((P, G, T), 5.0, np.float32)
    u[:, 31, :] = 0.0
    bits, cbits, counts, smax, _, _ = _device_decide(eng, u)
    assert counts == (P, P, P) and int(np.unpackbits(cbits.view(np.uint8)).sum()) == P
    with pytest.raises(g.GprError) as ei:
        eng.decide(np.zeros((2, 257, 4), np.float32))
    assert ei.value.code == g.ffi.GPR_E_UNSUPPORTED


@pytest.mark.parametrize("variant,mode", VARIANT_MODES, ids=VM_IDS)
@pytest.mark.parametrize("G", [33, 64, 65, 100, 256])
def test_pods_with_more_than_32_series_slots(G, variant, mode, engines, oracle_c, oracle_np, plan_exe, sm_count):
    """ADVICE r1: a pod may carry more than 32 series (duplicate exporters, a pod name reused across hosts): the
    per-pod flag mask is ceil(G / 32) words; verdicts, counts, every row's idle slot and the power veto equal the
    oracle's"""
    eng = engines[variant]
    rng = np.random.default_rng(G)
    P, T = 70, 24
    u = rng.choice(np.array([0, 0, 3, 50], np.float32), size=(P, G, T))
    u[rng.random((P, G)) < 0.6] = 7.0                       # most series busy
    u[rng.random((P, G)) < 0.1] = np.nan                    # some absent
    u[5] = 9.0
    u[5, G - 1] = 0.0                                       # the only idle series sits in the last mask word
    w = rng.choice(np.array([50, 60, 149, 151], np.float32), size=(P, G, T), p=[0.5, 0.47, 0.02, 0.01])
    w[7] = 60.0
    w[7, G - 1, 3] = 400.0                                  # the veto too
    e = (rng.random(P) < 0.9).astype(np.uint8)
    for thr in (0.0, 150.0):
        assert_ran(plan_exe, sm_count, variant, mode, T, P * G * (2 if thr else 1))
        d = eng.decide(u, w, e, power_threshold=thr, want_series_max=mode == "whole", want_veto=True,
                       want_idle_slots=mode == "early")
        exp = oracle_c.decide(u, w, e, power_threshold=thr)
        _check(d.decision_bits, d.candidate_bits, (d.n_series, d.n_candidates, d.n_decisions), exp, d.series_max,
               d.idle_slots)
        assert np.array_equal(d.veto_bits, oracle_np.decide(u, w, e, power_threshold=thr)["veto_bits"])
    # device-resident window through the same kernels
    bits, cbits, counts, smax, _, islots = _device_decide(eng, u, **_outputs(mode))
    exp0 = oracle_c.decide(u)
    _check(bits, cbits, counts, exp0, smax, islots)


def test_memory_and_timing_helpers(engines):
    """the small utility entry points of include/gpr.h: device/pinned allocation, copies, timer, L2 flush"""
    eng = engines["tma"]
    n = 1 << 16
    d = eng.device_alloc(4 * n)
    h = eng.host_array((n,), np.float32)
    h[:] = np.arange(n, dtype=np.float32)
    eng.memcpy(d, h, 4 * n, 1, 0)
    back = np.zeros(n, np.float32)
    eng.memcpy(back, d, 4 * n, 0, 1)
    assert np.array_equal(back, h)
    eng.timer_begin()
    eng.flush_l2()
    ms = eng.timer_end()
    assert ms > 0
    # a window living in gpr_device_alloc memory works like any other device pointer
    P, G, T = 64, 4, 256
    assert P * G * T == n
    h[:] = 0.0
    h.reshape(P, G, T)[::2] = 3.0
    eng.memcpy(d, h, 4 * n, 1, 0)
    bits = np.zeros(2, np.uint32)
    r = eng.decide_ptr(d, P, G, T, bits, out_kind=0)
    assert r.n_decisions == P // 2 and bits[0] == 0xAAAAAAAA and bits[1] == 0xAAAAAAAA
    eng.device_free(d)
    before = eng.launch_count()
    eng.decide(np.zeros((3, 1, 4), np.float32))
    assert eng.launch_count() >= before + 2          # one reduce + one fold


@pytest.mark.parametrize("variant", VARIANTS)
def test_step_stamps(variant, engines):
    """gpr_step_stamps: one %globaltimer completion stamp per retired decision, increasing, after the mark
    of gpr_timer_begin, consistent with the CUDA-event time of the same region"""
    import gpu_pruner_b200 as g
    eng = engines[variant]
    P, G, T = 2048, 4, 600
    u, _, e = _synth_device(eng, 4242, P, G, T, False)
    db = torch.zeros(P // 32, dtype=torch.int32, device="cuda:0")
    torch.cuda.synchronize()
    batch = eng.make_batch([dict(util=u, eligible=e, P=P, G=G, T=T, decision_bits=db)] * 16)
    eng.decide_batch_async(batch)
    eng.sync()
    eng.timer_begin()
    eng.decide_batch_async(batch)
    ms = eng.timer_end()
    eng.sync()
    t0, st = eng.step_stamps()
    assert len(st) == 16 and t0 > 0
    d = np.diff(np.concatenate([np.array([t0], np.uint64), st]).astype(np.int64))
    assert np.all(d > 0)
    assert abs(d.sum() / 1e6 - ms) < 0.25 * ms + 0.05
    # a blocking call retires exactly one decision
    eng.decide_ptr(u, P, G, T, db, eligible=e)
    assert len(eng.step_stamps()[1]) == 1
    with pytest.raises(g.GprError):
        eng.p2p_debug(7)
    eng.p2p_debug(0)


@pytest.mark.parametrize("variant", VARIANTS)
def test_veto_bits_output(variant, engines, oracle_np):
    """gpr_result.veto_bits: the pods with a power series at or above the threshold (query.promql.j2:36-44), whether or
    not they have an idle GPU — what the host needs to re-derive a pod's verdict (exact `sum by`)"""
    eng = engines[variant]
    rng = np.random.default_rng(17)
    P, G, T = 333, 3, 64
    u = rng.choice(np.array([0, 0, 9], np.float32), size=(P, G, T))
    w = rng.choice(np.array([50, 149.5, 150, 700], np.float32), size=(P, G, T), p=[0.9, 0.08, 0.01, 0.01])
    w[rng.random((P, G)) < 0.2] = np.nan
    exp = oracle_np.decide(u, w, power_threshold=150.0)
    d = eng.decide(u, w, power_threshold=150.0, want_veto=True)
    assert np.array_equal(d.veto_bits, exp["veto_bits"]) and np.array_equal(d.candidate_bits, exp["candidate_bits"])
    assert 0 < int(exp["veto"].sum()) < P
    d0 = eng.decide(u, w, power_threshold=0.0, want_veto=True)          # clause absent: nobody is vetoed
    assert not d0.veto_bits.any()
    # device window, device output
    vb = torch.full(((P + 31) // 32,), 0x5A5A5A5A, dtype=torch.int32, device="cuda:0")
    db = torch.zeros((P + 31) // 32, dtype=torch.int32, device="cuda:0")
    ut, wt = torch.from_numpy(u).cuda(), torch.from_numpy(w).cuda()
    torch.cuda.synchronize()
    eng.decide_ptr(ut, P, G, T, db, power=wt, power_threshold=150.0, veto_bits=vb)
    assert np.array_equal(vb.cpu().numpy().view(np.uint32), exp["veto_bits"])
