"""k_reduce_probe on the H100, through libgpr.so with the AUTO kernel (the one that runs when every row may stop):
the windows of tests/test_probe_emul.py (a settling sample at every head and chunk boundary, and the f32 edge values)
from dense, strided, host (staged) and resident-ring memory, with the power plane on and off; a PDL batch in which
early-exit calls alternate with series_max calls, so the probe kernel and k_reduce_tma follow each other with different
shared-memory footprints; the C2- and C3-shaped synthetic windows; and every ring layout the kernel can take, all
against the oracles."""
import numpy as np
import pytest
import torch

import geometry
import test_early_exit_emul as EE
import test_probe_emul as PE
from test_gpu_geometry import DEV, _check, _device_decide, _oracle_synth, _synth, _u32

pytestmark = pytest.mark.gpu
THR = PE.THR


@pytest.fixture(scope="module")
def plan_exe(tmp_path_factory):
    return geometry.build(tmp_path_factory.mktemp("launch_plan"))


def _windows():
    out = []
    for T in (1800, 3600, 100):
        out.append((f"boundary T{T}", PE._boundary_window(T, False), PE._boundary_window(T, True)))
        out.append((f"edges T{T}", EE._edge_window(T, PE.HEAD), EE._edge_power(T, PE.HEAD)))
    return out


def test_boundary_and_edge_windows(oracle_np):
    import gpu_pruner_b200 as g
    with g.IdleEngine(device=0, max_pods=64, max_gpus=4, max_samples=3600, power_plane=True) as eng:
        for name, util, power in _windows():
            P, G, T = util.shape
            for use_power in (False, True):
                exp = oracle_np.decide(util, power if use_power else None, None, None, 0, THR if use_power else 0.0)
                thr = THR if use_power else 0.0
                # device memory: dense and strided (ld = T + 4): both are bulk-copied
                for stride in (0, T + 4):
                    ld = stride or T
                    rows = np.full((P * G, ld), 77.0, np.float32)
                    rows[:, :T] = util.reshape(P * G, T)
                    u_t = torch.from_numpy(rows).to(DEV)
                    w_t = None
                    if use_power:
                        wrows = np.full((P * G, ld), 1e9, np.float32)
                        wrows[:, :T] = power.reshape(P * G, T)
                        w_t = torch.from_numpy(wrows).to(DEV)
                    bits, cbits, counts, _, vb, _ = _device_decide(
                        eng, u_t.data_ptr(), P, G, T, w_t.data_ptr() if use_power else None, {}, thr,
                        stride=stride, want_smax=False, want_veto=True)
                    _check(bits, cbits, counts, exp, None, vb if use_power else None)
                # pinned host memory, through the staging planes
                d = eng.decide(util, power if use_power else None, None, None, 0, thr, want_veto=use_power)
                tag = (name, use_power)
                assert np.array_equal(d.decision_bits, exp["decision_bits"]), tag
                assert (d.n_series, d.n_candidates, d.n_decisions) == (
                    exp["n_series"], exp["n_candidates"], exp["n_decisions"]), tag


@pytest.mark.parametrize("power", [False, True], ids=["util", "util+power"])
def test_resident_window_ring(power, oracle_c):
    """daemon mode without series_max: columns appended tick by tick into the HBM ring, every head position"""
    import gpu_pruner_b200 as g
    seed, P, G, T = 0x5EED0005, 777, 4, 240
    full = oracle_c.synth_fill(seed, 0, 0, P, G, 900)
    fullw = oracle_c.synth_fill(seed, 1, 0, P, G, 900)
    with g.IdleEngine(device=0) as eng:
        eng.resident_init(P, G, T, power_plane=power)
        W = (P + 31) // 32
        db, cb = np.zeros(W, np.uint32), np.zeros(W, np.uint32)
        t = 0
        for n_new in (60, 1, 179, 240, 37, 300, 83):
            eng.append(full[:, :, t:t + n_new], fullw[:, :, t:t + n_new] if power else None)
            t += n_new
            r = eng.decide_ptr(None, 0, 0, 0, db, candidate_bits=cb, power_threshold=150.0 if power else 0.0,
                               in_kind=0, out_kind=0, resident=True)
            lo = max(0, t - T)
            win = np.full((P, G, T), np.nan, np.float32)
            win[:, :, : t - lo] = full[:, :, lo:t]
            winw = np.full((P, G, T), np.nan, np.float32)
            winw[:, :, : t - lo] = fullw[:, :, lo:t]
            exp = oracle_c.decide(win, winw if power else None, power_threshold=150.0 if power else 0.0)
            _check(db, cb, (r.n_series, r.n_candidates, r.n_decisions), exp)


def test_pdl_batch_alternating_with_series_max(oracle_c):
    """back-to-back decisions: early-exit calls (probe kernel, 197 KB per CTA at T 1800) interleaved with series_max
    calls (k_reduce_tma, 117 KB), so each kernel starts while the other drains"""
    import gpu_pruner_b200 as g
    rng = np.random.default_rng(5)
    with g.IdleEngine(device=0) as eng:
        calls, keep = [], []
        wins = _windows()
        for i in range(12):
            name, util, power = wins[i % len(wins)]
            util = util[rng.permutation(util.shape[0])]
            P, G, T = util.shape
            use_power, smax = i % 3 != 2, i % 2 == 1
            W = (P + 31) // 32
            c = dict(util=torch.from_numpy(np.ascontiguousarray(util)).to(DEV), P=P, G=G, T=T,
                     decision_bits=torch.full((W,), -1, dtype=torch.int32, device=DEV),
                     candidate_bits=torch.full((W,), -1, dtype=torch.int32, device=DEV))
            kw = {}
            if use_power:
                c["power"], c["power_threshold"] = torch.from_numpy(power).to(DEV), THR
                kw = {"power": power, "power_threshold": THR}
            if smax:
                c["series_max"] = torch.full((P * G,), -777.0, dtype=torch.float32, device=DEV)
            calls.append(c)
            keep.append((util, kw))
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


@pytest.mark.parametrize("shape", [(10000, 4, 1800), (20000, 8, 3600)], ids=["c2", "c3-shaped"])
def test_synthetic_windows_equal_the_c_oracle(shape, oracle_c):
    import gpu_pruner_b200 as g
    P, G, T = shape
    with g.IdleEngine(device=0) as eng:
        for power in (False, True):
            u, w, e = _synth(eng, 0x5EED0002, P, G, T, power)
            exp = _oracle_synth(oracle_c, 0x5EED0002, P, G, T, power, smax=False)
            for rep in range(2):
                bits, cbits, counts, _, vb, _ = _device_decide(
                    eng, u, P, G, T, w, {"eligible": e.cpu().numpy()}, 150.0 if power else 0.0, want_smax=False,
                    want_veto=power)
                _check(bits, cbits, counts, exp, None, vb if power else None)


def _ring_layouts(plan_exe, sm_count):
    """(stage_bytes, depth) -> the window lengths T = 4 .. 7200 (multiples of 4) whose probe ring has that layout"""
    Ts = list(range(4, 7201, 4))
    knobs = geometry.Knobs(sm_count=sm_count)
    out = {}
    for T, p in zip(Ts, geometry.plans(plan_exe, [(knobs, "auto", T, 1 << 20, True, False, 1, True) for T in Ts])):
        assert p.kernel == "probe", p
        out.setdefault((p.stage_bytes, p.depth), []).append(T)
    return out


def _base_rows(T, power, rng):
    """the rows a window is drawn from: a settling sample at every head and chunk boundary (one row each, and one
    that nothing settles), idle rows, and rows with gaps of no sample; -> (rows, how often each is drawn)"""
    quiet = 100.0 if power else 0.0
    boundary = PE._boundary_window(T, power).reshape(-1, T)
    idle = np.full((4, T), quiet, np.float32)
    gapped = np.full((8, T), quiet, np.float32)
    for r in range(gapped.shape[0]):
        for _ in range(3):
            a = int(rng.integers(0, T))
            gapped[r, a:a + int(rng.integers(1, max(2, T // 4)))] = np.nan
    gapped[-1] = np.nan                               # no sample at all: never idle, never vetoes
    rows = np.concatenate([boundary, idle, gapped])
    share = (0.2, 0.7) if power else (0.4, 0.3)         # (boundary, idle): the rest have gaps
    p = np.concatenate([np.full(len(boundary), share[0] / len(boundary)), np.full(len(idle), share[1] / len(idle)),
                        np.full(len(gapped), (1 - sum(share)) / len(gapped))])
    return rows, p


def _pack(flags):
    b = np.zeros((len(flags) + 31) // 32 * 32, bool)
    b[:len(flags)] = flags
    return np.packbits(b, bitorder="little").view("<u4")


def test_every_ring_layout(plan_exe, oracle_c):
    """each of the probe kernel's ring layouts (stage size and depth, gpr_launch.h probe_layout) at the shortest and
    the longest window that takes it: enough rows that every warp of every CTA refills its ring several times, and a
    single series (P = G = 1, fewer rows than one CTA has stages); util alone and util + power, with gates; the bitmaps,
    counts, veto bits and every row's idle slot against the oracle"""
    import gpu_pruner_b200 as g
    with g.IdleEngine(device=0) as eng:
        sm_count = eng.device_info()["sm_count"]
        layouts = _ring_layouts(plan_exe, sm_count)
        assert len(layouts) == 16 and {d for _, d in layouts} >= {3, 32}
        for (stage_bytes, depth), Ts in sorted(layouts.items()):
            for T in sorted({Ts[0], Ts[-1]}):
                rng = np.random.default_rng(T)
                for use_power in (False, True):
                    planes = 2 if use_power else 1
                    for many in (True, False):
                        G = 4 if many else 1
                        # 4 rows per warp stage: each ring is refilled with new rows at least 3 times
                        P = -(-4 * sm_count * 32 * depth // (planes * G)) if many else 1
                        rows, pr = _base_rows(T, False, rng)
                        u = rows[rng.choice(len(rows), P * G, p=pr)].reshape(P, G, T)
                        w = None
                        if use_power:
                            rows, pr = _base_rows(T, True, rng)
                            w = rows[rng.choice(len(rows), P * G, p=pr)].reshape(P, G, T)
                        kw = {"eligible": (rng.random(P) < 0.9).astype(np.uint8),
                              "created_ts": rng.integers(1000, 2000, P).astype(np.int64), "cutoff_ts": 1500}
                        thr = THR if use_power else 0.0
                        tag = (T, stage_bytes, depth, use_power, P, G)
                        p = geometry.plan(plan_exe, geometry.Knobs(sm_count=sm_count), "auto", T, P * G * planes,
                                          True, False, P, True)
                        assert p.kernel == "probe" and (p.stage_bytes, p.depth) == (stage_bytes, depth), (tag, p)
                        assert p.grid == (sm_count if many else 1), (tag, p)
                        assert (P * G * planes >= 3 * p.grid * 32 * depth) if many else (P * G * planes < 32 * depth)
                        exp = oracle_c.decide(u, w, kw["eligible"], kw["created_ts"], kw["cutoff_ts"], thr,
                                              n_threads=8)
                        exp["veto_bits"] = _pack(np.any(w.astype(np.float64) >= THR, axis=(1, 2)) if use_power
                                                 else np.zeros(P, bool))
                        assert 0 < exp["n_candidates"] < P or not many, tag
                        u_t = torch.from_numpy(u).to(DEV)
                        w_t = torch.from_numpy(w).to(DEV) if use_power else None
                        bits, cbits, counts, _, vb, isl = _device_decide(eng, u_t, P, G, T, w_t, kw, thr,
                                                                          want_smax=False, want_veto=True,
                                                                          want_slots=True)
                        _check(bits, cbits, counts, exp, None, vb, isl)
                        del u_t, w_t
