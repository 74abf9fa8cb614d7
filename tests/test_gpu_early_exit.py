"""Early exit on the H100: the windows of tests/test_early_exit_emul.py (a settling sample at every head, chunk and
batch boundary, and the f32 edge values) through libgpr.so with both reduce kernels, from device memory (dense,
strided and 4 bytes off alignment) and from host memory through the staging path, with and without the power plane and
series_max; an async batch of unlike windows; and the C2 / C3 synthetic windows against the C oracle."""
import numpy as np
import pytest
import torch

import test_early_exit_emul as EE
from test_gpu_geometry import DEV, _check, _device_decide, _oracle_synth, _synth, _u32

pytestmark = pytest.mark.gpu


def _windows():
    out = []
    for T in (1800, 1000):
        util = EE._boundary_window(T, EE.LAYOUTS.values(), False)
        out.append((f"boundary T{T}", util, EE._boundary_window(T, EE.LAYOUTS.values(), True)))
        h = min(EE.HEAD, EE._tma_layout((1, 16, 8192, 3, 2), T)[1])
        out.append((f"edges T{T}", EE._edge_window(T, h), EE._edge_power(T, h)))
    return out


@pytest.mark.parametrize("kernel", ["ldg", "tma"])
def test_boundary_and_edge_windows(kernel, oracle_np):
    import gpu_pruner_b200 as g
    with g.IdleEngine(device=0, kernel=kernel, max_pods=64, max_gpus=4, max_samples=1800, power_plane=True) as eng:
        for name, util, power in _windows():
            P, G, T = util.shape
            for use_power in (False, True):
                exp = oracle_np.decide(util, power if use_power else None, None, None, 0, EE.THR if use_power else 0.0)
                for smax in (False, True):
                    tag = (kernel, name, use_power, smax)
                    # device memory: dense, strided (ld = T + 4) and 4 bytes off 16-byte alignment
                    for stride, offset in ((0, 0), (T + 4, 0), (0, 1)):
                        ld = stride or T
                        flat = np.full((P * G * ld + 4,), 77.0, np.float32)
                        rows = flat[offset:offset + P * G * ld].reshape(P * G, ld)
                        rows[:, :T] = util.reshape(P * G, T)
                        u_t = torch.from_numpy(flat).to(DEV)
                        w_t = w_dev = None
                        if use_power:
                            wflat = np.full((P * G * ld + 4,), 1e9, np.float32)
                            wrows = wflat[offset:offset + P * G * ld].reshape(P * G, ld)
                            wrows[:, :T] = power.reshape(P * G, T)
                            w_dev = torch.from_numpy(wflat).to(DEV)
                            w_t = w_dev[offset:].data_ptr()
                        bits, cbits, counts, sm, vb, _ = _device_decide(
                            eng, u_t[offset:].data_ptr(), P, G, T, w_t, {}, EE.THR if use_power else 0.0,
                            stride=stride, want_smax=smax, want_veto=True)
                        _check(bits, cbits, counts, exp, sm, vb if use_power else None)
                    # host memory, through the staging planes
                    d = eng.decide(util, power if use_power else None, None, None, 0,
                                   EE.THR if use_power else 0.0, want_series_max=smax, want_veto=use_power)
                    assert np.array_equal(d.decision_bits, exp["decision_bits"]), tag
                    assert (d.n_series, d.n_candidates, d.n_decisions) == (
                        exp["n_series"], exp["n_candidates"], exp["n_decisions"]), tag
                    if smax:
                        assert EE.KAT.smax_equal(d.series_max, exp["series_max"]), tag


@pytest.mark.parametrize("kernel", ["ldg", "tma"])
def test_async_batch_of_unlike_windows(kernel, oracle_c):
    """back-to-back decisions under PDL whose rows settle at different places: stages change rows mid-flight and
    the row counter restarts in every launch"""
    import gpu_pruner_b200 as g
    rng = np.random.default_rng(99)
    with g.IdleEngine(device=0, kernel=kernel) as eng:
        calls, keep = [], []
        wins = _windows()
        for i in range(10):
            name, util, power = wins[i % len(wins)]
            util = util[rng.permutation(util.shape[0])]
            P, G, T = util.shape
            use_power, smax = i % 3 != 0, i % 4 == 1
            W = (P + 31) // 32
            c = dict(util=torch.from_numpy(np.ascontiguousarray(util)).to(DEV), P=P, G=G, T=T,
                     decision_bits=torch.full((W,), -1, dtype=torch.int32, device=DEV),
                     candidate_bits=torch.full((W,), -1, dtype=torch.int32, device=DEV))
            kw = {}
            if use_power:
                c["power"], c["power_threshold"] = torch.from_numpy(power).to(DEV), EE.THR
                kw = {"power": power, "power_threshold": EE.THR}
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


@pytest.mark.parametrize("kernel", ["ldg", "tma"])
@pytest.mark.parametrize("shape", [(10000, 4, 1800), (20000, 8, 3600)], ids=["c2", "c3-shaped"])
def test_synthetic_windows_equal_the_c_oracle(kernel, shape, oracle_c):
    import gpu_pruner_b200 as g
    P, G, T = shape
    with g.IdleEngine(device=0, kernel=kernel) as eng:
        for power in (False, True):
            u, w, e = _synth(eng, 0x5EED0002, P, G, T, power)
            for smax in (False, True):
                exp = _oracle_synth(oracle_c, 0x5EED0002, P, G, T, power, smax=True)
                bits, cbits, counts, sm, vb, _ = _device_decide(
                    eng, u, P, G, T, w, {"eligible": e.cpu().numpy()}, 150.0 if power else 0.0, want_smax=smax,
                    want_veto=power)
                _check(bits, cbits, counts, exp, sm, vb if power else None)
