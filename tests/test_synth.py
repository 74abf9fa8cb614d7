"""CPU: the synthetic DCGM universe is identical in the C oracle and the numpy oracle, and has
the class mix SURVEY.md §8(d) asks for.  (The CUDA generator is checked against these on the GPU.)"""
import numpy as np
import pytest

SEED = 0x5EED0002


@pytest.mark.parametrize("P,G,T,off", [(50, 4, 64, 0), (33, 1, 7, 1000), (20, 8, 180, 12345), (5, 4, 1800, 99)])
@pytest.mark.parametrize("plane", [0, 1])
def test_c_and_numpy_generators_agree(P, G, T, off, plane, oracle_c, oracle_np):
    a = oracle_c.synth_fill(SEED, plane, off, P, G, T, n_threads=3)
    b = oracle_np.synth_fill(SEED, plane, off, P, G, T)
    assert a.dtype == b.dtype == np.float32
    assert np.array_equal(a.view(np.uint32) & 0x7fffffff, b.view(np.uint32) & 0x7fffffff) or \
        np.all((a == b) | (np.isnan(a) & np.isnan(b)))
    assert np.all((a == b) | (np.isnan(a) & np.isnan(b)))


def test_offset_windows_are_slices_of_one_universe(oracle_c):
    full = oracle_c.synth_fill(SEED, 0, 0, 96, 4, 50)
    part = oracle_c.synth_fill(SEED, 0, 32, 32, 4, 50)
    assert np.all((full[32:64] == part) | (np.isnan(full[32:64]) & np.isnan(part)))


def test_eligibility_agrees_and_rate(oracle_c, oracle_np):
    a = oracle_c.synth_eligible(SEED, 7, 20000)
    b = oracle_np.synth_eligible(SEED, 7, 20000)
    assert np.array_equal(a, b)
    assert 0.93 < a.mean() < 0.97  # 5 % ineligible


def test_class_mix(oracle_np):
    P, G, T = 4000, 4, 120
    u = oracle_np.synth_fill(SEED, 0, 0, P, G, T).reshape(P * G, T)
    with np.errstate(invalid="ignore"):
        m = np.fmax.reduce(u.astype(np.float64), axis=1)
    nz = np.sum(np.nan_to_num(u) > 0, axis=1)
    idle_like = (m == 0)                       # idle class + gappy-idle + bursts eaten by a gap
    burst = (nz == 1)
    assert 0.30 < idle_like.mean() < 0.36
    assert 0.08 < burst.mean() < 0.12
    assert 0.0005 < np.isnan(u[m > 0]).mean() < 0.03
    # values are small non-negative integers, exactly representable
    v = u[~np.isnan(u)]
    assert v.min() >= 0 and v.max() <= 100 and np.all(v == np.round(v))
    w = oracle_np.synth_fill(SEED, 1, 0, 200, G, T)
    wv = w[~np.isnan(w)]
    assert wv.min() >= 40 and wv.max() <= 700


def test_streaming_decision_equals_materialised(oracle_c):
    P, G, T = 500, 4, 90
    u = oracle_c.synth_fill(SEED, 0, 64, P, G, T)
    w = oracle_c.synth_fill(SEED, 1, 64, P, G, T)
    e = oracle_c.synth_eligible(SEED, 64, P)
    a = oracle_c.decide(u, w, e, power_threshold=150.0)
    b = oracle_c.decide_synth(SEED, 64, P, G, T, use_power=True, power_threshold=150.0, use_elig=True,
                              n_threads=4)
    for k in ("decision_bits", "candidate_bits", "n_series", "n_candidates", "n_decisions"):
        assert np.array_equal(a[k], b[k]), k
    c = oracle_c.decide(u)
    d = oracle_c.decide_synth(SEED, 64, P, G, T)
    assert np.array_equal(c["decision_bits"], d["decision_bits"])
    assert 0 < c["n_decisions"] < P


def test_streaming_decision_series_max_and_veto(oracle_c, oracle_np):
    """decide_synth's optional outputs (used to check every row of device windows too large for host RAM)"""
    import kat
    P, G, T = 203, 3, 61
    b = oracle_c.decide_synth(SEED, 5, P, G, T, use_power=True, power_threshold=150.0, use_elig=True, n_threads=3,
                              want_series_max=True, want_veto=True)
    u = oracle_c.synth_fill(SEED, 0, 5, P, G, T)
    w = oracle_c.synth_fill(SEED, 1, 5, P, G, T)
    a = oracle_np.decide(u, w, oracle_c.synth_eligible(SEED, 5, P), None, 0, 150.0)
    for k in ("decision_bits", "candidate_bits", "veto_bits", "n_series", "n_candidates", "n_decisions"):
        assert np.array_equal(a[k], b[k]), k
    assert kat.smax_equal(b["series_max"], a["series_max"])
    assert 0 < int(np.unpackbits(b["veto_bits"].view(np.uint8)).sum()) < P
    c = oracle_c.decide_synth(SEED, 5, P, G, T, want_veto=True)      # no power clause: nobody is vetoed
    assert not c["veto_bits"].any()
