"""CPU: the number conversion of the device-side text parser (gpu-pruner_b200/csrc/gpr_text.cuh: Clinger's fast
path + Eisel-Lemire with the generated 128-bit table) against Python's correctly rounded float().

The parser's contract is "equal to strtod + (float), or decline" (a declined number marks the span hard and the
CPU's strtod decides), so every ACCEPTED conversion must match bit for bit; the rate of declines on realistic input
(17-digit DCGM_FI_PROF_GR_ENGINE_ACTIVE ratios: shortest-round-trip doubles) must be negligible."""
import math
import os
import random
import struct

import numpy as np
import pytest

import numbers_corpus as NC

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def driver(tmp_path_factory):
    return NC.build_number_check(tmp_path_factory.mktemp("num") / "number_check")


def _run(driver, lines):
    return NC.run_number_check(driver, lines)


def _bits64(x):
    return struct.unpack("<Q", struct.pack("<d", x))[0]


def test_pow10_table_is_what_the_generator_writes():
    """the committed header is the generator's output (exact big-integer arithmetic)"""
    import importlib.util
    spec = importlib.util.spec_from_file_location("gen", os.path.join(ROOT, "tools", "gen_pow10_table.py"))
    gen = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(gen)
    text = open(os.path.join(ROOT, "gpu-pruner_b200", "csrc", "gpr_pow10_table.h")).read()
    for q in (-348, -27, -1, 0, 1, 22, 27, 55, 347):
        m = gen.mantissa128(q)
        assert f"{{0x{m >> 64:016X}ull, 0x{m & (2**64 - 1):016X}ull}}, /* 1e{q} */" in text
    assert gen.mantissa128(0) == 1 << 127 and gen.mantissa128(-1) >> 64 == 0xCCCCCCCCCCCCCCCC


def test_eisel_lemire_matches_correct_rounding(driver):
    cases, realistic = NC.eisel_lemire_cases()
    out = _run(driver, [f"E {m} {e}" for m, e in cases])
    declined = 0
    for (m, e), line in zip(cases, out):
        ok, bits = line.split()
        if ok == "0":
            declined += 1
            assert (m, e) not in realistic, (m, e)     # what Prometheus prints is always decided on the device
            continue   # subnormal / overflowing results (random exponents reach both) or a genuine half-way case
        want = float(f"{m}e{e}")
        assert int(bits, 16) == _bits64(want), (m, e, bits, hex(_bits64(want)))
    assert declined < len(cases) // 20


def test_parse_value_matches_strtod_then_float(driver):
    texts = NC.value_texts()
    out = _run(driver, ["V " + t for t in texts])
    declined = []
    for t, line in zip(texts, out):
        q, bits, tiny = line.split()
        if q == "0":
            declined.append(t)
            continue
        want = np.float32(float(t))
        if float(t) != 0.0 and want == 0.0:      # below the f32 denormal range: kept non-zero (to_f32 in ingest.cpp)
            assert int(bits, 16) in (0x00000001, 0x80000001) and tiny == "1", t
            continue
        assert int(bits, 16) == struct.unpack("<I", struct.pack("<f", want))[0], (t, bits)
    # declined: more than 19 significant digits, results in the subnormal range, and the handful of exactly-half-way
    # products Eisel-Lemire leaves to a slower method — never a shortest-round-trip decimal below 1e21
    realistic = {t for t in texts if "e" not in t and 0 <= float(t) <= 1000}
    for t in declined:
        digits = len(t.lstrip("-+").split("e")[0].replace(".", "").lstrip("0"))
        assert digits > 19 or t not in realistic, t
    assert len(declined) < len(texts) // 100, declined[:10]
    assert "0.30000000000000004" not in declined and "123456789012345678" not in declined


def test_parse_value_declines_what_it_cannot_decide(driver):
    out = _run(driver, ["V .5", "V 5.", "V 12345678901234567890", "V 1.2.3", "V abc", "V +", "V 0x10",
                        "V 1234567890123456789012", "V 1e", "V 1e+", "V 1e1234", "V e5", "V 1.e5"])
    assert all(line.split()[0] == "0" for line in out), out


def test_power_samples_snapped_to_the_threshold_decide_like_float64(driver):
    """parse_value into the power plane (power_snap / snap_power): for every threshold — exact in f32 or not, tiny,
    negative, beyond the f32 range — the stored f32 compares `>= up` (the smallest f32 >= thr, what gpr_decide
    compares with) exactly when the float64 reading compares `>= thr`, as Prometheus does; it is the plain f32
    rounding wherever that already agrees, and one step off it otherwise.  0 and NaN turn the snap off."""
    import edges as E
    rng = random.Random(150)
    thresholds = E.THRESHOLDS + [1e-40, -5.0, 1e-3, 123456.789, 3.4028235677973366e38, 1e39]
    cases = []
    for thr in thresholds:
        vals = E.power_edges(thr) + [thr * (1 + rng.uniform(-1e-7, 1e-7)) for _ in range(200)]
        vals += [0.0, -0.0, thr / 2, thr * 2, 1e-45, 1e-50]
        cases += [(thr, v) for v in vals if math.isfinite(v)]     # (NaN / Inf are parse_sample's, never snapped)
    cases += [(t, 149.999999) for t in (0.0, math.nan)] + [(t, 150.5) for t in (0.0, math.nan)]
    out = _run(driver, [f"S {thr!r} {E.go_float(v)}" for thr, v in cases])
    f32 = lambda b: float(np.frombuffer(struct.pack("<I", b), np.float32)[0])
    flipped = 0
    for (thr, v), line in zip(cases, out):
        q, bits, up, down = (int(x, 16) if i else int(x) for i, x in enumerate(line.split()))
        assert q, (thr, v)
        # rn: the plain f32 rounding, a non-zero value below the f32 range kept at +-denorm_min (to_f32)
        got, rn = f32(bits), float(np.float32(v)) if np.float32(v) != 0 or v == 0 else math.copysign(f32(1), v)
        if thr == 0 or math.isnan(thr):
            assert got == rn, (thr, v)
            continue
        assert f32(up) == E.f32_up(thr) and f32(down) == float(np.nextafter(np.float32(E.f32_up(thr)), np.float32(-np.inf)))
        assert (got >= f32(up)) == (v >= thr) and (got >= thr) == (v >= thr), (thr, v, got)
        if (rn >= f32(up)) == (v >= thr):
            assert got == rn, (thr, v, got, rn)
        else:
            flipped += 1
            assert got in (f32(up), f32(down)), (thr, v, got)
    # the cases that matter are there: plain rounding would have decided them wrongly
    assert flipped >= 10
    assert out[cases.index((150.0, 149.999999))].split()[1] == "4315ffff"        # 149.999999 -> just below 150.0f
    assert out[cases.index((149.99, 149.99))].split()[1] == "4315fd71"           # == a decimal threshold: vetoes


def test_parse_timestamp_is_exact_in_milliseconds(driver):
    texts = ["1700000000", "1700000000.4", "1700000000.5", "1700000000.499", "1700000000.500", "1700000000.123",
             "0", "0.001", "9999999999999", "4000000000000", "3999999999999.5", "1700000000.05"]
    out = _run(driver, ["T " + t for t in texts])
    for t, line in zip(texts, out):
        q, ts = line.split()
        assert int(q) == len(t) + 1, t
        x = float(t)
        if not (x < 4e12):
            assert int(ts) < -(1 << 60)          # "no sane epoch time": far outside every window
        else:
            assert int(ts) == round(x * 1000), t  # what the CPU path computes: llround(strtod(t) * 1000)
    # finer than a millisecond, signs, exponents: declined (the span goes to the CPU parser)
    out = _run(driver, ["T 1700000000.1234", "T 17000000001234", "T -5", "T +5", "T 1e9", "T ", "T 5."])
    assert all(line.split()[0] == "0" for line in out), out
