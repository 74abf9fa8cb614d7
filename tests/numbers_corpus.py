"""Decimal inputs for the number conversion of the device text parser, and the host build of that conversion
(tests/cpp/number_check.cpp).  TEST INFRASTRUCTURE, shared by tests/test_text_numbers.py (the parser core compiled
by g++) and tests/test_gpu_text_numbers.py (the same core in k_text_parse on the GPU), so both draw the same
inputs.  The expected answers are computed by each test, never here."""
import os
import random
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def build_number_check(out: str) -> str:
    """compile tests/cpp/number_check.cpp (gpr_text.cuh as plain C++) to `out`"""
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fsanitize=undefined", "-fno-sanitize-recover=all",
                           os.path.join(ROOT, "tests", "cpp", "number_check.cpp"), "-o", str(out)])
    return str(out)


def run_number_check(driver: str, lines: list) -> list:
    """one output line per input line (see number_check.cpp for the commands)"""
    r = subprocess.run([driver], input="\n".join(lines) + "\n", capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr[-2000:]
    out = r.stdout.splitlines()
    assert len(out) == len(lines)
    return out


def eisel_lemire_cases():
    """(mantissa, exp10) pairs: random mantissas of 1..19 digits at random exponents, the shortest round-trip
    representations of random doubles (the second value: that subset, which Prometheus prints) and the numbers at
    and around rounding boundaries"""
    rng = random.Random(20260921)
    cases = []
    realistic = set()
    for _ in range(120_000):
        nd = rng.randrange(1, 20)
        man = rng.randrange(10 ** (nd - 1), 10 ** nd)
        if man >= 1 << 64:
            continue
        cases.append((man, rng.randrange(-340, 300)))
    # shortest-round-trip representations of random doubles (what Prometheus prints), as mantissa / exponent
    for _ in range(80_000):
        x = rng.random() if rng.random() < 0.7 else rng.uniform(0, 1000)
        s = repr(x)
        if "e" in s or "." not in s:
            continue
        ip, fp = s.split(".")
        cases.append((int(ip + fp), -len(fp)))
        realistic.add(cases[-1])
    cases += boundary_cases()
    return cases, realistic


def boundary_cases():
    """(mantissa, exp10) at and around rounding boundaries"""
    cases = []
    for k in (53, 54, 60, 63):
        for d in (-1, 0, 1):
            cases.append(((1 << k) + d, 0))
            cases.append(((1 << k) + d, -5))
    cases += [(9007199254740993, 0), (9007199254740993, -3), (1, -324), (1, 308), (17976931348623157, 292),
              (22250738585072014, -324), (4, -324), (12345678901234567890, 0), (1, 0), (5, -1)]
    return cases


def value_texts():
    """sample value spellings: a list of edge forms, then shortest round-trip reprs of random doubles with some
    scaled, integer and negated forms among them"""
    rng = random.Random(7)
    texts = ["0", "-0", "100", "37", "0.5", "0.25", "12.25", "0.30000000000000004", "123456789012345678",
             "0.1", "0.07", "99.99999999999999", "1234567.1234567", "16777216", "16777217", "4294967296.5",
             "0.000000000000000000000000000000000000000000001", "0.0000000000000000000000000000000000000000000001",
             "340282350000000000000000000000000000000", "0.1234567890123456789", "1.7976931348623157",
             "000123", "0.000", "5.0000000000000000000", "5e-07", "1.2345e+21", "1e2", "1E1", "1e-50", "1e23",
             "9.999999e-07", "1e+21", "0e0", "3.4028235e+38", "1e39", "4.9e-324", "1.5e-46"]
    for _ in range(60_000):
        x = rng.random() if rng.random() < 0.6 else rng.uniform(0, 700)
        texts.append(repr(x))          # includes Go-style exponent forms for the tiny ones ("5e-07")
        if rng.random() < 0.05:
            texts.append(repr(x * 10.0 ** rng.randrange(-30, 30)))
        if rng.random() < 0.1:
            texts.append(str(rng.randrange(0, 101)))
        if rng.random() < 0.05:
            texts.append("-" + texts[-1])
    return texts
