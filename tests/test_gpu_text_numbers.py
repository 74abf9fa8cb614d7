"""GPU: the device text parser's machine code (k_text_parse / k_text_scan_chunk, gpr_text.cuh and
gpr_text_kernels.cuh compiled for sm_90a) against plain Python references of the same operations.

tests/test_text_numbers.py and tests/test_text_device_cpu.py check the parser's source on the CPU; the device build
differs from it (the 128-bit product, clz, bit casts and the table of powers of ten have __CUDA_ARCH__ branches,
the merge into a cell is an integer atomicMax or a CAS loop, the upload is chunked with an overlap, the kernel lists
'[' offsets in passes of kListCap).  So here the device's output is compared with:
  * numbers: Python's correctly rounded float() (strtod), then the f32 rounding with the to_f32 clamp, bit for bit,
    and the device's float64 pinned exactly through the power snap (`x >= thr`, evaluated in double);
  * bucketing and merging: a model in integer milliseconds with a NaN-aware max per cell;
  * the scan: the offsets re.finditer finds, around every upload-chunk boundary.
Only the C ABI is driven (engine.py); the texts are bare sample lists whose spans the test hands to gpr_text_parse
itself.  The host build of the same parser core (tests/cpp/number_check.cpp) only says which values the core
declines — a declined value marks its span hard, which is the device's contract too."""
import decimal
import importlib.util
import math
import os
import random
import re
import struct

import numpy as np
import pytest

import edges as E
import numbers_corpus as NC

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
T_END = 1_700_000_000
FILL = 0xFFFFFFFF
M64 = (1 << 64) - 1
SPECIAL_BITS = {"+Inf": 0x7F800000, "Inf": 0x7F800000, "-Inf": 0xFF800000}
BAD_TS = object()          # a timestamp of 4e12 s or more: no sane epoch time, outside every window


# ---- engines and the host build ------------------------------------------------------------------------------
def _engine(**env):
    import gpu_pruner_b200 as g
    torch = pytest.importorskip("torch")
    if not torch.cuda.is_available():
        pytest.fail("-m gpu tests need a CUDA device; the engine has no CPU fallback")
    old = {k: os.environ.get(k) for k in env}
    os.environ.update(env)
    try:
        return g.IdleEngine(device=0)
    finally:
        for k, v in old.items():
            if v is None:
                del os.environ[k]
            else:
                os.environ[k] = v


@pytest.fixture(scope="module")
def eng():
    e = _engine()
    yield e
    e.close()


@pytest.fixture(scope="module")
def driver(tmp_path_factory):
    return NC.build_number_check(tmp_path_factory.mktemp("num") / "number_check")


def _host_declines(driver, texts):
    """the values the parser core declines (a '0' from number_check's V command); NaN / +-Inf are the sample
    grammar's, never declined"""
    num = [t for t in texts if t not in SPECIAL_BITS and t != "NaN"]
    out = NC.run_number_check(driver, ["V " + t for t in num])
    return {t for t, line in zip(num, out) if line.split()[0] == "0"}


# ---- references ----------------------------------------------------------------------------------------------
def _f32(bits):
    return float(np.uint32(bits).view(np.float32))


def _want_bits(text):
    """strtod + (float) with the to_f32 clamp (a non-zero value that rounds to 0 is kept at +-denorm_min), as the
    bits the plane holds; None for NaN, which never replaces anything"""
    if text == "NaN":
        return None
    if text in SPECIAL_BITS:
        return SPECIAL_BITS[text]
    x = float(text)
    with np.errstate(over="ignore"):
        f = np.float32(x)
    if f == 0 and x != 0:
        return 0x80000001 if x < 0 else 0x00000001
    return int(f.view(np.uint32))


def _tiny(text):
    if text == "NaN" or text in SPECIAL_BITS:
        return False
    x = float(text)
    with np.errstate(over="ignore"):
        return x != 0 and np.float32(x) == 0


def _ts_ms(t):
    """milliseconds of a timestamp text; None = the device declines it (sub-millisecond, more than 13 integer
    digits); BAD_TS = 4e12 s or later"""
    ip, dot, fp = t.partition(".")
    if not ip.isdigit() or len(ip) > 13 or (dot and not (fp.isdigit() and len(fp) <= 3)):
        return None
    if int(ip) >= 4_000_000_000_000:
        return BAD_TS
    return int(ip) * 1000 + int(fp.ljust(3, "0") if fp else 0)


def _column(ts, t_end_s, window_s, step_s, T, col_end):
    """t_lo < ts <= t_end (ms), back = (t_end - ts) // step, col = (col_end - back) mod T; -1 = outside"""
    t_end, t_lo = t_end_s * 1000, (t_end_s - window_s) * 1000
    if ts is BAD_TS or not (t_lo < ts <= t_end):
        return -1
    back = (t_end - ts) // (step_s * 1000)
    return -1 if back >= T else (col_end - back) % T


def _merge(plane, row, col, bits):
    """NaN-aware max: a NaN sample never replaces anything, anything replaces the fill"""
    if bits is None:
        return
    cur = plane[row, col]
    if cur == FILL or math.isnan(_f32(cur)) or _f32(cur) < _f32(bits):
        plane[row, col] = bits


def _reference(spans, grid, n_rows, T, plane=None, declined=frozenset()):
    """spans: [(row, [(ts_text, value_text), ...])]; grid: (t_end_s, window_s, step_s, col_end).
    -> (plane bits, hard flags, [n_in, n_oow, n_tiny] per span)"""
    plane = np.full((n_rows, T), FILL, np.uint32) if plane is None else plane
    hard = np.zeros(len(spans), bool)
    counts = np.zeros((len(spans), 3), np.int64)
    for i, (row, samples) in enumerate(spans):
        for ts_text, v in samples:
            ts = _ts_ms(ts_text)
            if ts is None or v in declined:
                hard[i] = True
                continue
            col = _column(ts, grid[0], grid[1], grid[2], T, grid[3])
            counts[i, 0] += 1
            if col < 0:
                counts[i, 1] += 1
                continue
            counts[i, 2] += _tiny(v)
            _merge(plane, row, col, _want_bits(v))
    return plane, hard, counts


def _assert_cells(got, want, what, describe=None):
    """cell for cell: == on the values (the sign of a zero max is not part of the contract), the fill bits
    exactly where no sample that is a number arrived"""
    gf, wf = got.view(np.float32), want.view(np.float32)
    bad = ~(((want == FILL) & (got == FILL)) | ((want != FILL) & (gf == wf)))
    if bad.any():
        idx = np.argwhere(bad)[:8]
        lines = [f"cell {tuple(int(x) for x in i)}: got {int(got[tuple(i)]):08x} want {int(want[tuple(i)]):08x}"
                 + (f" ({describe(*i)})" if describe else "") for i in idx]
        pytest.fail(f"{what}: {int(bad.sum())} of {bad.size} cells differ\n" + "\n".join(lines))


def _assert_spans(out, hard, counts, what):
    got_hard = (out["flags"] & 2) != 0
    assert np.array_equal(got_hard, hard), (what, np.nonzero(got_hard != hard)[0][:10])
    got = np.stack([out["n_in"], out["n_oow"], out["n_tiny"]], 1).astype(np.int64)
    bad = np.nonzero((got != counts).any(1))[0]
    assert len(bad) == 0, (what, [(int(i), got[i].tolist(), counts[i].tolist()) for i in bad[:8]])


# ---- texts of bare sample lists -------------------------------------------------------------------------------
class _Text:
    """bare sample lists ('[' + samples + ']'); every list is one span feeding one row"""

    def __init__(self):
        self.buf = bytearray()
        self.spans = []       # (begin, end, row)
        self.samples = []     # (row, [(ts_text, value_text)])

    def pad_to(self, pos, byte=b" "):
        assert pos >= len(self.buf), (pos, len(self.buf))
        self.buf += byte * (pos - len(self.buf))

    def span(self, row, samples):
        self.buf += b"["
        begin = len(self.buf)
        self.buf += b",".join(b'[%s,"%s"]' % (t.encode(), v.encode()) for t, v in samples)
        self.spans.append((begin, len(self.buf), row))
        self.samples.append((row, list(samples)))
        self.buf += b"]\n"
        return begin

    def span_array(self):
        import gpu_pruner_b200 as g
        sp = np.zeros(len(self.spans), g.IdleEngine.SPAN_DTYPE)
        for i, (b, e, r) in enumerate(self.spans):
            sp[i]["begin"], sp[i]["end"], sp[i]["row"] = b, e, r
        return sp


def _read_plane(eng, n_rows, T, plane=0):
    out = np.empty((n_rows, T), np.uint32)
    eng.memcpy(out, eng.text_planes()[plane], out.nbytes, 0, 1)
    return out


def _parse(eng, text, grid, n_rows, T, slot=0, plane=0, thr=0.0):
    """scan `text` into `slot`, parse all its spans into a filled context plane; -> (spans out, plane bits)"""
    t_end, window, step, _ = grid
    eng.text_scan(bytes(text.buf), slot=slot)
    out = eng.text_parse(text.span_array(), t_end, step, T, n_rows, slot=slot, plane=plane, window_seconds=window,
                         power_threshold=thr)
    return out, _read_plane(eng, n_rows, T, plane)


# ---- 1. every number form, bit for bit ------------------------------------------------------------------------
def _gen_table():
    spec = importlib.util.spec_from_file_location("gen_pow10_table", os.path.join(ROOT, "tools", "gen_pow10_table.py"))
    gen = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(gen)
    return gen


def _el_needs_second_product(m, e10, gen):
    """True when Eisel-Lemire's first product m * hi(10^e10) lacks a carry that only the second product (with the
    low 64 bits of the table entry) supplies: the value the device converts wrongly without that refinement"""
    if m == 0 or m >= 1 << 64 or not (gen.QMIN <= e10 <= gen.QMAX):
        return False
    p = gen.mantissa128(e10)
    man = m << (64 - m.bit_length())
    x = man * (p >> 64)
    x_hi, x_lo = x >> 64, x & M64
    if (x_hi & 0x1FF) != 0x1FF or x_lo + man <= M64:
        return False
    return x_lo + ((man * (p & M64)) >> 64) > M64


def _mantissa_exp(text):
    """(integer of the significant digits, exp10) of a plain decimal spelling, trailing zeros stripped as the
    parser strips them above 2^53"""
    s = text.lstrip("+-")
    mant, _, ex = s.replace("E", "e").partition("e")
    ip, _, fp = mant.partition(".")
    m, e10 = int(ip + fp), (int(ex) if ex else 0) - len(fp)
    while m > 1 << 53 and m % 10 == 0:
        m, e10 = m // 10, e10 + 1
    return m, e10


def _spell(d):
    sign, digits, exp = d.as_tuple()
    return ("-" if sign else "") + "".join(map(str, digits)) + "e" + str(exp)


def binary64_midpoint_decimals(rng, n):
    """19-significant-digit decimals just below and just above the midpoint between two adjacent normal doubles
    (and one unit of the 19th digit further out): where Eisel-Lemire's truncated product needs its carry checks"""
    D = decimal.Decimal
    wide = decimal.Context(prec=1200)
    out = []
    while len(out) < 4 * n:
        x = math.ldexp(1.0 + rng.getrandbits(52) / 2.0 ** 52, rng.randrange(-1000, 1000))
        y = math.nextafter(x, math.inf)
        if math.isinf(y):
            continue
        mid = wide.divide(wide.add(D(x), D(y)), 2)
        for rounding, step in ((decimal.ROUND_FLOOR, -1), (decimal.ROUND_CEILING, 1)):
            q = decimal.Context(prec=19, rounding=rounding).plus(mid)
            m, e = _mantissa_exp(_spell(q))
            out += [f"{m}e{e}", f"{m + step}e{e}"]
    return out


def f32_midpoint_decimals(rng, n):
    """the shortest spellings of doubles that are an f32 midpoint, and of their double neighbours: strtod then
    (float) rounds twice, and only a conversion through the exact double gets all three right"""
    out = []
    for i in range(n):
        b = rng.randrange(1, 0x7F7FFFFF) if i % 8 else rng.randrange(1, 0x00800000)     # some in the f32 denormals
        f = np.uint32(b).view(np.float32)
        mid = (float(f) + float(np.nextafter(f, np.float32(np.inf)))) / 2
        sign = -1.0 if i % 3 == 0 else 1.0
        out += [E.go_float(sign * d) for d in (mid, math.nextafter(mid, -math.inf), math.nextafter(mid, math.inf))]
    return out


EDGE_SPELLINGS = [
    # Clinger's boundaries: m = 2^53 and 2^53 + 1 against the exact powers 10^22 and the first inexact one
    *[f"{m}e{e}" for m in (2 ** 53 - 1, 2 ** 53, 2 ** 53 + 1) for e in (22, -22, 23, -23, 0, 1, -1)],
    # trailing zeros stripped above 2^53, and what is left after the strip
    "13098385200945040.0", "9007199254740993000e-3", "9007199254740994000e-3", "130983852009450400e-1",
    "18014398509481984000e-4", "9007199254740992000", "900719925474099300000e-5",
    # zeros past the 19th significant digit, leading zeros, exponent spellings, signs
    "5.0000000000000000000000", "1.2345678901234567890000", "1.2345678901234567891", "0.0000000000000000000000000123",
    "0000000000000000000000012.5", "000.000", "1E5", "1e+5", "1e-0", "1E-05", "2e+000", "1e0001", "7e-000", "+1.5",
    "-1.5", "+0", "-0", "-0.0", "+0e5", "-0e-5", "-0.000e+12", "+.5", "-5.", "1e", "--1",
    # the integer fast path and its edge
    "16777216", "16777217", "16777215", "16777218", "-16777217", "16777217.0", "16777217e0", "33554431", "33554433",
    "4294967297", "18446744073709551615", "9999999999999999999",
    # the f32 range's ends
    "1e-45", "1.4e-45", "7e-46", "7.1e-46", "-7e-46", "1e-46", "1.1754942e-38", "1.17549435e-38", "3.4028235e38",
    "3.4028235677973366e38", "3.4028236e38", "-1e39", "1e308", "1.7976931348623157e308", "1.8e308", "2.2250738585072014e-308",
    "4.9e-324", "Inf", "+Inf", "-Inf", "NaN",
]


def number_corpus():
    """every spelling the CPU tests convert, Go's spellings of random doubles across the whole range, the edge
    lists of edges.py, and the exact-decimal edge cases above"""
    rng = random.Random(20261016)
    cases, _ = NC.eisel_lemire_cases()
    texts = [f"{m}e{e}" for m, e in cases] + NC.value_texts()
    for _ in range(20_000):
        x = struct.unpack("<d", struct.pack("<Q", rng.getrandbits(64)))[0]
        if math.isfinite(x):
            texts.append(E.go_float(x))
    texts += [E.go_float(x) for x in E.ZEROISH + E.RATIOS + E.SPECIAL]
    texts += binary64_midpoint_decimals(rng, 1500) + f32_midpoint_decimals(rng, 1500) + EDGE_SPELLINGS
    return [t for t in texts if len(t) <= 60]     # a value starts 13 bytes into its sample: all within kMaxSample


def _number_layout(texts, declined, T=256):
    """one value per column (1 s step), T columns per span, one row per span; a declined value in a span of its own"""
    text = _Text()
    ts = [str(T_END - T + 1 + j) for j in range(T)]
    cur = []
    for t in texts:
        if t in declined:
            text.span(len(text.spans), [(ts[0], t)])
            continue
        cur.append(t)
        if len(cur) == T:
            text.span(len(text.spans), list(zip(ts, cur)))
            cur = []
    if cur:
        text.span(len(text.spans), list(zip(ts, cur)))
    return text


def test_every_number_form_bit_for_bit(eng, driver):
    texts = number_corpus()
    declined = _host_declines(driver, texts)
    T = 256
    text = _number_layout(texts, declined, T)
    grid = (T_END, T, 1, T - 1)
    n_rows = len(text.spans)
    want, hard, counts = _reference(text.samples, grid, n_rows, T, declined=declined)
    assert hard.sum() == sum(t in declined for t in texts)
    out, got = _parse(eng, text, grid, n_rows, T)
    cell_text = {(r, j): v for r, samples in text.samples for j, (_, v) in enumerate(samples)}
    _assert_spans(out, hard, counts, "number spans")
    _assert_cells(got, want, "number forms", lambda r, c: repr(cell_text.get((int(r), int(c)))))
    print(f"\n[numbers] {len(texts)} values ({len(declined & set(texts))} distinct declined, {int(hard.sum())} hard "
          f"spans), {n_rows} spans, {got.size} cells compared, {int(counts[:, 2].sum())} clamped to denorm_min")


# ---- 2. the device's float64, pinned through the power snap ---------------------------------------------------
def _through_snap(text):
    """the value takes the Clinger / Eisel-Lemire path, whose float64 the power snap compares with the threshold
    (not zero, not an integer below 2^24 without point or exponent)"""
    if text == "NaN" or text in SPECIAL_BITS:
        return False
    s = text.lstrip("+-")
    mant = s.replace("E", "e").partition("e")[0]
    m = int(mant.replace(".", ""))
    return m != 0 and ("e" in s.lower() or "." in mant or m >= 1 << 24)


def probe_corpus(driver):
    """values whose correctly rounded double is a normal one and which take the snapped path: binary64-midpoint
    decimals, Clinger's multiply and divide, Eisel-Lemire across the exponent range, 17-digit ratios"""
    rng = random.Random(54)
    mids = binary64_midpoint_decimals(rng, 300)
    clinger = []
    for _ in range(300):
        m = rng.randrange(10 ** rng.randrange(1, 16), 1 << 53)
        e = rng.randrange(-22, 23)
        clinger.append(f"{m}e{e}" if rng.random() < 0.5 else f"{m / 10 ** 6:.6f}e{e}")
    cases, _ = NC.eisel_lemire_cases()
    el = [f"{m}e{e}" for m, e in rng.sample(cases, 3000)]
    ratios = [repr(x) for x in E.RATIOS] + [repr(rng.random()) for _ in range(400)]
    texts = list(dict.fromkeys(mids + clinger + el + ratios))
    declined = _host_declines(driver, texts)
    return [t for t in texts if t not in declined and _through_snap(t)
            and 2.2250738585072014e-308 <= abs(float(t)) <= 1.7976931348623157e308][:3000]


def test_device_float64_is_the_correctly_rounded_double(eng, driver):
    """the power plane stores x snapped against thr by `x >= thr` in float64: a value whose double is d stores at
    least up(d) under thr = d and less than up(d+) under thr = d+ = nextafter(d, +inf) — exactly when the
    device's double is d.  One value per parse; the probe text sits in slot 2 (a few tiles)."""
    gen = _gen_table()
    texts = probe_corpus(driver)
    carries = sum(_el_needs_second_product(*_mantissa_exp(t), gen) for t in texts)
    assert len(texts) >= 2500 and carries >= 20, (len(texts), carries)
    text = _Text()
    for i, t in enumerate(texts):
        text.span(i, [(str(T_END), t)])
    eng.text_scan(bytes(text.buf), slot=2)
    spans = text.span_array()
    N = len(texts)
    stored = {}
    for name, thr_of in (("d", lambda d: d), ("next", lambda d: math.nextafter(d, math.inf))):
        for i, t in enumerate(texts):
            out = eng.text_parse(spans[i:i + 1], T_END, 1, 1, N, slot=2, plane=1, fill=(i == 0),
                                 power_threshold=thr_of(float(t)))
            assert out["n_in"][0] == 1 and not out["flags"][0] & 2, t
        stored[name] = _read_plane(eng, N, 1, 1)[:, 0].view(np.float32).astype(np.float64)
    bad = []
    for i, t in enumerate(texts):
        d = float(t)
        if not (stored["d"][i] >= E.f32_up(d) and stored["next"][i] < E.f32_up(math.nextafter(d, math.inf))):
            bad.append((t, d.hex(), stored["d"][i], stored["next"][i]))
    assert not bad, bad[:10]
    print(f"\n[float64 probe] {N} values pinned to their correctly rounded double ({carries} need Eisel-Lemire's "
          f"second product), {2 * N} parses")


SWEEP_THRESHOLDS = E.THRESHOLDS + [1e-40, -5.0, 1e-3, 123456.789, 3.4028235677973366e38, 1e39, 0.0, math.nan]


def test_power_snap_sweep_matches_the_host_build_and_float64(eng, driver):
    rng = random.Random(151)
    vals = []
    for thr in SWEEP_THRESHOLDS:
        if thr == 0 or math.isnan(thr):
            continue
        vals += E.power_edges(thr) + [thr * (1 + rng.uniform(-1e-7, 1e-7)) for _ in range(200)]
        vals += [-thr, thr / 2, thr * 2]
    texts = [E.go_float(v) for v in vals if math.isfinite(v)]
    corpus = [t for t in number_corpus() if t != "NaN" and t not in SPECIAL_BITS]
    texts += rng.sample(corpus, 3000)
    declined = _host_declines(driver, texts)
    texts = list(dict.fromkeys(t for t in texts if t not in declined and math.isfinite(float(t))))
    T = 256
    text = _number_layout(texts, set(), T)
    grid = (T_END, T, 1, T - 1)
    eng.text_scan(bytes(text.buf), slot=1)
    cells = [(r, j, v) for r, samples in text.samples for j, (_, v) in enumerate(samples)]
    flipped = 0
    for thr in SWEEP_THRESHOLDS:
        out = eng.text_parse(text.span_array(), T_END, 1, T, len(text.spans), slot=1, plane=1, power_threshold=thr)
        assert not np.any(out["flags"] & 2) and int(out["n_in"].sum()) == len(texts), thr
        got = _read_plane(eng, len(text.spans), T, 1)
        host = NC.run_number_check(driver, [f"S {thr!r} {v}" for _, _, v in cells])
        up = E.f32_up(thr) if thr == thr and thr != 0 else None
        for (r, j, v), line in zip(cells, host):
            bits = int(got[r, j])
            assert bits == int(line.split()[1], 16), (thr, v, f"{bits:08x}", line)
            x, s = float(v), _f32(bits)
            if up is None:
                assert bits == _want_bits(v), (thr, v)
            else:
                assert (s >= up) == (x >= thr), (thr, v, s)
                flipped += bits != _want_bits(v)
    assert flipped >= 10
    print(f"\n[power sweep] {len(texts)} values x {len(SWEEP_THRESHOLDS)} thresholds, {flipped} stored off the plain "
          f"rounding")


# ---- 3. bucketing and merging, cell by cell ------------------------------------------------------------------
VALUES = ["0", "-0", "+0", "0.0", "-0.0", "37", "100", "-5", "-2.5", "-3.4e38", "3.4e38", "1e39", "-1e39", "1e-40",
          "-1e-40", "1.4e-45", "1e-50", "-1e-50", "-7e-46", "+Inf", "-Inf", "NaN", "0.30000000000000004",
          "0.12345678901234568", "-0.9999999999999999", "16777217", "-16777217", "4294967296.5",
          "2.220446049250313e-16", "99.99999999999999", "-149.999999"]
NEGATIVE = ["-5", "-2.5", "-3.4e38", "-1e39", "-1e-40", "-1e-50", "-7e-46", "-0.9999999999999999", "-16777217",
            "-149.999999", "-Inf", "NaN", "-0"]


def _ts_text(ms, rng):
    s, f = divmod(ms, 1000)
    if f == 0:
        return rng.choice([f"{s}", f"{s}.0", f"{s}.000"])
    if f % 100 == 0:
        return rng.choice([f"{s}.{f // 100}", f"{s}.{f:03d}"])
    if f % 10 == 0:
        return rng.choice([f"{s}.{f // 10:02d}", f"{s}.{f:03d}"])
    return f"{s}.{f:03d}"


# name: (step s, window s, columns, t_end s)
GRIDS = {
    "step1": (1, 300, 300, T_END),
    "step2_window_not_a_multiple": (2, 301, 160, T_END),
    "step7": (7, 600, 90, T_END),
    "step15_t_lo_negative": (15, 900, 60, 500),
    "step60": (60, 3599, 64, T_END),
    "step3600_60_days": (3600, 60 * 86400, 1440, T_END),      # t_end - ts > 2^32 ms: the 64-bit division
    "abi_limits": (4_000_000, 4_000_000_000, 1000, 3_999_999_999),
}


def _bucket_samples(rng, step, window, T, t_end_s, n_rows):
    """[(row, [(ts_text, value_text)])]: borders, window ends, fractions, far-future stamps, declined stamps, and
    cells that receive many samples in shuffled order"""
    t_end, step_ms = t_end_s * 1000, step * 1000
    t_lo = t_end - window * 1000
    stamps = [t_lo, t_lo + 1, t_lo - 1, t_end, t_end - 1, t_end + 1, t_end + 1000, 0, 1]
    for k in range(-(-window // step) + 1):
        stamps += [t_end - k * step_ms + d for d in (-1, 0, 1)]
    for _ in range(40):
        s = rng.randrange(max(0, t_lo // 1000), t_end_s + 1)
        stamps += [s * 1000 + f for f in (1, 500, 999)]
    stamps += [rng.randrange(max(0, t_lo - step_ms), t_end + step_ms) for _ in range(3 * T)]
    plain = [(_ts_text(ms, rng), rng.choice(VALUES)) for ms in stamps if ms >= 0]
    plain += [(t, rng.choice(VALUES)) for t in ("4000000000000", "4000000000000.5", "9999999999999")]
    rows = [[] for _ in range(n_rows)]
    for smp in plain:
        rows[rng.randrange(n_rows)].append(smp)
    for r in rows:
        rng.shuffle(r)
    # many samples per cell: rows of their own, the cell's samples contiguous (every lane of a warp on one cell) in
    # odd rows, spread through the row in even ones; some cells see negative values only
    n_buckets = min(T, -(-window // step), t_end // step_ms + 1)      # buckets that hold stamps >= 0
    for c in range(8):
        k = rng.randrange(n_buckets)
        hi = t_end - k * step_ms
        lo = max(hi - step_ms, t_lo, -1)
        pool = NEGATIVE if c % 3 == 0 else VALUES
        cell = [(_ts_text(rng.randrange(lo + 1, hi + 1), rng), rng.choice(pool)) for _ in range(48)]
        extra = [(_ts_text(rng.randrange(max(0, t_lo + 1), t_end + 1), rng), rng.choice(VALUES)) for _ in range(40)]
        if c % 2:
            rows.append(extra[:20] + cell + extra[20:])
        else:
            mixed = cell + extra
            rng.shuffle(mixed)
            rows.append(mixed)
    spans = [(r, s) for r, s in enumerate(rows)]
    # stamps finer than a millisecond or longer than 13 digits: the span goes hard (rows of their own)
    for t in ("1700000000.1234", "17000000001234"):
        spans.append((len(spans), [(t, "1")]))
    spans.append((len(spans), []))      # an empty list
    return spans


@pytest.mark.parametrize("name", list(GRIDS))
def test_bucketing_and_merge_cell_by_cell(eng, name):
    step, window, T, t_end = GRIDS[name]
    rng = random.Random(name)
    spans = _bucket_samples(rng, step, window, T, t_end, 12)
    text = _Text()
    for row, samples in spans:
        text.span(row, samples)
    grid = (t_end, window, step, T - 1)
    n_rows = len(spans)
    want, hard, counts = _reference(text.samples, grid, n_rows, T)
    assert hard.sum() == 2 and counts[:, 1].sum() > 0 and counts[:, 2].sum() > 0
    out, got = _parse(eng, text, grid, n_rows, T)
    _assert_spans(out, hard, counts, name)
    _assert_cells(got, want, name)
    print(f"\n[bucketing {name}] {sum(len(s) for _, s in spans)} samples, {n_rows} spans, {got.size} cells, "
          f"{int(counts[:, 1].sum())} out of the window")


def test_resident_ring_merges_at_every_head_position(eng):
    """GPR_TEXT_RESIDENT on a ring of 37 buckets of 7 s: open buckets with gpr_resident_advance until the head has
    stood at every position, parse a slice each time and compare the raw ring with a model ring; buckets outside
    the slice keep what they had"""
    P, G, T, step = 5, 2, 37, 7
    rows = P * G
    rng = random.Random(37)
    eng.resident_init(P, G, T)
    eng.resident_advance(T)
    ring, head, t_end, seen, tick = np.full((rows, T), FILL, np.uint32), 0, T_END, set(), 0
    plan = [T + 3, T, 1]
    while len(seen) < T or tick < 45:
        n_new = plan[tick] if tick < len(plan) else rng.choice([1, 1, 2, 3, 4, 6])
        eng.resident_advance(n_new)
        for j in range(min(n_new, T)):
            ring[:, (head + j) % T] = FILL
        head = (head + n_new) % T
        seen.add(head)
        t_end += n_new * step
        window = min(T * step, n_new * step + rng.choice([0, 0, 5, 3 * step]))
        t_end_ms, t_lo_ms = t_end * 1000, (t_end - window) * 1000
        spans = []
        for r in range(rows):
            if rng.random() < 0.15:
                continue                                    # a series without samples in this slice
            stamps = [rng.randrange(t_lo_ms - 3000, t_end_ms + 2000) for _ in range(rng.randrange(1, 12))]
            b = rng.randrange(-(-window // step))                # several samples in one bucket
            stamps += [t_end_ms - b * step * 1000 - rng.randrange(step * 1000) for _ in range(rng.randrange(6))]
            stamps += [t_lo_ms, t_lo_ms + 1, t_end_ms, t_end_ms + 1]
            spans.append((r, [(_ts_text(ms, rng), rng.choice(VALUES)) for ms in stamps]))
        text = _Text()
        for r, s in spans:
            text.span(r, s)
        grid = (t_end, window, step, (head + T - 1) % T)
        ring, hard, counts = _reference(text.samples, grid, rows, T, plane=ring)
        eng.text_scan(bytes(text.buf), slot=0)
        out = eng.text_parse(text.span_array(), t_end, step, T, rows, resident=True, window_seconds=window)
        got = np.empty((rows, T), np.uint32)
        eng.memcpy(got, eng.resident_planes()[0], got.nbytes, 0, 1)
        assert eng.resident_head() == head
        _assert_spans(out, hard, counts, f"tick {tick}")
        _assert_cells(got, ring, f"tick {tick} (head {head}, {n_new} new, window {window} s)")
        tick += 1
        assert tick < 400
    assert seen == set(range(T))
    print(f"\n[resident] {tick} ticks, head at all {T} positions, {tick * got.size} ring cells compared")


# ---- 4. chunk and tile boundaries -----------------------------------------------------------------------------
OPEN, CLOSE = b'},"values":[', b'"]]'
SERIES = b'{"metric":{"__name__":"DCGM_FI_DEV_GPU_UTIL","UUID":"GPU-7"},"values":[[1700000000,"1"],[1700000001,"0"]]},'


def _boundary_text(n, chunk, gap, placements=()):
    """n bytes of series every `gap` bytes (at most one marker pair per 128 bytes: a 2 MB chunk stays within its
    16,384-marker room), the 64 bytes either side of every chunk boundary cleared, then `placements`
    (offset, pattern) written"""
    period = SERIES + b" " * (gap - len(SERIES))
    buf = np.frombuffer(period * (n // gap + 1), np.uint8)[:n].copy()
    for b in range(chunk, n, chunk):
        buf[b - 64:b + 64] = ord(" ")
    for off, pat in placements:
        buf[off:off + len(pat)] = np.frombuffer(pat, np.uint8)
    return buf


def _markers(buf):
    t = buf.tobytes()
    return (np.array([m.start() for m in re.finditer(re.escape(OPEN), t)], np.uint64),
            np.array([m.start() for m in re.finditer(re.escape(CLOSE), t)], np.uint64))


AROUND = [(pat, d) for pat in (OPEN, CLOSE) for d in range(-16, 2)]   # every offset from -16 to +1


def _check_scan(e, decoy, target, host, what, slot=0, n=None, mem_kind=0, chunks=False):
    """scan a decoy of the same length first (all blanks: bytes a chunk's scan reads beyond its overlap, before the
    next chunk has landed, are then wrong ones, so a short overlap fails every time), then the target; its markers
    must be the offsets the regex finds in `host`, also chunk by chunk"""
    e.text_scan(decoy(), slot=slot, n_bytes=n, mem_kind=mem_kind)
    o, c = e.text_scan(target(), slot=slot, n_bytes=n, mem_kind=mem_kind)
    eo, ec = _markers(host)
    assert np.array_equal(o, eo), (what, np.setxor1d(o, eo)[:10])
    assert np.array_equal(c, ec), (what, np.setxor1d(c, ec)[:10])
    if chunks:
        e.text_scan(decoy(), slot=slot, n_bytes=n, mem_kind=mem_kind)
        parts = list(e.text_scan_chunks(target(), slot=slot, n_bytes=n, mem_kind=mem_kind))
        assert np.array_equal(np.concatenate([p[0] for p in parts]), eo), what
        assert np.array_equal(np.concatenate([p[1] for p in parts]), ec), what
    return len(eo) + len(ec)


@pytest.mark.parametrize("threads", ["8", "1"])
def test_scan_markers_at_every_offset_around_pageable_chunks(threads):
    """pageable text staged through the pinned ring in 1 MB chunks (GPR_TEXT_CHUNK_MB=1), by 8 producer threads
    and by one (chunks copied in order on one stream); one boundary per (marker, offset)"""
    chunk = 1 << 20
    n = (len(AROUND) + 2) * chunk + 777
    buf = _boundary_text(n, chunk, 320, [((k + 1) * chunk + d, pat) for k, (pat, d) in enumerate(AROUND)])
    target, blanks = buf.tobytes(), b" " * n
    e = _engine(GPR_TEXT_CHUNK_MB="1", GPR_TEXT_UPLOAD_THREADS=threads)
    try:
        k = _check_scan(e, lambda: blanks, lambda: target, buf, f"pageable, {threads} thread(s)", chunks=True)
    finally:
        e.close()
    print(f"\n[scan pageable x{threads}] {n} bytes, {n // chunk} boundaries, {k} markers")


@pytest.mark.parametrize("source", ["pinned", "device"])
def test_scan_markers_at_every_offset_around_16mb_chunks(eng, source):
    """pinned host text and device-memory text go up in 16 MB chunks: 35 MB texts, a `},"values":[` at offset d
    around the first boundary and a `"]]` at offset d around the second, for every d in [-16, +1]"""
    import gpu_pruner_b200 as g
    chunk = 16 << 20
    n = 35 * (1 << 20) + 333
    base = _boundary_text(n, chunk, 2048)
    blanks = np.full(n, ord(" "), np.uint8)
    pinned = eng.host_array((n,), np.uint8)
    dev = eng.device_alloc(n) if source == "device" else None
    kind = g.ffi.GPR_MEM_DEVICE if dev is not None else g.ffi.GPR_MEM_HOST

    def put(arr):
        pinned[:] = arr
        if dev is None:
            return pinned
        eng.memcpy(dev, pinned, n, 1, 0)
        return dev

    try:
        total = 0
        for d in range(-16, 2):
            buf = base.copy()
            for off, pat in ((chunk + d, OPEN), (2 * chunk + d, CLOSE)):
                buf[off:off + len(pat)] = np.frombuffer(pat, np.uint8)
            total += _check_scan(eng, lambda: put(blanks), lambda: put(buf), buf, f"{source} d={d}", slot=1, n=n,
                                 mem_kind=kind, chunks=d in (-16, -3, -1, 1))
    finally:
        if dev is not None:
            eng.device_free(dev)
    print(f"\n[scan {source}] 18 texts of {n} bytes, {total} markers")


def _long_value(rng, mlen, exp):
    """a decimal with 19 significant digits whose mantissa (sign, digits, point) is exactly `mlen` bytes: the
    digits after the 19th are zeros behind the point"""
    sig = str(rng.randrange(10 ** 18, 10 ** 19))
    form = rng.randrange(3)
    if form == 0:
        body = sig[0] + "." + sig[1:]
    elif form == 1:
        body = "-" + "0" * rng.randrange(1, 20) + sig[:3] + "." + sig[3:]
    else:
        body = "0." + "0" * rng.randrange(0, 12) + sig
    return body + "0" * (mlen - len(body)) + exp


def tile_text(T):
    """the text of the test below: (text, declined values)"""
    rng = random.Random(4096)
    ts = [f"{T_END - T + j}.{(j * 389 + 123) % 999 + 1:03d}" for j in range(T)]    # column j: bucket (t - 1, t]
    exps = ["", "e-5", "E+12", "e7", "e-123", "e+000", "E-38"]

    def longest():
        return _long_value(rng, 60, rng.choice(exps))

    text = _Text()
    declined = set()
    k = 1
    for delta in range(0, 85):
        for kind in ("list", "alone", "too_long"):
            if kind == "too_long":
                v = _long_value(rng, 61, rng.choice(exps))
                declined.add(v)
                pre, target, post = [], v, []
            elif kind == "alone":
                pre, target, post = [], longest(), []
            else:
                pre, target, post = [longest() for _ in range(3)], longest(), [longest() for _ in range(3)]
            vals = pre + [target] + post
            samples = [(ts[j], v) for j, v in enumerate(vals)]
            head = sum(len(b'[%s,"%s"],' % (t.encode(), v.encode())) for t, v in samples[:len(pre)])
            while 4096 * k - delta - head - 1 < len(text.buf) + 1:
                k += 1
            text.pad_to(4096 * k - delta - head - 1)
            b = text.span(len(text.spans), samples)
            assert b + head == 4096 * k - delta
            k += 1
    # lists across several tiles
    for _ in range(2):
        text.span(len(text.spans), [(ts[j], longest()) for j in range(150)])
    # tiles with more than 512 '[' outside every list, real samples before and after them in the same tile
    short = ["0", "-5", "1e-50", "NaN", "-0", "37.5", "+Inf", "-1e-40", "16777217", "0.30000000000000004"]
    for n_brackets in (513, 600, 1023, 1500, 3000):
        text.pad_to((len(text.buf) // 4096 + 1) * 4096 + 7)
        text.span(len(text.spans), [(ts[j], rng.choice(short)) for j in range(4)])
        text.buf += b"[" * n_brackets
        room = 4096 - (len(text.buf) % 4096)
        n = max(2, min(T, room // 24 + 4))
        text.span(len(text.spans), [(ts[j], rng.choice(short)) for j in range(n)])
    return text, declined


def test_samples_at_every_offset_before_a_tile_boundary(eng):
    """a sample's '[' at every offset in [4096 k - 84, 4096 k] with the longest accepted samples (3-digit
    millisecond fraction, a 60-byte mantissa and an exponent: 84 bytes from '[') inside lists, alone, and one
    byte too long (hard); lists across several tiles; and tiles with more than kListCap (512) '[' bytes outside
    every list, whose samples are listed in the kernel's later passes"""
    T = 256
    text, declined = tile_text(T)
    grid = (T_END, T, 1, T - 1)
    n_rows = len(text.spans)
    want, hard, counts = _reference(text.samples, grid, n_rows, T, declined=declined)
    assert hard.sum() == 85
    out, got = _parse(eng, text, grid, n_rows, T)
    _assert_spans(out, hard, counts, "tile boundaries")
    _assert_cells(got, want, "tile boundaries", lambda r, c: repr(text.samples[int(r)][1][int(c)][1])
                  if int(c) < len(text.samples[int(r)][1]) else "-")
    print(f"\n[tiles] {sum(len(s) for _, s in text.samples)} samples, {n_rows} spans, {got.size} cells, "
          f"{len(text.buf)} bytes")
