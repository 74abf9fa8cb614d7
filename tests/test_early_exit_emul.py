"""Early exit in the reduce kernels, checked byte for byte on the CPU.

A row may stop being read at the first read sample that settles its flag (util: a sample > 0; power: a sample >=
thr), unless the call asks for series_max.  k_reduce_tma and k_reduce_ldg are compiled from the source text of
gpu-pruner_b200/csrc/gpr_kernels.cuh as in test_hotpath_emul.py, with every load and bulk copy renamed to a counting
version (tests/cpp/early_exit_emul.cpp) that charges its bytes to the row it reads.  For each window the test
requires the decision, candidate and veto bits, the counts and series_max to equal the numpy oracle, and the bytes of
every row to equal a numpy model of the rule:
  * tma: copies [0, h), then chunk_elems at a time, each requested after the previous one was examined;
  * ldg: the peel to 16-byte alignment plus one float4 per lane, then batches of kLdgUnroll float4 per lane, the
    scalar tail last; the warp leaves after any of these once a lane has seen a settling sample;
  * with series_max, 4 * T bytes per row."""
import os
import subprocess

import numpy as np
import pytest

import kat as KAT
from test_hotpath_emul import ROOT, _extract, _thr_bits

LDG_UNROLL = 8          # gpr_launch.h kLdgUnroll
HEAD = 128              # gpr_launch.h kTmaHeadElems
RENAMES = [("ldg_stream(", "cnt_ldg_stream("), ("__ldg(", "cnt_ldg("), ("tma_load_1d(", "cnt_tma_load_1d(")]
THR = 150.0


def _source():
    body = _extract()
    for old, new in RENAMES:
        assert old in body, old
        body = body.replace(old, new)
    return body


def _build(d, sanitize=None):
    (d / "early_exit_extract.inc").write_text(_source())
    exe = d / ("early_exit_emul_tsan" if sanitize else "early_exit_emul")
    cmd = ["g++", "-std=c++20", "-O1", "-pthread", "-Wall", "-Wno-unknown-pragmas", "-Wno-unused-function"]
    if sanitize:
        cmd += ["-g", "-fsanitize=" + sanitize]
    subprocess.run(cmd + ["-I", str(d), os.path.join(ROOT, "tests", "cpp", "early_exit_emul.cpp"), "-o", str(exe)],
                   check=True, capture_output=True, text=True)
    return str(exe)


@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    return _build(tmp_path_factory.mktemp("early_exit"))


# (sm_count, tma_warps, tma_chunk_bytes, tma_depth, ldg_ctas)
LAYOUTS = {
    "one rest chunk": (2, 4, 8192, 3, 1),     # T 1800: head 128, the rest in one copy (the C2 layout)
    "four chunks": (3, 8, 2048, 2, 1),        # T 1800: head 128, then 452-sample chunks
    "head = chunk": (1, 4, 512, 2, 2),        # T 1800: 120-sample chunks, the head is one of them
    "depth 1": (2, 16, 2048, 1, 1),           # T 1000: head 128, chunks of 500
}


def _tma_layout(knobs, T):
    chunk = knobs[2]
    n = -(-4 * T // chunk)
    ce = -(-T // n)
    ce = (ce + 3) // 4 * 4
    return min(HEAD, ce), ce


def _settling(x, power):
    with np.errstate(invalid="ignore"):
        return (x >= np.float32(THR)) if power else (x > 0)


def _first(x, power):
    """index of the first settling sample of every row, T where none"""
    s = _settling(x, power)
    T = x.shape[-1]
    return np.where(s.any(-1), s.argmax(-1), T)


def model_tma(first, T, h, ce, smax):
    ends = [min(h, T)]
    while ends[-1] < T:
        ends.append(min(ends[-1] + ce, T))
    ends = np.array(ends)
    if smax:
        return np.full(first.shape, 4 * T, np.int64)
    idx = np.searchsorted(ends, first, side="right")       # copy that holds the first settling sample
    return 4 * np.where(first < T, ends[np.minimum(idx, len(ends) - 1)], T).astype(np.int64)


def model_ldg(first, T, offsets, smax):
    """offsets: each row's start in elements from a 16-byte boundary"""
    out = np.empty(first.shape, np.int64)
    for r, (f, off) in enumerate(zip(first.ravel(), offsets.ravel())):
        peel = min((4 - off % 4) % 4, T)
        nv = (T - peel) // 4
        # the points where the warp tests: after the head, after every batch; the scalar tail comes last
        stops = [peel + 4 * min(32, nv)]
        i = 32
        while i < nv:
            i = min(i + 32 * LDG_UNROLL, nv)
            stops.append(peel + 4 * i)
        n = T
        if not smax:
            n = next((s for s in stops if f < s), T)
        out.flat[r] = 4 * n
    return out


def _write(d, util, power, smax, shift, knobs, variant, ld=None):
    P, G, T = util.shape
    ld = ld or T
    os.makedirs(d, exist_ok=True)

    def strided(x, fill):
        out = np.full((P * G, ld), fill, np.float32)
        out[:, :T] = x.reshape(P * G, T)
        return out
    strided(util, 77.0).tofile(os.path.join(d, "util.f32"))
    if power is not None:
        strided(power, 1e9).tofile(os.path.join(d, "power.f32"))
    with open(os.path.join(d, "params.txt"), "w") as f:
        f.write(f"{P} {G} {T} {ld} {int(power is not None)} {_thr_bits(THR)} {int(smax)} {shift} "
                f"{' '.join(str(k) for k in knobs)} {variant}\n")


def _run(emul, dirs, env=None):
    r = subprocess.run([emul] + [str(d) for d in dirs], capture_output=True, text=True, timeout=1800, env=env)
    assert r.returncode == 0 and "ThreadSanitizer" not in r.stderr, r.stderr[-2000:]
    out = {}
    words = lambda h: np.array([int(h[i:i + 8], 16) for i in range(0, len(h), 8)], np.uint32) if h != "-" else np.zeros(0, np.uint32)
    for l in r.stdout.splitlines():
        f = l.split()
        out[f[0]] = {"kernel": f[1], "d": words(f[2]), "c": words(f[3]), "v": words(f[4]),
                     "counts": tuple(int(x) for x in f[5:8]), "smax": words(f[8]).view(np.float32),
                     "head": int(f[9].split("=")[1]), "chunk": int(f[10].split("=")[1])}
        n = np.fromfile(os.path.join(f[0], "bytes.u64"), np.uint64).astype(np.int64)
        out[f[0]]["bytes"] = n.reshape(2, -1)
    return out


def _positions(T, layouts):
    """the first settling sample at every boundary of every layout and of the LDG batches"""
    pos = {0, T - 1}
    for knobs in layouts:
        h, ce = _tma_layout(knobs, T)
        pos |= {h - 1, h, h + 1}
        e = h
        while e < T:
            pos |= {e, min(e + ce, T) - 1}
            e += ce
    for peel in (0, 3):           # aligned rows, and rows 4 bytes off alignment
        e = peel + 128
        pos |= {e - 1, e, e + 1}
        while e < T:
            e += 4 * 32 * LDG_UNROLL
            pos |= {min(e, T) - 1, min(e, T)}
    return sorted(p for p in pos if 0 <= p < T)


def _boundary_window(T, layouts, power):
    pos = _positions(T, layouts)
    rows = []
    for p in pos:
        r = np.full(T, 100.0 if power else 0.0, np.float32)
        r[p] = THR if power else 1.0
        rows.append(r)
    rows.append(np.full(T, 100.0 if power else 0.0, np.float32))            # nothing settles it: read to the end
    while len(rows) % 4:
        rows.append(np.full(T, 100.0 if power else 0.0, np.float32))
    return np.stack(rows).reshape(-1, 4, T)


def _edge_window(T, h):
    """util: the values that settle nothing before a zero, and the ones that do, at awkward places"""
    nan = np.float32(np.nan)
    rows = []
    r = np.zeros(T, np.float32); r[:h] = -1.0; r[1:h:3] = nan; rows.append(r)                 # negatives, NaN, zero
    r = np.zeros(T, np.float32); r[:h] = nan; rows.append(r)                                   # all-NaN head, zeros behind
    rows.append(np.full(T, nan, np.float32))                                                   # no sample at all
    rows.append(np.full(T, -0.0, np.float32))                                                  # -0.0 is idle
    r = np.full(T, -0.0, np.float32); r[T - 2] = np.float32(1e-45); rows.append(r)            # denormal, last chunk
    r = np.full(T, nan, np.float32); r[h + 1] = np.inf; rows.append(r)                        # +Inf
    r = np.full(T, -5.0, np.float32); rows.append(r)                                           # busy? no: max -5
    r = np.zeros(T, np.float32); r[0] = np.float32(1e-45); rows.append(r)                     # denormal first
    return np.stack(rows).reshape(-1, 4, T)


def _edge_power(T, h):
    below = np.nextafter(np.float32(THR), np.float32(0))
    nan = np.float32(np.nan)
    rows = []
    r = np.full(T, below, np.float32); rows.append(r)                                          # one ulp below: never
    r = np.full(T, below, np.float32); r[T - 1] = THR; rows.append(r)                         # exactly thr, last
    r = np.full(T, nan, np.float32); r[h] = THR; rows.append(r)
    r = np.full(T, nan, np.float32); rows.append(r)
    r = np.full(T, -np.inf, np.float32); r[3] = np.inf; rows.append(r)
    r = np.full(T, 0.0, np.float32); r[h - 1] = 1e30; rows.append(r)
    r = np.full(T, 149.0, np.float32); rows.append(r)
    r = np.full(T, 149.0, np.float32); r[T // 2] = 151.0; rows.append(r)
    return np.stack(rows).reshape(-1, 4, T)


def _check(res, util, power, smax, oracle_np, variant, knobs, shift, ld):
    P, G, T = util.shape
    want = oracle_np.decide(util, power, None, None, 0, THR if power is not None else 0.0)
    tag = (variant, knobs, shift, smax, T)
    assert np.array_equal(res["d"], want["decision_bits"]), tag
    assert np.array_equal(res["c"], want["candidate_bits"]), tag
    assert np.array_equal(res["v"], want["veto_bits"]), tag
    assert res["counts"] == (want["n_series"], want["n_candidates"], want["n_decisions"]), tag
    if smax:
        assert KAT.smax_equal(res["smax"].reshape(P, G), want["series_max"]), tag
    planes = [(util, False)] + ([(power, True)] if power is not None else [])
    for k, (x, is_power) in enumerate(planes):
        first = _first(x.reshape(P * G, T), is_power)
        if res["kernel"] == "tma":
            h, ce = _tma_layout(knobs, T)
            assert (res["head"], res["chunk"]) == (h, ce), tag
            model = model_tma(first, T, h, ce, smax)
        else:
            offsets = (shift + np.arange(P * G, dtype=np.int64) * ld) % 4
            model = model_ldg(first, T, offsets, smax)
        got = res["bytes"][k]
        bad = np.nonzero(got != model)[0]
        assert bad.size == 0, (tag, "power" if is_power else "util", bad[:5], got[bad[:5]], model[bad[:5]], first[bad[:5]])


RUNS = [("tma", 0), ("ldg", 0), ("ldg", 1)]


@pytest.mark.parametrize("layout", sorted(LAYOUTS))
def test_settling_sample_at_every_boundary(emul, tmp_path, oracle_np, layout):
    knobs = LAYOUTS[layout]
    T = 1000 if layout == "depth 1" else 1800
    cases = []
    for power_plane in (False, True):
        util = _boundary_window(T, LAYOUTS.values(), False)
        power = _boundary_window(T, LAYOUTS.values(), True) if power_plane else None
        for variant, shift in RUNS:
            for smax in (False, True):
                d = tmp_path / f"{variant}{shift}_{int(power_plane)}_{int(smax)}"
                _write(str(d), util, power, smax, shift, knobs, variant)
                cases.append((d, util, power, smax, variant, shift))
    res = _run(emul, [c[0] for c in cases])
    kernels = set()
    for d, util, power, smax, variant, shift in cases:
        r = res[str(d)]
        kernels.add(r["kernel"])
        _check(r, util, power, smax, oracle_np, variant, knobs, shift, T)
        if smax:
            assert r["bytes"][0].sum() == 4 * util.size, d
    assert kernels == {"tma", "ldg", "ldg+1"}


def test_edge_values(emul, tmp_path, oracle_np):
    cases = []
    for layout, knobs in sorted(LAYOUTS.items()):
        T = 1000 if layout == "depth 1" else 1800
        h, _ = _tma_layout(knobs, T)
        util, power = _edge_window(T, h), _edge_power(T, h)
        for variant, shift in RUNS:
            for smax in (False, True):
                d = tmp_path / f"{layout.replace(' ', '_')}_{variant}{shift}_{int(smax)}"
                _write(str(d), util, power, smax, shift, knobs, variant)
                cases.append((d, util, power, smax, variant, shift, knobs, T))
    res = _run(emul, [c[0] for c in cases])
    for d, util, power, smax, variant, shift, knobs, T in cases:
        _check(res[str(d)], util, power, smax, oracle_np, variant, knobs, shift, T)


def test_strided_rows_and_short_windows(emul, tmp_path, oracle_np):
    """rows further apart than T (every LDG row at its own alignment with ld % 4 != 0), and windows no longer than
    one head"""
    rng = np.random.default_rng(7)
    cases = []
    for T, ld, knobs in ((1800, 1803, LAYOUTS["one rest chunk"]), (1800, 1808, LAYOUTS["four chunks"]),
                         (64, 64, LAYOUTS["one rest chunk"]), (8, 12, LAYOUTS["head = chunk"]),
                         (132, 132, LAYOUTS["head = chunk"])):
        P, G = 9, 4
        util = np.where(rng.random((P, G, 1)) < 0.4, 0.0,
                        rng.integers(0, 3, (P, G, T)) * (rng.random((P, G, T)) < 0.1)).astype(np.float32)
        util[rng.random((P, G, T)) < 0.05] = np.nan
        power = np.where(rng.random((P, G, T)) < 0.999, 140.0, 150.0).astype(np.float32)
        for variant, shift in RUNS:
            if variant == "tma" and ld % 4:
                continue
            d = tmp_path / f"T{T}_{ld}_{variant}{shift}"
            _write(str(d), util, power, False, shift, knobs, variant, ld)
            cases.append((d, util, power, variant, shift, knobs, ld))
    res = _run(emul, [c[0] for c in cases])
    for d, util, power, variant, shift, knobs, ld in cases:
        _check(res[str(d)], util, power, False, oracle_np, variant, knobs, shift, ld)


def test_synthetic_window_byte_share(emul, tmp_path, oracle_np):
    """a C2-shaped window (T 1800, 4 GPUs per pod, bench.py's generator and seed): the share of the bytes read equals
    the model's, on both kernels, and is well below one"""
    P, G, T = 60, 4, 1800
    util = oracle_np.synth_fill(0x5EED0002, 0, 0, P, G, T)
    power = oracle_np.synth_fill(0x5EED0002, 1, 0, P, G, T)
    knobs = (2, 16, 8192, 3, 2)                       # the library's default tiling
    cases = []
    for variant, shift in RUNS:
        d = tmp_path / f"synth_{variant}{shift}"
        _write(str(d), util, power, False, shift, knobs, variant)
        cases.append((d, variant, shift))
    res = _run(emul, [c[0] for c in cases])
    shares = {}
    for d, variant, shift in cases:
        r = res[str(d)]
        _check(r, util, power, False, oracle_np, variant, knobs, shift, T)
        shares[variant + str(shift)] = r["bytes"][0].sum() / (4.0 * util.size)
    assert all(0.2 < s < 0.8 for s in shares.values()), shares


def test_early_exit_under_thread_sanitizer(tmp_path, oracle_np):
    """the TMA stages that change rows mid-flight, the shared row counter and the warp's early leave, under
    ThreadSanitizer"""
    exe = _build(tmp_path, sanitize="thread")
    T = 1800
    util = _boundary_window(T, LAYOUTS.values(), False)[:6]
    power = np.full(util.shape, 100.0, np.float32)
    power[1, :, 130] = THR
    cases = []
    for variant, shift in (("tma", 0), ("ldg", 1)):
        d = tmp_path / f"tsan_{variant}"
        _write(str(d), util, power, False, shift, LAYOUTS["four chunks"], variant)
        cases.append((d, variant, shift))
    env = dict(os.environ, TSAN_OPTIONS="halt_on_error=1")
    res = _run(exe, [c[0] for c in cases], env=env)
    for d, variant, shift in cases:
        _check(res[str(d)], util, power, False, oracle_np, variant, LAYOUTS["four chunks"], shift, T)
