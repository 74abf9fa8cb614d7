"""gpr_samples_scatter on the CPU: k_samples_check and k_samples_scatter of gpu-pruner_b200/csrc/gpr_samples.cuh,
compiled from their source under tests/cpp/cuda_shim.hpp (tests/cpp/samples_emul.cpp) with the text kernel's
atomic_merge, under AddressSanitizer + UndefinedBehaviorSanitizer and ThreadSanitizer, against a numpy model of the
text path's rules (window membership and bucket in milliseconds, to_f32 keeping non-zero values non-zero, the power
snap, the NaN-aware max) — cell for cell, bit for bit, with the out-of-window and tiny counts:
  * ragged series, empty series, several series into one row, unsorted samples, aligned and unaligned arrays;
  * the window edges t_end, t_end - N, t_end - N + 1 ms and t_end + 1 ms;
  * the power plane at 149.999999 / 150 / 150.0000001 W against 150 W, -0.0, negatives, 1e-50, 1e39, NaN, +-Inf;
  * a resident ring whose newest bucket is not the last column (wrap-around);
  * host batches cut into tiny pieces, inside and between series: every sample merged exactly once;
  * every malformed batch rejected by the host check and the check kernel alike, the plane untouched.
tests/test_gpu_samples.py checks the library on an H100 against the text parser itself."""
import os
import subprocess

import numpy as np
import pytest

import emul_build

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FILL = np.uint32(0xFFFFFFFF)


def _extract_samples():
    src = open(os.path.join(ROOT, "gpu-pruner_b200", "csrc", "gpr_samples.cuh")).read()
    body = src[src.index("namespace samples {") + len("namespace samples {"):src.index("}  // namespace samples")]
    assert "asm" not in body and "__shared__" not in body
    for name in ("k_samples_scatter", "k_samples_check", "for_each_piece", "series_faults", "series_from"):
        assert name in body, name
    return body


def _build(d, sanitize):
    (d / "samples_extract.inc").write_text(_extract_samples())
    (d / "text_kernel_extract.inc").write_text(emul_build.extract_parse_kernel())
    exe = d / ("samples_emul_" + sanitize.replace(",", "_"))
    cmd = ["g++", "-std=c++20", "-O1", "-g", "-pthread", "-Wno-unknown-pragmas", "-fsanitize=" + sanitize,
           "-fno-omit-frame-pointer"]
    if sanitize != "thread":
        cmd.append("-fno-sanitize-recover=all")
    subprocess.run(cmd + ["-I", str(d), "-I", os.path.join(ROOT, "tests", "cpp"),
                          os.path.join(ROOT, "tests", "cpp", "samples_emul.cpp"), "-o", str(exe)],
                   check=True, capture_output=True, text=True)
    return str(exe)


@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    return _build(tmp_path_factory.mktemp("samples"), "address,undefined")


# ---- the model: what gpr_text_parse makes of the same samples written as text ------------------------------------
def _f32_up(thr):
    up = np.float32(thr)
    if float(up) < thr:
        up = np.nextafter(up, np.float32(np.inf))
    return up


def _values_f32(v, thr):
    """to_f32 (a non-zero value stays non-zero) and, with a threshold, the power snap; returns (f32, tiny mask)"""
    with np.errstate(over="ignore"):
        f = v.astype(np.float32)
    tiny = (v != 0) & (f == 0) & ~np.isnan(v)
    f[tiny] = np.where(v[tiny] < 0, np.float32(-1e-45), np.float32(1e-45))
    if thr is not None and thr != 0 and not np.isnan(thr):
        up = _f32_up(thr)
        down = up if np.isneginf(up) else np.nextafter(up, np.float32(-np.inf))
        f = np.where((v >= thr) & (f < up), up, f).astype(np.float32)
        f = np.where((v < thr) & (f >= up), down, f).astype(np.float32)
    return f, tiny


def _merge(cell_bits, v):
    """NaN-aware max, +0 above -0 (the atomic merge's order)"""
    if np.isnan(v):
        return cell_bits
    c = cell_bits.view(np.float32)
    if np.isnan(c) or c < v or (c == v == 0 and np.signbit(c) and not np.signbit(v)):
        return np.float32(v).view(np.uint32)
    return cell_bits


def model(b):
    offsets, rows, ts, vals = b["offsets"], b["rows"], b["ts"], b["values"]
    plane = b["plane"].copy()
    T = b["T"]
    sidx = np.repeat(np.arange(len(rows)), np.diff(offsets.astype(np.int64)))
    inw = (ts <= b["t_end"]) & (ts > b["t_lo"])
    back = np.where(inw, (b["t_end"] - ts) // b["step"], 0)
    inw &= back < T
    col = (b["col_end"] - back) % T
    f, tiny = _values_f32(vals, b["thr"])
    for i in np.flatnonzero(inw):
        r = rows[sidx[i]]
        plane[r, col[i]] = _merge(plane[r, col[i]], f[i])
    return plane, int((~inw).sum()), int((tiny & inw).sum())


def _write(d, b, piece=0, unaligned=0):
    d.mkdir(parents=True, exist_ok=True)
    thr = b["thr"] if b["thr"] is not None else 0.0
    (d / "params.txt").write_text(" ".join(str(x) for x in (
        len(b["rows"]), b["plane"].shape[0], b["T"], b["t_end"], b["t_lo"], b["step"], b["col_end"], repr(float(thr)),
        piece, unaligned)) + "\n")
    b["offsets"].astype(np.uint64).tofile(d / "offsets.u64")
    b["rows"].astype(np.uint32).tofile(d / "rows.u32")
    b["ts"].astype(np.int64).tofile(d / "ts.i64")
    b["values"].astype(np.float64).tofile(d / "values.f64")
    b["plane"].astype(np.uint32).tofile(d / "plane.u32")


def run(exe, d, b, piece=0, unaligned=0, sm=1, env=None):
    _write(d, b, piece, unaligned)
    r = subprocess.run([exe, str(sm), str(d)], capture_output=True, text=True, timeout=1800, env=env)
    assert r.returncode == 0, r.stderr[-3000:]
    raw = np.fromfile(d / "out.bin", np.uint8)
    bad = int(raw[:4].view(np.uint32)[0])
    n_oow, n_tiny = (int(x) for x in raw[8:24].view(np.uint64))
    plane = raw[24:].view(np.uint32).reshape(b["plane"].shape)
    return bad, n_oow, n_tiny, plane


def check(exe, d, b, **kw):
    bad, n_oow, n_tiny, plane = run(exe, d, b, **kw)
    assert bad == 0
    want, w_oow, w_tiny = model(b)
    if not np.array_equal(plane, want):
        r, c = np.argwhere(plane != want)[0]
        raise AssertionError(f"cell ({r}, {c}): {plane[r, c]:#010x} != {want[r, c]:#010x}")
    assert (n_oow, n_tiny) == (w_oow, w_tiny)
    return b


# ---- batches --------------------------------------------------------------------------------------------------
T_END = 1_700_000_000_000   # ms
STEP = 1000
T = 60


def batch(lengths, rows, n_rows, values_fn, rng, T=T, thr=None, col_end=None, shuffle=True, ts_fn=None, plane=None):
    lengths = np.asarray(lengths, np.int64)
    offsets = np.concatenate([[0], np.cumsum(lengths)]).astype(np.uint64)
    n = int(offsets[-1])
    if ts_fn is None:   # mostly inside the window, some before it and some after t_end
        ts = T_END - rng.integers(-3 * STEP, (T + 5) * STEP, n)
    else:
        ts = ts_fn(n)
    if shuffle:   # samples of a series in any order
        for s in range(len(lengths)):
            a, e = int(offsets[s]), int(offsets[s + 1])
            ts[a:e] = rng.permutation(ts[a:e])
    return dict(offsets=offsets, rows=np.asarray(rows, np.uint32), ts=ts.astype(np.int64),
                values=values_fn(n).astype(np.float64), T=T, t_end=T_END, t_lo=T_END - T * STEP, step=STEP,
                col_end=T - 1 if col_end is None else col_end, thr=thr,
                plane=np.full((n_rows, T), FILL, np.uint32) if plane is None else plane)


def util_values(rng):
    def f(n):
        v = rng.integers(0, 101, n).astype(np.float64)
        v[rng.random(n) < 0.3] = 0.0
        ratio = rng.random(n) < 0.3
        v[ratio] = rng.random(int(ratio.sum()))   # 17-digit PROF ratios
        v[rng.random(n) < 0.05] = np.nan
        return v
    return f


SPECIAL = np.array([0.0, -0.0, -3.5, -1e-50, 1e-50, 1e39, -1e39, np.nan, np.inf, -np.inf, 149.999999, 150.0,
                    150.0000001, 149.99999999999997, 1e-45, 7e-46, 3.4028235e38, 0.1, 1 / 3])


def special_values(rng):
    def f(n):
        v = rng.integers(0, 400, n).astype(np.float64)
        pick = rng.random(n) < 0.5
        v[pick] = rng.choice(SPECIAL, int(pick.sum()))
        return v
    return f


def test_ragged_series_into_shared_rows(emul, tmp_path):
    """ragged and empty series, several series feeding one row, unsorted samples, about ten 2048-sample chunks over
    8 CTAs; the device batch read with 128-bit pairs and with scalar loads"""
    rng = np.random.default_rng(1)
    lengths = rng.integers(0, 500, 80)
    lengths[[0, 7, 8, 9, 79]] = 0
    rows = rng.integers(0, 30, 80)
    b = batch(lengths, rows, 30, util_values(rng), rng)
    assert int(b["offsets"][-1]) > 8 * 2048
    check(emul, tmp_path / "a", b)
    check(emul, tmp_path / "u", b, unaligned=1)


def test_power_plane_snaps_to_the_threshold(emul, tmp_path):
    rng = np.random.default_rng(2)
    lengths = rng.integers(1, 300, 40)
    for thr in (150.0, 149.99, -2.0):
        b = batch(lengths, rng.integers(0, 12, 40), 12, special_values(rng), rng, thr=thr)
        check(emul, tmp_path / str(thr), b)
    # the plane without a power clause: plain rounding
    check(emul, tmp_path / "plain", batch(lengths, rng.integers(0, 12, 40), 12, special_values(rng), rng))
    # 149.999999 W stays below a 150 W threshold, 150.0000001 W reaches it
    b = batch([3], [0], 1, lambda n: np.array([149.999999, 150.0000001, 149.999999]), rng, thr=150.0,
              ts_fn=lambda n: np.array([T_END, T_END - STEP, T_END - 2 * STEP]), shuffle=False)
    check(emul, tmp_path / "edge", b)
    got = run(emul, tmp_path / "edge2", b)[3][0].view(np.float32)
    assert got[T - 1] < np.float32(150) and got[T - 2] == np.float32(150) and got[T - 3] < np.float32(150)


def test_window_edges(emul, tmp_path):
    """t_end and t_end - N + 1 ms are inside; t_end - N and t_end + 1 ms are not; bucket borders at whole steps"""
    rng = np.random.default_rng(3)
    N = T * STEP
    edges = np.array([T_END, T_END - N, T_END - N + 1, T_END + 1, T_END - STEP, T_END - STEP + 1, T_END - N + STEP,
                      T_END - N + STEP + 1, 0, -T_END, 2 ** 62])
    b = batch([len(edges)], [2], 3, lambda n: np.arange(1, n + 1, dtype=np.float64), rng,
              ts_fn=lambda n: edges.copy(), shuffle=False)
    bad, n_oow, _, plane = run(emul, tmp_path / "e", b)
    assert n_oow == 5   # t_end - N, t_end + 1, 0, -t_end, 2^62
    row = plane[2].view(np.float32)
    # newest bucket: t_end (1) and t_end - step + 1 (6); one back: t_end - step (5); oldest: t_end - N + 1 (3) and
    # t_end - N + step (7); the one after it: t_end - N + step + 1 (8)
    assert (row[T - 1], row[T - 2], row[0], row[1]) == (6, 5, 7, 8)
    check(emul, tmp_path / "m", b)


def test_resident_ring_wraps(emul, tmp_path):
    """a ring whose newest bucket sits at column 3 of 10: buckets wrap to the end of the row; cells merged into a
    pre-filled ring keep their larger values"""
    rng = np.random.default_rng(4)
    Tr = 10
    plane = np.full((6, Tr), FILL, np.uint32)
    plane[:, :5] = rng.integers(0, 60, (6, 5)).astype(np.float32).view(np.uint32)
    lengths = rng.integers(0, 40, 12)
    b = batch(lengths, rng.integers(0, 6, 12), 6, util_values(rng), rng, T=Tr, col_end=3, plane=plane)
    check(emul, tmp_path / "r", b)
    for col_end in (0, 9):
        b = batch(lengths, rng.integers(0, 6, 12), 6, util_values(rng), rng, T=Tr, col_end=col_end, plane=plane)
        check(emul, tmp_path / f"r{col_end}", b)


@pytest.mark.parametrize("piece", [1, 2, 3, 7, 64, 2049, 5000])
def test_host_pieces_merge_every_sample_once(emul, tmp_path, piece):
    """the host piece walk (gpr::samples::for_each_piece, the loop gpr_api.cu uploads by) at tiny piece sizes, cuts
    inside and between series and around empty ones, each piece in buffers of exactly its size: the out-of-window and
    tiny counts, which a sample merged twice or never would change, equal the model's, and so does every cell"""
    rng = np.random.default_rng(5 + piece)
    lengths = rng.integers(0, 9 if piece < 64 else 700, 60)
    lengths[[3, 4, 30]] = 0

    def vals(n):
        v = util_values(rng)(n)
        v[rng.random(n) < 0.2] = 1e-50   # tiny: counted once per in-window sample
        return v
    b = batch(lengths, rng.integers(0, 20, 60), 20, vals, rng)
    check(emul, tmp_path / "p", b, piece=piece)
    check(emul, tmp_path / "pu", b, piece=piece, unaligned=1)


def test_malformed_batches_leave_the_plane_untouched(emul, tmp_path):
    rng = np.random.default_rng(6)
    plane = rng.integers(0, 100, (8, T)).astype(np.float32).view(np.uint32)
    good = batch([5, 0, 9, 4], [1, 2, 7, 0], 8, util_values(rng), rng, plane=plane)
    assert run(emul, tmp_path / "ok", good)[0] == 0
    cases = {}
    b = dict(good, rows=np.array([1, 2, 8, 0], np.uint32))
    cases["row >= n_rows"] = (b, 1)
    off = good["offsets"].copy()
    off[2], off[3] = off[3], off[2]   # decreasing
    cases["decreasing offsets"] = (dict(good, offsets=off), 2)
    off = good["offsets"].copy() + np.uint64(1)
    cases["offsets[0] != 0"] = (dict(good, offsets=off, ts=np.append(good["ts"], 0),
                                     values=np.append(good["values"], 0.0)), 4)
    cases["no series, offsets[0] != 0"] = (dict(good, offsets=np.array([3], np.uint64), rows=np.zeros(0, np.uint32),
                                                ts=good["ts"][:3], values=good["values"][:3]), 4)
    for k, (name, (b, bits)) in enumerate(cases.items()):
        bad, n_oow, n_tiny, got = run(emul, tmp_path / f"bad{k}", b)
        assert bad & bits, name
        assert np.array_equal(got, plane) and n_oow == n_tiny == 0, name


def test_empty_batches(emul, tmp_path):
    rng = np.random.default_rng(7)
    for k, lengths in enumerate(([], [0, 0, 0])):
        b = batch(lengths, np.zeros(len(lengths), np.uint32), 2, util_values(rng), rng)
        assert check(emul, tmp_path / f"e{k}", b)


def test_scatter_under_thread_sanitizer(tmp_path):
    """16 CTAs (two SMs' worth) over ragged series that share rows, cut into host pieces and read in place: the merges
    of concurrent threads into one cell go through atomics only.  Values are non-negative (NaN, zero, tiny, integers,
    ratios, +Inf): the merge of a negative value reads its cell before its compare-and-swap, which the GPU's memory
    model allows and C++'s calls a race."""
    exe = _build(tmp_path, "thread")
    rng = np.random.default_rng(8)
    lengths = rng.integers(0, 900, 40)

    def vals(n):
        v = np.abs(util_values(rng)(n))
        v[rng.random(n) < 0.05] = 1e-50
        v[rng.random(n) < 0.02] = np.inf
        return v
    b = batch(lengths, rng.integers(0, 4, 40), 4, vals, rng)
    env = dict(os.environ, TSAN_OPTIONS="halt_on_error=1")
    for piece in (0, 3000):
        bad, n_oow, n_tiny, plane = run(exe, tmp_path / f"t{piece}", b, piece=piece, sm=2, env=env)
        want, w_oow, w_tiny = model(b)
        assert bad == 0 and np.array_equal(plane, want) and (n_oow, n_tiny) == (w_oow, w_tiny)
