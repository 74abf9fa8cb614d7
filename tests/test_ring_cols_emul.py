"""gpr_resident_cols on the CPU: k_ring_cols of gpu-pruner_b200/csrc/gpr_ring.cuh, compiled from its source under
tests/cpp/cuda_shim.hpp (tests/cpp/ring_cols_emul.cpp) with ASan/UBSan and once with TSan, launched at the position
gpr::ring_cols_start gives, against a numpy model: band column j of row r is the bucket (n_cols - 1 - j + newer) back
from the newest, which sits at ring position (head + T - 1) % T.
  * T in {1, 3, 4, 63, 64, 65, 1800}, heads at both ends of the ring and inside it;
  * newer and n_cols at their edges: one column, the whole ring, a band that ends at the newest bucket, one that starts
    at the oldest, and bands across the ring's wrap point;
  * the util and the power plane (the kernel does not know which it reads: both are rows of T words), any NaN payload
    and the special values, odd row counts.
tests/test_gpu_late_samples.py runs the library on an H100."""
import os
import subprocess

import numpy as np
import pytest

from test_hotpath_emul import ROOT, _extract
from test_live_rows_emul import other_nans
from test_ring_emul import _extract_ring

TS = [1, 3, 4, 63, 64, 65, 1800]


def band_model(plane, head, newer, n_cols):
    """[rows, n_cols]: the n_cols buckets that end `newer` buckets before the newest, oldest first"""
    T = plane.shape[1]
    back = n_cols - 1 - np.arange(n_cols) + newer
    return plane[:, (head + T - 1 - back) % T]


def bands(T):
    """(newer, n_cols) pairs at the edges of newer + n_cols <= T"""
    out = {(0, 1), (0, T), (T - 1, 1), (0, max(1, T // 2)), (T - max(1, T // 2), max(1, T // 2))}
    if T > 2:
        out |= {(1, T - 1), (T - 2, 2), (1, 1), (T // 3, T - T // 3 - 1)}
    return sorted(out)


def heads(T):
    return sorted({0, 1 % T, 2 % T, T // 3, T // 2, T - 2 if T > 1 else 0, T - 1})


def plane_of(rng, n_rows, T, power):
    """values a util or a power plane holds: the fill, samples, other NaNs, +-0, +-Inf, denormals"""
    a = rng.random((n_rows, T), np.float32) * (1000.0 if power else 100.0)
    bits = a.view(np.uint32).copy()
    kind = rng.integers(0, 6, (n_rows, T))
    bits[kind == 0] = 0xFFFFFFFF
    odd = kind == 1
    bits[odd] = other_nans(rng, int(odd.sum()))
    special = np.array([0x00000000, 0x80000000, 0x7F800000, 0xFF800000, 0x00000001, 0x80000001], np.uint32)
    sp = kind == 2
    bits[sp] = special[rng.integers(0, special.size, int(sp.sum()))]
    return bits


class Case:
    def __init__(self, n_rows, T, head, newer, n_cols, plane):
        self.n_rows, self.T, self.head, self.newer, self.n_cols = n_rows, T, head, newer, n_cols
        self.plane = plane
        self.want = band_model(plane, head, newer, n_cols)

    def line(self):
        return f"{self.n_rows} {self.T} {self.head} {self.newer} {self.n_cols}"


def matrix(T):
    rng = np.random.default_rng(T)
    out = []
    for k, head in enumerate(heads(T)):
        n_rows = int(rng.integers(1, 12)) * 2 + 1 if T < 1800 else 5
        plane = plane_of(rng, n_rows, T, power=bool(k % 2))
        for newer, n_cols in bands(T):
            out.append(Case(n_rows, T, head, newer, n_cols, plane))
    return out


def _build(d, sanitize="address,undefined"):
    (d / "hotpath_extract.inc").write_text(_extract())
    (d / "ring_extract.inc").write_text(_extract_ring())
    exe = d / ("ring_cols_emul_" + sanitize.replace(",", "_"))
    cmd = ["g++", "-std=c++20", "-O1", "-g", "-pthread", "-Wall", "-Wno-unknown-pragmas", "-Wno-unused-function",
           "-fsanitize=" + sanitize, "-fno-omit-frame-pointer"]
    if sanitize != "thread":
        cmd.append("-fno-sanitize-recover=all")
    subprocess.run(cmd + ["-I", str(d), os.path.join(ROOT, "tests", "cpp", "ring_cols_emul.cpp"), "-o", str(exe)],
                   check=True, capture_output=True, text=True)
    return str(exe)


def _run(exe, cases, d, sm=1, env=None):
    d.mkdir(parents=True, exist_ok=True)
    (d / "cases.txt").write_text("".join(c.line() + "\n" for c in cases))
    np.concatenate([c.plane.ravel() for c in cases]).astype(np.uint32).tofile(d / "data.u32")
    r = subprocess.run([exe, str(sm), str(d / "cases.txt"), str(d / "data.u32"), str(d / "out.u32")],
                       capture_output=True, text=True, timeout=1800, env=env)
    assert r.returncode == 0, r.stderr[-3000:]
    out, pos, res = np.fromfile(d / "out.u32", np.uint32), 0, []
    for c in cases:
        n = c.n_rows * c.n_cols
        res.append(out[pos:pos + n].reshape(c.n_rows, c.n_cols))
        pos += n
    assert pos == out.size
    return r, res


def _check(c, got):
    if not np.array_equal(got, c.want):
        r, j = map(int, np.argwhere(got != c.want)[0])
        raise AssertionError(f"{c.line()}: row {r} col {j}: {got[r, j]:#010x} != {c.want[r, j]:#010x}")


def test_model_pins_the_band():
    T, head = 5, 3                                        # ring positions 3 4 0 1 2, newest at 2
    plane = np.arange(T, dtype=np.uint32)[None, :]
    assert band_model(plane, head, 0, 1).tolist() == [[2]]
    assert band_model(plane, head, 0, T).tolist() == [[3, 4, 0, 1, 2]]
    assert band_model(plane, head, 1, 2).tolist() == [[0, 1]]
    assert band_model(plane, head, 4, 1).tolist() == [[3]]


@pytest.fixture(scope="module")
def asan_exe(tmp_path_factory):
    return _build(tmp_path_factory.mktemp("ring_cols_asan"))


@pytest.mark.parametrize("T", TS)
def test_band_equals_the_model(asan_exe, tmp_path, T):
    cases = matrix(T)
    assert {c.head for c in cases} == set(heads(T)) and any(c.n_rows % 2 for c in cases)
    _, res = _run(asan_exe, cases, tmp_path / "c")
    for c, got in zip(cases, res):
        _check(c, got)


def test_band_under_thread_sanitizer(tmp_path):
    """many rows over 2 SMs: every CTA writes rows of its own, no cell twice"""
    exe = _build(tmp_path, sanitize="thread")
    rng = np.random.default_rng(5)
    cases = [Case(67, 1800, 1700, 30, 200, plane_of(rng, 67, 1800, False)),
             Case(129, 65, 64, 0, 65, plane_of(rng, 129, 65, True)),
             Case(33, 4, 2, 1, 3, plane_of(rng, 33, 4, False))]
    env = dict(os.environ, TSAN_OPTIONS="halt_on_error=1")
    r, res = _run(exe, cases, tmp_path / "c", sm=2, env=env)
    assert "ThreadSanitizer" not in r.stderr, r.stderr[-3000:]
    for c, got in zip(cases, res):
        _check(c, got)
