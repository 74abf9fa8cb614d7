"""gpr_resident_retime on the CPU: k_retime_rows of gpu-pruner_b200/csrc/gpr_ring.cuh, compiled from its source under
tests/cpp/cuda_shim.hpp (tests/cpp/retime_emul.cpp) with ASan/UBSan and once with TSan, against a numpy model of the
merge, and gpr::retime_plan (gpu-pruner_b200/csrc/gpr_retime.h) against a table of accepted and refused grid changes.
The model: keep the newest n_keep buckets of the ring (chronological from the head), new bucket b (0 = newest) is old
buckets [factor b, min(factor b + factor, n_keep)) counted from the newest, written oldest first; a group's value is
the maximum of its cells that are not NaN, +0 when the maximum is a zero and a +0 is among them, and the fill
0xFFFFFFFF when every cell is a NaN — what text::atomic_merge leaves in a fill cell.
  * T in {1, 2, 3, 4, 5, 63, 64, 65, 1800}, heads 0, 1, T/2, T-1, factor in {1, 2, 3, 4, 7, 32, 33, T}, n_keep in
    {1, factor-1, factor, factor+1, T-1, T}: new rows of T' % 4 == 0 (16-byte stores) and others (4-byte stores);
  * cells: the fill, NaNs of other payloads and either sign, +-0 in both orders inside one group, negatives, +-Inf,
    denormals of either sign;
  * the index rebuilt from the new plane, padding included.
tests/test_gpu_resident_retime.py runs the library on an H100."""
import os
import subprocess

import numpy as np
import pytest

from test_hotpath_emul import ROOT, _extract
from test_live_rows_emul import block_index, index_ld, other_nans
from test_ring_emul import _extract_ring

FILL = 0xFFFFFFFF
TS = [1, 2, 3, 4, 5, 63, 64, 65, 1800]
SPECIAL = np.array([0x00000000, 0x80000000, 0x7F800000, 0xFF800000, 0x00000001, 0x80000001, 0x007FFFFF, 0x807FFFFF,
                    0x3F800000, 0xBF800000, 0x42C80000, 0xC2C80000], np.uint32)


def _merge(bits):
    """one group's value, from the float semantics of the rule (not the key trick the kernel uses)"""
    v = bits.view(np.float32)
    ok = ~np.isnan(v)
    if not ok.any():
        return FILL
    m = v[ok].max()
    if m == 0:
        return 0 if (bits[ok] == 0).any() else 0x80000000
    return int(np.float32(m).view(np.uint32))


def _merge_rows(bits):
    """_merge of every row of [rows, n] at once"""
    v = bits.view(np.float32)
    ok = ~np.isnan(v)
    m = np.where(ok, v, -np.inf).max(axis=1)
    plus = (ok & (bits == 0)).any(axis=1)
    out = m.astype(np.float32).view(np.uint32).copy()
    out[m == 0] = np.where(plus[m == 0], 0, 0x80000000)
    out[~ok.any(axis=1)] = FILL
    return out


def retime_model(plane, head, n_keep, factor):
    rows, T = plane.shape
    chron = plane[:, (head + np.arange(T)) % T]
    keep = chron[:, T - n_keep:]           # oldest first, the newest last
    T_new = -(-n_keep // factor)
    out = np.empty((rows, T_new), np.uint32)
    for p in range(T_new):
        b = T_new - 1 - p
        lo, hi = factor * b, min(factor * b + factor, n_keep)   # old buckets from the newest
        out[:, p] = _merge_rows(keep[:, n_keep - hi:n_keep - lo])
    return out


def cells(rng, n):
    kind = rng.integers(0, 6, n)
    out = np.full(n, FILL, np.uint32)
    out[kind == 1] = other_nans(rng, int((kind == 1).sum()))
    out[kind == 2] = rng.choice(SPECIAL, int((kind == 2).sum()))
    out[kind >= 3] = (rng.random(int((kind >= 3).sum())) * 200 - 50).astype(np.float32).view(np.uint32)
    return out


class Case:
    def __init__(self, T, head, n_keep, factor, index, seed, rows=5):
        self.T, self.head, self.n_keep, self.factor, self.index = T, head % T, n_keep, factor, index
        rng = np.random.default_rng(seed)
        plane = np.stack([cells(rng, T) for _ in range(rows)])
        plane[0] = FILL                                        # a row without a sample
        plane[1] = other_nans(rng, T)                          # only other NaNs: no sample either
        if T >= 2:                                             # +-0 in both orders next to each other, -0 alone
            for r, pair in ((2, (0x80000000, 0x00000000)), (3, (0x00000000, 0x80000000))):
                plane[r] = FILL
                for c in range(0, T - 1, 2):
                    plane[r, (self.head + c) % T], plane[r, (self.head + c + 1) % T] = pair
            plane[4, rng.random(T) < 0.5] = 0x80000000
        self.plane = plane
        self.T_new = -(-n_keep // factor)
        self.want = retime_model(plane, self.head, n_keep, factor)
        self.want_idx = block_index(self.want) if index else None
        self.name = f"T={T} head={self.head} n_keep={n_keep} factor={factor} index={index}"

    def line(self):
        return f"{self.plane.shape[0]} {self.T} {self.head} {self.n_keep} {self.factor} {self.index}"


def matrix():
    out, k = [], 0
    for T in TS:
        for head in sorted({0, 1 % T, T // 2, T - 1}):
            for factor in sorted({1, 2, 3, 4, 7, 32, 33, T}):
                for n_keep in sorted({1, factor - 1, factor, factor + 1, T - 1, T}):
                    if not 1 <= n_keep <= T:
                        continue
                    k += 1
                    out.append(Case(T, head, n_keep, factor, k % 2, k))
    return out


_CASES = []


def cases():
    if not _CASES:
        _CASES.extend(matrix())
    return _CASES


def _build(d, sanitize="address,undefined"):
    (d / "hotpath_extract.inc").write_text(_extract())
    (d / "ring_extract.inc").write_text(_extract_ring())
    exe = d / ("retime_emul_" + sanitize.replace(",", "_"))
    cmd = ["g++", "-std=c++20", "-O1", "-g", "-pthread", "-Wall", "-Wno-unknown-pragmas", "-Wno-unused-function",
           "-fsanitize=" + sanitize, "-fno-omit-frame-pointer"]
    if sanitize != "thread":
        cmd.append("-fno-sanitize-recover=all")
    subprocess.run(cmd + ["-I", str(d), "-I", os.path.join(ROOT, "gpu-pruner_b200", "csrc"),
                          os.path.join(ROOT, "tests", "cpp", "retime_emul.cpp"), "-o", str(exe)],
                   check=True, capture_output=True, text=True)
    return str(exe)


def _run(exe, cases, d, sm=1, env=None):
    d.mkdir(parents=True, exist_ok=True)
    (d / "cases.txt").write_text("".join(c.line() + "\n" for c in cases))
    np.concatenate([c.plane.ravel() for c in cases]).astype(np.uint32).tofile(d / "data.u32")
    r = subprocess.run([exe, "rows", str(sm), str(d / "cases.txt"), str(d / "data.u32"), str(d / "out.u32")],
                       capture_output=True, text=True, timeout=1800, env=env)
    assert r.returncode == 0, r.stderr[-3000:]
    out, pos, res = np.fromfile(d / "out.u32", np.uint32), 0, []
    for c in cases:
        rows = c.plane.shape[0]
        n = rows * c.T_new
        plane = out[pos:pos + n].reshape(rows, c.T_new)
        pos += n
        idx = None
        if c.index:
            m = rows * index_ld(c.T_new)
            idx = out[pos:pos + m].reshape(rows, index_ld(c.T_new))
            pos += m
        res.append((plane, idx))
    assert pos == out.size
    return r, res


def _check(c, got):
    plane, idx = got
    if not np.array_equal(plane, c.want):
        r, p = map(int, np.argwhere(plane != c.want)[0])
        raise AssertionError(f"{c.name}: row {r} cell {p}: {plane[r, p]:#010x} != {c.want[r, p]:#010x}")
    if c.index:
        # block maxima compare as floats (k_reindex's fmaxf may keep either zero of a block holding +0 and -0)
        assert np.array_equal(idx.view(np.float32), c.want_idx.view(np.float32), equal_nan=True), c.name
        pad = idx[:, -(-c.T_new // 64):]
        assert (pad == FILL).all(), c.name


def test_matrix_covers_every_shape():
    for T in TS:
        cs = [c for c in cases() if c.T == T]
        assert {c.head for c in cs} == {0, 1 % T, T // 2, T - 1}
        assert {c.factor for c in cs} == {f for f in (1, 2, 3, 4, 7, 32, 33, T)}
        assert {c.n_keep for c in cs} >= {1, T}
    assert any(c.T_new % 4 == 0 for c in cases()) and any(c.T_new % 4 for c in cases())
    assert any(c.index and c.T_new % 4 == 0 for c in cases()) and any(c.index and c.T_new % 4 for c in cases())


def test_model_pins_the_merge_rule():
    assert _merge(np.array([0x80000000, 0x00000000], np.uint32)) == 0
    assert _merge(np.array([0x00000000, 0x80000000], np.uint32)) == 0
    assert _merge(np.array([0x80000000, FILL], np.uint32)) == 0x80000000
    assert _merge(np.array([0x7FC00001, FILL, 0xFFC00000], np.uint32)) == FILL
    assert _merge(np.array([0x80000001, 0x80000000], np.uint32)) == 0x80000000          # -denormal < -0
    assert _merge(np.array([0x00000001, 0x00000000], np.uint32)) == 0x00000001          # denormal > +0
    assert _merge(np.array([0xFF800000, 0xBF800000], np.uint32)) == 0xBF800000
    groups = np.array([[0x80000000, 0x00000000], [0x80000000, FILL], [0x7FC00001, 0xFFC00000], [0x80000001, 0x80000000],
                       [0xFF800000, 0xBF800000]], np.uint32)
    assert _merge_rows(groups).tolist() == [_merge(g) for g in groups]
    plane = np.arange(1, 7, dtype=np.float32).view(np.uint32).reshape(1, 6)             # oldest first at head 0
    assert retime_model(plane, 0, 5, 2).view(np.float32).tolist() == [[2.0, 4.0, 6.0]]
    assert retime_model(plane, 2, 6, 4).view(np.float32).tolist() == [[4.0, 6.0]]        # newest is ring pos 1


@pytest.fixture(scope="module")
def asan_exe(tmp_path_factory):
    return _build(tmp_path_factory.mktemp("retime_asan"))


@pytest.mark.parametrize("T", TS)
def test_retime_equals_the_model(asan_exe, tmp_path, T):
    todo = [c for c in cases() if c.T == T]
    _, res = _run(asan_exe, todo, tmp_path / "c")
    for c, got in zip(todo, res):
        _check(c, got)


def test_rows_under_thread_sanitizer(tmp_path):
    """several rows per CTA over 2 SMs, with the index rebuilt in the CTA that wrote the row"""
    exe = _build(tmp_path, sanitize="thread")
    cases = [Case(65, 30, 64, 2, 1, 91, rows=40), Case(1800, 900, 1800, 3, 1, 92, rows=6),
             Case(63, 62, 62, 7, 0, 93, rows=40)]
    env = dict(os.environ, TSAN_OPTIONS="halt_on_error=1")
    r, res = _run(exe, cases, tmp_path / "c", sm=2, env=env)
    assert "ThreadSanitizer" not in r.stderr, r.stderr[-3000:]
    for c, got in zip(cases, res):
        _check(c, got)


# ---- retime_plan -----------------------------------------------------------------------------------------------------
def _T(N, s):
    return -(-N // s)


PLANS = [
    # (N, s, N', s') -> (n_keep, factor) or a refusal's words
    ((1800, 15, 1800, 30), (120, 2)),                 # step x2
    ((1800, 15, 1800, 45), (120, 3)),                 # step x3
    ((1800, 15, 900, 15), (60, 1)),                   # --duration 30 -> 15
    ((1800, 15, 900, 30), (60, 2)),                   # both
    ((120, 2, 60, 6), (30, 3)),
    ((100, 15, 100, 30), (7, 2)),                     # N % s != 0, N' == N: T = 7 -> 4
    ((100, 15, 90, 15), (6, 1)),                      # N' % s == 0
    ((60, 5, 60, 600), (12, 120)),                    # one new bucket
    ((1800, 15, 1800, 15), "did not change"),
    ((1800, 30, 1800, 15), "finer"),
    ((1800, 15, 1800, 10), "finer"),
    ((1800, 10, 1800, 15), "not a whole multiple"),    # x1.5
    ((1800, 15, 1800, 20), "not a whole multiple"),
    ((900, 15, 1800, 15), "longer"),
    ((900, 15, 1800, 30), "longer"),
    ((1800, 15, 890, 15), "cuts a bucket"),            # N' < N, N' % s != 0
    ((100, 15, 95, 30), "cuts a bucket"),
    ((0, 15, 60, 15), "not a ring's grid"),
    ((60, 0, 60, 15), "not a ring's grid"),
    ((60, 15, 60, 0), "not a ring's grid"),
]


def test_retime_plan_table(tmp_path):
    exe = _build(tmp_path)
    lines = [f"{N} {s} {_T(N, s) if s > 0 else 1} {N2} {s2}" for (N, s, N2, s2), _ in PLANS]
    lines.append("60 15 5 60 30")                     # T that is not ceil(N / s)
    (tmp_path / "plans.txt").write_text("\n".join(lines) + "\n")
    r = subprocess.run([exe, "plan", str(tmp_path / "plans.txt")], capture_output=True, text=True, timeout=60)
    assert r.returncode == 0, r.stderr
    got = r.stdout.splitlines()
    assert len(got) == len(PLANS) + 1
    for ((N, s, N2, s2), want), line in zip(PLANS, got):
        if isinstance(want, tuple):
            assert line == "keep %d %d" % want, (N, s, N2, s2, line)
            n_keep, k = want
            assert -(-n_keep // k) == _T(N2, s2)             # T' = ceil(n_keep / k) = ceil(N' / s')
        else:
            assert line.startswith("refused ") and want in line, (N, s, N2, s2, line)
    assert got[-1] == "refused the grid is not a ring's grid"


def test_plan_accepts_exactly_the_exact_changes():
    """the conditions of gpr_retime.h, checked by brute force on small grids: a retime is exact iff every integer
    timestamp's new bucket is the merge of the old buckets the plan groups, and the new window is the kept part"""
    for N in range(1, 40):
        for s in range(1, 8):
            T = _T(N, s)
            for N2 in range(1, N + 1):
                for k in range(1, 5):
                    s2 = k * s
                    exact = N2 == N or N2 % s == 0
                    if not exact:
                        continue
                    n_keep = T if N2 == N else N2 // s
                    for d in range(N2):                    # d = t_end - ts of every second in the new window
                        b_old = d // s
                        assert b_old < n_keep and (d // s2) == b_old // k
                    # every second of the kept old buckets that the old window holds lies in the new window
                    for b in range(n_keep):
                        for d in range(b * s, min((b + 1) * s, N)):
                            assert d < N2 or (N2 == N)
