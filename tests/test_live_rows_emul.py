"""gpr_resident_live_rows on the CPU: k_live_rows of gpu-pruner_b200/csrc/gpr_ring.cuh, compiled from its source under
tests/cpp/cuda_shim.hpp (tests/cpp/live_rows_emul.cpp) with ASan/UBSan and once with TSan, on the buffers the entry
point picks (gpr::live_rows_from_index), against a numpy model: row r is live iff a cell of it is not NaN in the util
plane or the power plane.
  * T in {1, 3, 4, 63, 64, 65, 1800} (4-byte and 16-byte rows), heads 0, 1, T/2 and T-1;
  * rows with exactly one sample at each ring position, in either plane; rows of fill only, of other NaNs (any payload,
    either sign), of +-0, +-Inf and denormals only;
  * row counts that are not multiples of 32 (the padding bits must be zero, every word written once);
  * with and without the block index: a current index is read instead of the planes, a stale one is not.
tests/test_gpu_resident_live_rows.py runs the library on an H100."""
import os
import subprocess

import numpy as np
import pytest

import ring_scripts as RS
from test_hotpath_emul import ROOT, _extract
from test_ring_emul import _extract_ring

TS = [1, 3, 4, 63, 64, 65, 1800]
FLAGS = [0, 1, 2, 3, 6, 7]            # 1 = power plane, 2 = block index, 4 = the index is stale
FILL = RS.NO_SAMPLE


def index_ld(T):
    return ((T + 63) // 64 + 3) & ~3


def block_index(plane_bits):
    """[rows, idx_ld] of the block maxima (NaN iff the block holds no sample, as k_reindex's fmaxf gives them), NaN
    padding.  (np.fmax is not used: with a signalling NaN among the cells it may return NaN.)"""
    v = plane_bits.view(np.float32)
    rows, T = v.shape
    out = np.full((rows, index_ld(T)), np.nan, np.float32)
    for b in range((T + 63) // 64):
        blk = v[:, b * 64:min(T, b * 64 + 64)]
        has = ~np.isnan(blk)
        m = np.where(has, blk, -np.inf).max(axis=1)
        out[:, b] = np.where(has.any(axis=1), m, np.nan)
    return out.view(np.uint32)


def live_model(planes):
    live = np.zeros(planes[0].shape[0], bool)
    for p in planes:
        live |= (~np.isnan(p.view(np.float32))).any(axis=1)
    return live


def words_of(live):
    n = (live.size + 31) // 32
    padded = np.zeros(n * 32, bool)
    padded[:live.size] = live
    return np.packbits(padded, bitorder="little").view(np.uint32)


def other_nans(rng, n):
    """NaNs that are not the fill: any payload, either sign, quiet and signalling"""
    payload = rng.integers(1, 1 << 23, n, dtype=np.uint64).astype(np.uint32)
    sign = rng.integers(0, 2, n).astype(np.uint32) << 31
    out = sign | 0x7F800000 | payload
    out[out == FILL] = 0x7FC00000
    return out


class Case:
    def __init__(self, name, T, flags, head, seed, positions=None):
        self.name, self.T, self.flags, self.head = name, T, flags, head % T
        rng = np.random.default_rng(seed)
        power = flags & 1
        n_planes = 2 if power else 1
        rows = [[], []]

        def add(cells0, cells1=None):
            rows[0].append(cells0)
            rows[1].append(cells1 if cells1 is not None else np.full(T, FILL, np.uint32))

        dead = lambda: np.full(T, FILL, np.uint32)
        # exactly one sample, at chronological position c = ring position (head + c) % T, alternating planes
        for i, c in enumerate(range(T) if positions is None else positions):
            row = dead()
            row[(self.head + c) % T] = np.float32(rng.choice([0.0, 37.5, 100.0, 1e-42])).view(np.uint32)
            if power and i % 2:
                add(dead(), row)
            else:
                add(row)
        # no sample: the fill, other NaNs, both
        add(dead())
        add(other_nans(rng, T))
        mixed = other_nans(rng, T)
        mixed[rng.random(T) < 0.5] = FILL
        add(mixed, other_nans(rng, T) if power else None)
        # one special value among other NaNs: a sample
        for bits in (0x00000000, 0x80000000, 0x7F800000, 0xFF800000, 0x00000001, 0x80000001):
            row = other_nans(rng, T)
            row[rng.integers(0, T)] = bits
            add(row)
        # random rows, then rows up to a count that is not a multiple of 32
        extra = int(rng.integers(3, 40))
        if (len(rows[0]) + extra) % 32 == 0:
            extra += 1
        for _ in range(extra):
            row = dead()
            live = rng.random(T) < rng.choice([0.0, 0.01, 0.3])
            row[live] = rng.random(int(live.sum()), np.float32).view(np.uint32)
            add(row, None)
        self.planes = [np.stack(rows[k]).astype(np.uint32) for k in range(n_planes)]
        self.n_rows = self.planes[0].shape[0]
        self.index = []
        if flags & 2:
            self.index = [block_index(p) for p in self.planes]
            if flags & 4:   # stale: anything at all, the planes decide
                self.index = [rng.integers(0, 2 ** 32, i.shape, dtype=np.uint64).astype(np.uint32) for i in self.index]
        self.want = live_model(self.planes)

    def line(self):
        return f"{self.n_rows} {self.T} {self.flags}"


def matrix():
    out, k = [], 0
    for T in TS:
        for head in sorted({0, 1 % T, T // 2, T - 1}):
            for flags in FLAGS:
                k += 1
                # T = 1800: every position once per flag set (at head 0), a stride of them elsewhere
                pos = None if T < 1800 or head == 0 else sorted(set(range(0, T, 97)) | {T - 1})
                out.append(Case(f"T={T} head={head} flags={flags}", T, flags, head, k, pos))
    return out


def _build(d, sanitize="address,undefined"):
    (d / "hotpath_extract.inc").write_text(_extract())
    (d / "ring_extract.inc").write_text(_extract_ring())
    exe = d / ("live_rows_emul_" + sanitize.replace(",", "_"))
    cmd = ["g++", "-std=c++20", "-O1", "-g", "-pthread", "-Wall", "-Wno-unknown-pragmas", "-Wno-unused-function",
           "-fsanitize=" + sanitize, "-fno-omit-frame-pointer"]
    if sanitize != "thread":
        cmd.append("-fno-sanitize-recover=all")
    subprocess.run(cmd + ["-I", str(d), os.path.join(ROOT, "tests", "cpp", "live_rows_emul.cpp"), "-o", str(exe)],
                   check=True, capture_output=True, text=True)
    return str(exe)


def _run(exe, cases, d, sm=1, env=None):
    d.mkdir(parents=True, exist_ok=True)
    (d / "cases.txt").write_text("".join(c.line() + "\n" for c in cases))
    np.concatenate([b.ravel() for c in cases for b in c.planes + c.index]).astype(np.uint32).tofile(d / "data.u32")
    r = subprocess.run([exe, str(sm), str(d / "cases.txt"), str(d / "data.u32"), str(d / "out.u32")],
                       capture_output=True, text=True, timeout=1800, env=env)
    assert r.returncode == 0, r.stderr[-3000:]
    out, pos, res = np.fromfile(d / "out.u32", np.uint32), 0, []
    for c in cases:
        n = (c.n_rows + 31) // 32
        res.append(out[pos:pos + n])
        pos += n
    assert pos == out.size
    return r, res


def _check(c, got):
    want = words_of(c.want)
    if not np.array_equal(got, want):
        w = int(np.flatnonzero(got != want)[0])
        raise AssertionError(f"{c.name}: word {w}: {got[w]:#010x} != {want[w]:#010x}")


CASES = matrix()


def test_matrix_covers_every_position_head_and_flag():
    for T in TS:
        cs = [c for c in CASES if c.T == T]
        assert {c.head for c in cs} == {0, 1 % T, T // 2, T - 1}
        assert {c.flags for c in cs} == set(FLAGS)
    assert all(c.n_rows % 32 for c in CASES)
    assert any(c.T % 4 for c in CASES) and any(c.T % 4 == 0 for c in CASES)


@pytest.fixture(scope="module")
def asan_exe(tmp_path_factory):
    return _build(tmp_path_factory.mktemp("live_rows_asan"))


@pytest.mark.parametrize("T", TS)
def test_live_rows_equal_the_model(asan_exe, tmp_path, T):
    cases = [c for c in CASES if c.T == T]
    _, res = _run(asan_exe, cases, tmp_path / "c")
    for c, got in zip(cases, res):
        _check(c, got)


def test_model_pins_the_row_semantics():
    T = 5
    rows = np.full((4, T), FILL, np.uint32)
    rows[1, 2] = 0x7FC00000                            # another NaN: no sample
    rows[2, 4] = 0x80000000                            # -0: a sample
    p1 = np.full((4, T), FILL, np.uint32)
    p1[3, 0] = 0xFF800000                              # -Inf in the power plane
    assert live_model([rows, p1]).tolist() == [False, False, True, True]
    assert words_of(np.array([True] + [False] * 31 + [True])).tolist() == [1, 1]


def test_a_current_index_is_read_instead_of_the_planes(asan_exe, tmp_path):
    """the call reads 1/64 of the bytes from a current index: an index that says "no sample" where the planes hold one
    (which a current index never does) shows which of the two was read; marked stale, the planes are read"""
    rng = np.random.default_rng(3)
    out = []
    for flags in (3, 7):
        c = Case(f"index flags={flags}", 130, flags, 7, 40 + flags)
        lie = rng.random(c.n_rows) < 0.5
        for ix in c.index:
            ix[lie] = FILL
        out.append((c, lie))
    _, res = _run(asan_exe, [c for c, _ in out], tmp_path / "c")
    (cur, lie), (stale, _) = out
    _check(stale, res[1])
    want = words_of(live_model(cur.planes) & ~lie)
    assert np.array_equal(res[0], want)


def test_rows_and_words_under_thread_sanitizer(tmp_path):
    """many words over 2 SMs (every warp owns words of its own: no word is written twice, no atomics)"""
    exe = _build(tmp_path, sanitize="thread")
    cases = [Case("tsan 63", 63, 1, 5, 91, positions=list(range(63)) * 9),
             Case("tsan 1800", 1800, 3, 900, 92, positions=list(range(0, 1800, 7))),
             Case("tsan stale", 65, 7, 64, 93)]
    env = dict(os.environ, TSAN_OPTIONS="halt_on_error=1")
    r, res = _run(exe, cases, tmp_path / "c", sm=2, env=env)
    assert "ThreadSanitizer" not in r.stderr, r.stderr[-3000:]
    for c, got in zip(cases, res):
        _check(c, got)
