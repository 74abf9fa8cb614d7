"""gpr_resident_remap on the CPU: k_remap_check, k_remap_rows and remap_first_bad of gpu-pruner_b200/csrc/gpr_ring.cuh,
compiled from their source under tests/cpp/cuda_shim.hpp (tests/cpp/remap_emul.cpp) with ASan/UBSan and once with
TSan, against a numpy model of the remap (remap_model below):
  * every new buffer, bit for bit: new row i is old row src_rows[i], "no sample" for GPR_ROW_NONE, in the util and
    power planes and in their block index (the padding included);
  * the contract: the unrolled window of the new ring, at the unchanged head, is the window a rebuild would give with
    new row i fed by the series of old row src_rows[i]; a current index stays the block maxima of its rows;
  * a bad map (an old row out of range, or named twice) names its first bad new row, the check kernel and the host
    walk agree on it, and nothing is built.
Maps grow P, widen G, shrink both, permute, compact away departed pods and leave rows without a source, for T in
{1, 3, 4, 63, 64, 65, 1800} and heads 0, 1, 63, 64 and T - 1, with and without the power plane and the index.
tests/test_gpu_resident_remap.py runs the library on an H100."""
import concurrent.futures as cf
import os
import subprocess

import numpy as np
import pytest

import ring_scripts as RS
from test_hotpath_emul import ROOT, _extract
from test_ring_emul import _extract_ring

NONE = 0xFFFFFFFF
TS = [1, 3, 4, 63, 64, 65, 1800]
HEADS = [0, 1, 63, 64, -1]          # -1: T - 1
FLAGS = [0, 1, 2, 3]                # 1 = power plane, 2 = block index
P0, G0 = 5, 3                       # the old shape: 15 rows; new shapes reach 28 rows, past one SM's 16 CTAs
KINDS = ["grow P", "widen G", "shrink", "permutation", "compaction", "none rows"]


def remap_model(bufs, src):
    """the new buffers: row i of each is row src[i] of the old one, or "no sample" (all NO_SAMPLE) for NONE"""
    src = np.asarray(src, np.uint64)
    out = []
    for b in bufs:
        n = np.full((src.size, b.shape[1]), RS.NO_SAMPLE, np.uint32)
        keep = src != NONE
        n[keep] = b[src[keep].astype(np.int64)]
        out.append(n)
    return out


def first_bad(src, n_old):
    """the first new row whose entry is out of range or shared with another new row; len(src) if none"""
    src = np.asarray(src, np.uint64)
    live = src != NONE
    inside = live & (src < n_old)
    uses = np.bincount(src[inside].astype(np.int64), minlength=n_old)
    shared = np.zeros(src.size, bool)
    shared[inside] = uses[src[inside].astype(np.int64)] > 1
    bad = np.flatnonzero(live & (~inside | shared))
    return int(bad[0]) if bad.size else src.size


def make_map(kind, rng):
    """(P, G, src_rows) of one map kind over the old [P0][G0] ring"""
    old = np.arange(P0 * G0, dtype=np.uint32).reshape(P0, G0)
    if kind == "grow P":
        P, G = P0 + 2, G0
        src = np.concatenate([old.ravel(), np.full(2 * G0, NONE, np.uint32)])
    elif kind == "widen G":
        P, G = P0, G0 + 1
        src = np.concatenate([old, np.full((P0, 1), NONE, np.uint32)], axis=1).ravel()
    elif kind == "shrink":
        P, G = P0 - 1, G0 - 1
        src = old[:P, :G].ravel()
    elif kind == "permutation":
        P, G = P0, G0
        src = rng.permutation(old.ravel()).astype(np.uint32)
    elif kind == "compaction":
        kept = np.sort(rng.choice(P0, 3, replace=False))
        P, G = 3, G0
        src = old[kept].ravel()
    else:
        P, G = P0 + 2, G0 + 1
        src = np.full(P * G, NONE, np.uint32)
        at = rng.choice(P * G, P0 * G0 - 4, replace=False)
        src[at] = rng.choice(P0 * G0, at.size, replace=False)
    return P, G, np.ascontiguousarray(src, np.uint32)


class Case:
    def __init__(self, name, T, flags, head, src, P, G, n_old=P0 * G0, seed=0):
        self.name, self.T, self.flags, self.P, self.G, self.n_old = name, T, flags, P, G, n_old
        self.head = head % T
        self.src = np.asarray(src, np.uint32)
        rng = np.random.default_rng(seed)
        self.model = RS.Ring(n_old, 1, T, flags)
        for pl in range(len(self.model.planes)):
            cells = rng.integers(0, 2 ** 32, (n_old, T), dtype=np.uint64).astype(np.uint32)
            cells[rng.random((n_old, T)) < 0.3] = RS.NO_SAMPLE
            self.model.planes[pl] = cells
        self.model.head = self.head
        self.bufs = list(self.model.planes)
        if flags & 2:
            self.bufs += [self.model.block_max(pl)[0].view(np.uint32) for pl in range(len(self.model.planes))]

    def line(self):
        return f"{self.n_old} {self.T} {self.flags} {self.src.size}"


def matrix():
    rng = np.random.default_rng(11)
    out, k = [], 0
    for T in TS:
        for kind in KINDS:
            for flags in FLAGS:
                P, G, src = make_map(kind, rng)
                head = HEADS[k % len(HEADS)]
                k += 1
                out.append(Case(f"T={T} {kind} flags={flags} head={head % T}", T, flags, head, src, P, G, seed=k))
    return out


CASES = matrix()


def _build(d, sanitize="address,undefined"):
    (d / "hotpath_extract.inc").write_text(_extract())
    (d / "ring_extract.inc").write_text(_extract_ring())
    exe = d / ("remap_emul_" + sanitize.replace(",", "_"))
    cmd = ["g++", "-std=c++20", "-O1", "-g", "-pthread", "-Wall", "-Wno-unknown-pragmas", "-Wno-unused-function",
           "-fsanitize=" + sanitize, "-fno-omit-frame-pointer"]
    if sanitize != "thread":
        cmd.append("-fno-sanitize-recover=all")
    subprocess.run(cmd + ["-I", str(d), os.path.join(ROOT, "tests", "cpp", "remap_emul.cpp"), "-o", str(exe)],
                   check=True, capture_output=True, text=True)
    return str(exe)


def _run(exe, cases, d, sm=1, env=None):
    """run the cases in one process; returns (process, [(first, new buffers or None)] per case)"""
    d.mkdir(parents=True, exist_ok=True)
    (d / "cases.txt").write_text("".join(c.line() + "\n" for c in cases))
    data = [w for c in cases for w in [b.ravel() for b in c.bufs] + [c.src]]
    np.concatenate(data).astype(np.uint32).tofile(d / "data.u32")
    r = subprocess.run([exe, str(sm), str(d / "cases.txt"), str(d / "data.u32"), str(d / "out.u32")],
                       capture_output=True, text=True, timeout=1800, env=env)
    if r.returncode != 0:
        return r, None
    out, pos, res = np.fromfile(d / "out.u32", np.uint32), 0, []
    for c in cases:
        first = int(out[pos])
        pos += 1
        if first < c.src.size:
            res.append((first, None))
            continue
        bufs = []
        for b in c.bufs:
            n = c.src.size * b.shape[1]
            bufs.append(out[pos:pos + n].reshape(c.src.size, b.shape[1]))
            pos += n
        res.append((first, bufs))
    assert pos == out.size, (pos, out.size)
    return r, res


def _check_good(c, first, bufs):
    assert first == c.src.size, (c.name, first)
    want = remap_model(c.bufs, c.src)
    for k, (got, w) in enumerate(zip(bufs, want)):
        if not np.array_equal(got, w):
            r, t = np.argwhere(got != w)[0]
            raise AssertionError(f"{c.name}: buffer {k} row {r} word {t}: {got[r, t]:#010x} != {w[r, t]:#010x}")
    # the contract: the new ring's window at the same head = a rebuild feeding new row i from old row src[i]
    new = RS.Ring(c.P, c.G, c.T, c.flags)
    new.planes = [bufs[pl] for pl in range(len(new.planes))]
    new.head = c.head
    for pl in range(len(new.planes)):
        old_w = c.model.window(pl).reshape(c.n_old, c.T).view(np.uint32)
        rebuilt = np.full((c.src.size, c.T), RS.NO_SAMPLE, np.uint32)
        live = c.src != NONE
        rebuilt[live] = old_w[c.src[live]]
        assert np.array_equal(new.window(pl).reshape(-1, c.T).view(np.uint32), rebuilt), (c.name, pl)
        if c.flags & 2:   # the old index was current, so the new one is too
            bad = RS.index_matches(bufs[len(new.planes) + pl], new, pl)
            assert bad is None, (c.name, pl, bad)


@pytest.fixture(scope="module")
def matrix_runs(tmp_path_factory):
    """the matrix under UBSan, one process per T, in parallel"""
    d = tmp_path_factory.mktemp("remap_matrix")
    exe = _build(d, sanitize="undefined")
    by_t = {T: [c for c in CASES if c.T == T] for T in TS}
    with cf.ThreadPoolExecutor(len(TS)) as ex:
        runs = dict(zip(TS, ex.map(lambda T: _run(exe, by_t[T], d / f"T{T}"), TS)))
    return {c.name: (runs[c.T][0], runs[c.T][1][i] if runs[c.T][1] else None)
            for T in TS for i, c in enumerate(by_t[T])}


def test_matrix_covers_every_kind_head_and_flag():
    for T in TS:
        cs = [c for c in CASES if c.T == T]
        assert {c.head for c in cs} == {h % T for h in HEADS}, T
        assert {c.flags for c in cs} == set(FLAGS)
        assert {c.name.split(" flags")[0].split(" ", 1)[1] for c in cs} == set(KINDS)
    assert any(c.src.size > 16 for c in CASES) and any((c.src == NONE).any() for c in CASES)
    assert any(c.T % 4 for c in CASES) and any(c.T % 4 == 0 for c in CASES)


@pytest.mark.parametrize("case", CASES, ids=[c.name for c in CASES])
def test_remap_equals_the_model(matrix_runs, case):
    r, res = matrix_runs[case.name]
    assert r.returncode == 0, r.stderr[-3000:]
    _check_good(case, *res)


def test_model_pins_the_row_semantics():
    """the numpy model itself, on a hand-written map: grown, widened, a row without a source"""
    old = [np.arange(12, dtype=np.uint32).reshape(3, 4)]
    (new,) = remap_model(old, [2, NONE, 0])
    assert new.tolist() == [[8, 9, 10, 11], [NONE] * 4, [0, 1, 2, 3]]
    assert first_bad([0, 1, NONE, 2], 3) == 4
    assert first_bad([0, 3, 1], 3) == 1
    assert first_bad([NONE, 2, 0, 2], 3) == 1
    assert first_bad([0, 1, 2, 1, 7], 3) == 1


BAD_MAPS = {
    "out of range": [0, 1, 2, 15, 4],
    "out of range late": [NONE, 0, 1, 2, 3, 4, 5, 6, 7, 8, 16],
    "just out of range": [14, 15],
    "NONE - 1": [0xFFFFFFFE, 1],
    "twice": [0, 1, 2, 1],
    "twice, NONE between": [NONE, 3, NONE, NONE, 3],
    "three times": [9, 9, NONE, 9],
    "twice after out of range": [1, 20, 1],
    "out of range after twice": [NONE, 5, 5, 100],
    "twice, late": list(range(15)) + [NONE] * 6 + [14],
}


@pytest.fixture(scope="module")
def asan_exe(tmp_path_factory):
    """AddressSanitizer build: a read or write past a buffer, the map or a bitmap fails the run"""
    return _build(tmp_path_factory.mktemp("remap_asan"))


def test_bad_maps_name_the_first_bad_row_and_build_nothing(asan_exe, tmp_path):
    cases = [Case(name, 64, 3, 5, np.asarray(src, np.uint32), len(src), 1, seed=i)
             for i, (name, src) in enumerate(BAD_MAPS.items())]
    r, res = _run(asan_exe, cases, tmp_path / "c")
    assert r.returncode == 0, r.stderr[-3000:]
    for c, (first, bufs) in zip(cases, res):
        assert first == first_bad(c.src, c.n_old) < c.src.size, (c.name, first)
        assert bufs is None, c.name


def test_row_loop_and_odd_rows_under_address_sanitizer(asan_exe, tmp_path):
    """every map kind on T = 65 (scalar rows) and 1800 (16-byte rows), one SM: 28 new rows over 16 CTAs"""
    cases = [c for c in CASES if c.T in (65, 1800) and c.flags == 3]
    r, res = _run(asan_exe, cases, tmp_path / "c")
    assert r.returncode == 0, r.stderr[-3000:]
    for c, out in zip(cases, res):
        _check_good(c, *out)


def test_stale_index_moves_with_its_rows(asan_exe, tmp_path):
    """an index that no longer matches its ring (a merge left it stale) is moved as it is, not recomputed"""
    rng = np.random.default_rng(5)
    P, G, src = make_map("none rows", rng)
    c = Case("stale", 130, 3, 64, src, P, G, seed=9)
    c.bufs[2] = rng.integers(0, 2 ** 32, c.bufs[2].shape, dtype=np.uint64).astype(np.uint32)
    r, res = _run(asan_exe, [c], tmp_path / "c")
    assert r.returncode == 0, r.stderr[-3000:]
    first, bufs = res[0]
    assert first == c.src.size
    for got, want in zip(bufs, remap_model(c.bufs, c.src)):
        assert np.array_equal(got, want)


def test_check_and_gather_under_thread_sanitizer(tmp_path):
    """many threads race on one bitmap word and on the first bad row (a map that names a few old rows many times),
    then a good map of 600 rows over 2 SMs: the check passes' atomics and the gather's stores"""
    exe = _build(tmp_path, sanitize="thread")
    rng = np.random.default_rng(2)
    n_old = 40
    dup = rng.integers(0, 8, 700).astype(np.uint32)
    dup[:5] = [NONE, 0, 1, 2, 3]
    good = rng.permutation(600).astype(np.uint32)
    good[rng.choice(600, 50, replace=False)] = NONE
    cases = [Case("dups", 8, 3, 3, dup, 700, 1, n_old=n_old, seed=1),
             Case("good", 9, 3, 8, good, 600, 1, n_old=600, seed=2)]
    env = dict(os.environ, TSAN_OPTIONS="halt_on_error=1")
    r, res = _run(exe, cases, tmp_path / "c", sm=2, env=env)
    assert r.returncode == 0 and "ThreadSanitizer" not in r.stderr, r.stderr[-3000:]
    assert res[0] == (first_bad(dup, n_old), None)
    _check_good(cases[1], *res[1])
