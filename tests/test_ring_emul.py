"""The resident ring of daemon mode on the CPU: k_append, k_open, k_reindex and block_max_warp of
gpu-pruner_b200/csrc/gpr_ring.cuh, compiled from their source under tests/cpp/cuda_shim.hpp (tests/cpp/ring_emul.cpp)
and launched with the spans, grids and per-plane choices the header gives gpr_api.cu, against the numpy ring model of
tests/ring_scripts.py:
  * the ring, bit for bit, and the head after every operation;
  * the block index: every block the fmax of its ring positions, the padding NaN;
  * the verdict: the float64 oracle on the unrolled ring equals the oracle on the index (a window of idx_ld
    "samples" per series, as gpr_decide_resident reads it).
The head visits the awkward positions (0, 1, 63, 64, 65, T - 1) for T from 1 to 1800, and every case asserts the regime
it was built for.  tests/test_gpu_resident.py runs the same scripts through libgpr.so on an H100."""
import concurrent.futures as cf
import os
import subprocess

import numpy as np
import pytest

import kat
import ring_scripts as RS
from test_hotpath_emul import ROOT, _extract

CASES = RS.cases()


def _extract_ring():
    src = open(os.path.join(ROOT, "gpu-pruner_b200", "csrc", "gpr_ring.cuh")).read()
    body = src[src.index("namespace gpr {") + len("namespace gpr {"):src.rindex("}  // namespace gpr")]
    assert "asm" not in body and "__shared__" not in body
    for name in ("k_append", "k_open", "k_reindex", "block_max_warp", "recompute_blocks", "ring_span"):
        assert name in body, name
    return body


def _build(d, sanitize="address,undefined"):
    (d / "hotpath_extract.inc").write_text(_extract())
    (d / "ring_extract.inc").write_text(_extract_ring())
    exe = d / ("ring_emul_" + sanitize.replace(",", "_"))
    cmd = ["g++", "-std=c++20", "-O1", "-g", "-pthread", "-Wall", "-Wno-unknown-pragmas", "-Wno-unused-function",
           "-fsanitize=" + sanitize, "-fno-omit-frame-pointer"]
    if sanitize != "thread":
        cmd.append("-fno-sanitize-recover=all")
    subprocess.run(cmd + ["-I", str(d), os.path.join(ROOT, "tests", "cpp", "ring_emul.cpp"), "-o", str(exe)],
                   check=True, capture_output=True, text=True)
    return str(exe)


@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    """AddressSanitizer build: a read or write past the end of a plane, an index or a source fails the run"""
    return _build(tmp_path_factory.mktemp("ring"))


@pytest.fixture(scope="module")
def matrix_runs(tmp_path_factory):
    """every case of the matrix, run in parallel (a CTA is 128 real threads, so the whole matrix takes a while)"""
    d = tmp_path_factory.mktemp("ring_matrix")
    exe = _build(d, sanitize="undefined")
    with cf.ThreadPoolExecutor(os.cpu_count() or 4) as ex:
        runs = list(ex.map(lambda ic: _run(exe, ic[1], d / f"c{ic[0]}"), enumerate(CASES)))
    return {c.name: r for c, r in zip(CASES, runs)}


def _serialize(case, d):
    """script + data files for ring_emul"""
    lines, data, off = [], [], 0
    for op in case.ops:
        if op[0] == "init":
            lines.append("init %d %d %d %d" % op[1:])
        elif op[0] == "append":
            _, n_new, ld, util, power = op
            lines.append(f"append {n_new} {ld} {off} {'nopower' if power is None else 'power'}")
            for a in (util, power):
                if a is not None:
                    data.append(a.ravel())
                    off += a.size
        elif op[0] == "advance":
            lines.append(f"advance {op[1]}")
        elif op[0] == "write":
            lines.append(f"write {op[1]} {off}")
            data.append(op[2].ravel())
            off += op[2].size
        else:
            lines.append("reindex")
    d.mkdir(parents=True, exist_ok=True)
    (d / "script.txt").write_text("\n".join(lines) + "\n")
    np.concatenate(data + [np.zeros(1, np.uint32)]).astype(np.uint32).tofile(d / "data.u32")


def _run(exe, case, d, env=None):
    _serialize(case, d)
    r = subprocess.run([exe, str(case.sm), str(d / "script.txt"), str(d / "data.u32"), str(d / "out.u32")],
                       capture_output=True, text=True, timeout=1800, env=env)
    return r, (np.fromfile(d / "out.u32", np.uint32) if r.returncode == 0 else None)


def decide_both(model):
    """the oracle's verdict on the unrolled ring and on the block-maxima index of the same ring"""
    from oracle import oracle_c
    power = model.window(1) if len(model.planes) > 1 else None
    full = oracle_c.decide(model.window(0), power, power_threshold=RS.THR)
    iu = model.block_max(0)[0].reshape(model.P, model.G, -1)
    ip = model.block_max(1)[0].reshape(model.P, model.G, -1) if power is not None else None
    return full, oracle_c.decide(iu, ip, power_threshold=RS.THR)


def _check_case(case, out):
    """walk the emulator's dumps along the model; returns the number of operations checked"""
    pos, n_checked, verdicts = 0, 0, 0
    for op, m in RS.run_model(case):
        head = int(out[pos])
        pos += 1
        assert head == m.head, (case.name, n_checked, op[0], head, m.head)
        for pl, plane in enumerate(m.planes):
            got = out[pos:pos + plane.size].reshape(plane.shape)
            pos += plane.size
            if not np.array_equal(got, plane):
                r, t = np.argwhere(got != plane)[0]
                raise AssertionError(f"{case.name} op {n_checked} ({op[0]}): ring plane {pl} row {r} position {t}: "
                                     f"{got[r, t]:#010x} != {plane[r, t]:#010x}")
        if m.index:
            for pl in range(len(m.planes)):
                n = m.rows * RS.index_ld(m.T)
                got = out[pos:pos + n]
                pos += n
                if op[0] != "write":   # a direct write leaves the index stale until the reindex that follows it
                    bad = RS.index_matches(got, m, pl)
                    assert bad is None, f"{case.name} op {n_checked} ({op[0]} {op[1:2]}): index plane {pl}: {bad}"
            if op[0] in ("append", "advance"):
                full, idx = decide_both(m)
                for k in ("decision_bits", "candidate_bits"):
                    assert np.array_equal(full[k], idx[k]), (case.name, n_checked, k)
                assert (full["n_series"], full["n_candidates"]) == (idx["n_series"], idx["n_candidates"])
                assert kat.smax_equal(full["series_max"], idx["series_max"]), (case.name, n_checked)
                verdicts += 1
        n_checked += 1
    assert pos == out.size, (case.name, pos, out.size)
    return n_checked, verdicts


def test_matrix_reaches_every_regime():
    """each case reaches the regime it was built for, the matrix as a whole every regime, and the head starts an
    operation at each of 0, 1, 63, 64, 65 and T - 1"""
    for c in CASES:
        assert c.regimes <= c.hit, (c.name, c.regimes - c.hit)
    assert set().union(*(c.hit for c in CASES)) == RS.ALL_REGIMES
    assert {c.T for c in CASES} >= set(RS.TS)
    for c in CASES:
        if c.name.startswith("T="):
            starts = set()
            for op, m in RS.run_model(c):
                if op[0] in ("append", "advance"):
                    starts.add(prev)
                prev = m.head if m is not None else 0
            assert starts >= {h for h in (0, 1, 63, 64, 65, c.T - 1) if h < c.T}, c.name


@pytest.mark.parametrize("case", CASES, ids=[c.name for c in CASES])
def test_ring_and_index_equal_the_model(matrix_runs, case):
    r, out = matrix_runs[case.name]
    assert r.returncode == 0, r.stderr[-3000:]
    n, verdicts = _check_case(case, out)
    assert n == len(case.ops)
    assert verdicts > 0 or not (case.flags & 2)


def test_row_loop_case_under_address_sanitizer(emul, tmp_path):
    """the strided CTA row loop of 18 rows on one SM, with every plane, index and source an exact-size allocation"""
    case = next(c for c in CASES if c.name == "row loop, 1 SM")
    r, out = _run(emul, case, tmp_path / "c")
    assert r.returncode == 0, r.stderr[-3000:]
    assert _check_case(case, out)[0] == len(case.ops)


def test_stale_power_columns_are_opened(emul, tmp_path):
    """gpr_append with power_cols NULL on a ring with a power plane: the power readings of T columns ago leave the
    window, so a pod whose only readings at or above the threshold were there is a candidate again"""
    T = 4
    ops = [("init", 1, 1, T, 3),
           ("append", T, T, RS._bits([0, 0, 0, 0]).reshape(1, T), RS._bits([200] * T).reshape(1, T)),
           ("append", T, T, RS._bits([0, 0, 0, 0]).reshape(1, T), None)]
    case = RS.Case("repro", 1, 1, 1, T, 3, ops, set())
    r, out = _run(emul, case, tmp_path / "c")
    assert r.returncode == 0, r.stderr[-3000:]
    _check_case(case, out)
    m = list(RS.run_model(case))[-1][1]
    assert (m.planes[1] == RS.NO_SAMPLE).all()
    full, idx = decide_both(m)
    assert full["n_candidates"] == 1 and idx["n_candidates"] == 1


def test_advance_recomputes_the_index(emul, tmp_path):
    """gpr_resident_advance on an index ring: opening the 64 buckets that held the only busy samples must take them
    out of the index too, or the series stays busy"""
    T = 128
    ops = [("init", 1, 1, T, 2),
           ("append", 64, 64, RS._bits([5.0] * 64).reshape(1, 64), None),
           ("append", 64, 64, RS._bits([0.0] * 64).reshape(1, 64), None),
           ("advance", 64)]
    case = RS.Case("repro", 1, 1, 1, T, 2, ops, set())
    r, out = _run(emul, case, tmp_path / "c")
    assert r.returncode == 0, r.stderr[-3000:]
    _check_case(case, out)
    m = list(RS.run_model(case))[-1][1]
    full, idx = decide_both(m)
    assert full["n_candidates"] == 1 and idx["n_candidates"] == 1 and idx["series_max"][0, 0] == 0


def test_wrapped_append_under_thread_sanitizer(tmp_path):
    """a wrapped append whose two runs of touched blocks meet in one block (head 200 of 240, 240 columns), on 5 rows
    of one CTA each: the column stores, the barrier and the block recomputes of the CTA's four warps"""
    exe = _build(tmp_path, sanitize="thread")
    rng = np.random.default_rng(3)
    T, rows = 240, 5
    ops = [("init", 5, 1, T, 3),
           ("append", 200, 200, RS._cells(rng, 0, rows, 200), RS._cells(rng, 1, rows, 200)),
           ("append", T, T + 7, RS._cells(rng, 0, rows, T + 7), None),
           ("append", T, T, RS._mixed(rng, 0, rows, T), RS._mixed(rng, 1, rows, T)),
           ("advance", 100)]
    case = RS.Case("tsan", 2, 5, 1, T, 3, ops, set())
    m = RS.Ring(5, 1, T, 3)
    m.head = 200
    assert "a block in both runs" in RS._regimes(m, ops[2], 2)
    env = dict(os.environ, TSAN_OPTIONS="halt_on_error=1")
    r, out = _run(exe, case, tmp_path / "c", env=env)
    assert r.returncode == 0 and "ThreadSanitizer" not in r.stderr, r.stderr[-3000:]
    _check_case(case, out)
