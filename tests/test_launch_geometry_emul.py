"""The decision kernels' source (tests/cpp/hotpath_emul.cpp) in the launch geometries the library itself picks: the
emulated device has 1, 2, 3 or 7 SMs, the tuning knobs take every value gpr_create accepts, and the reduce and fold
grids, the TMA ring layout and the TMA -> LDG fallbacks come from gpu-pruner_b200/csrc/gpr_launch.h, the header
gpr_api.cu launches from.  Every case names the regime it is there for and asserts that it reached it, so the matrix
cannot quietly shrink; every run is compared with the numpy oracle."""
import os
import subprocess

import numpy as np
import pytest

import geometry
import kat as KAT
from test_hotpath_emul import ROOT, _extract, _extract_synth, _parse, _run, _write_case

K = geometry.Knobs


def _build(d, sanitize=None):
    (d / "hotpath_extract.inc").write_text(_extract())
    (d / "synth_extract.inc").write_text(_extract_synth())
    exe = d / ("hotpath_emul_tsan" if sanitize else "hotpath_emul")
    cmd = ["g++", "-std=c++20", "-O1", "-pthread", "-Wall", "-Wno-unknown-pragmas", "-Wno-unused-function"]
    if sanitize:
        cmd += ["-g", "-fsanitize=" + sanitize]
    subprocess.run(cmd + ["-I", str(d), os.path.join(ROOT, "tests", "cpp", "hotpath_emul.cpp"), "-o", str(exe)],
                   check=True, capture_output=True, text=True)
    return str(exe)


@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    return _build(tmp_path_factory.mktemp("geometry"))


def _plan_of(line_plan):
    f = line_plan[len("plan="):].split(",")
    n = [int(x) for x in f[1:]]
    return {"kernel": f[0], "fallback": geometry.FALLBACKS[n[0]], "grid": n[1], "block": n[2], "smem": n[3],
            "depth": n[4], "stage_bytes": n[5], "chunk_elems": n[6], "n_chunks": n[7], "fold_grid": n[8],
            "fold_threads": n[9], "fold_rounds": n[10]}


def _run_with_plans(emul, dirs):
    r = subprocess.run([emul] + [str(d) for d in dirs], capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0, r.stderr[-2000:]
    res = _parse(r.stdout.splitlines())
    for l in r.stdout.splitlines():
        f = l.split()
        for run in res[f[0]]:
            if run["variant"] == f[1] and "plan" not in run:
                run["plan"] = _plan_of(f[-1])
                break
    return res


def _window(rng, P, G, T, power):
    kind = rng.random((P, G, 1))
    util = np.where(kind < 0.4, 0.0, rng.integers(0, 101, (P, G, T)) * (rng.random((P, G, T)) < 0.3)).astype(np.float32)
    util[rng.random((P, G, T)) < 0.02] = np.nan
    util[rng.random((P, G)) < 0.05] = np.nan
    # a single busy sample in the last column / the first column of some idle series: row heads and tails
    burst = rng.random((P, G)) < 0.05
    util[burst, T - 1] = 3.0
    util[rng.random((P, G)) < 0.05, 0] = 2.0
    kw = {}
    if power:
        w = np.where(rng.random((P, G, T)) < 0.995, rng.uniform(40, 149, (P, G, T)), 400.0).astype(np.float32)
        w[rng.random((P, G)) < 0.3] = 55.5
        w[rng.random((P, G)) < 0.05, T - 1] = 150.0
        kw = {"power": w, "thr": 150.0}
    elig = (rng.random(P) > 0.1).astype(np.uint8)
    created = rng.integers(1_700_000_000 - 5000, 1_700_000_000, P)
    return util, kw, elig, created


def _has(p, **want):
    return all(p[k] == v for k, v in want.items())


# (regime, knobs, P, G, T, ld, power, labels, check(plans by label, P, G, T) -> bool)
CASES = [
    ("depth 1", K(1, 8, 2048, 1, 1, 64), 37, 3, 1536, 1536, True, "ldg,tma,u8",
     lambda p, P, G, T: _has(p["tma"], kernel="tma", depth=1) and p["tma"]["n_chunks"] >= 3),
    ("depth 1", K(7, 16, 8192, 3, 2, 128), 45, 2, 2048, 2048, False, "ldg,tma",   # the budget, not the knob
     lambda p, P, G, T: _has(p["tma"], kernel="tma", depth=1, n_chunks=1)),
    ("fewer chunks than stages", K(2, 4, 2048, 3, 2, 128), 45, 2, 600, 604, True, "ldg,ldg+1,tma,u8",
     lambda p, P, G, T: _has(p["tma"], kernel="tma", depth=3) and p["tma"]["n_chunks"] < 3),
    ("4-element last chunk", K(3, 16, 512, 3, 1, 256), 5, 3, 4100, 4100, True, "ldg,tma",
     lambda p, P, G, T: p["tma"]["kernel"] == "tma" and T - (p["tma"]["n_chunks"] - 1) * p["tma"]["chunk_elems"] == 4),
    ("4-element last chunk", K(1, 4, 512, 2, 2, 64), 3, 2, 4100, 4108, False, "tma,u8",
     lambda p, P, G, T: _has(p["tma"], kernel="tma", depth=2) and T - (p["tma"]["n_chunks"] - 1) * p["tma"]["chunk_elems"] == 4),
    ("T smaller than one chunk", K(7, 32, 8192, 2, 2, 64), 70, 4, 100, 100, True, "ldg,tma,u8",
     lambda p, P, G, T: _has(p["tma"], kernel="tma", n_chunks=1, depth=2) and 4 * T < 8192 and p["tma"]["grid"] == 7),
    ("T smaller than one chunk", K(2, 8, 2048, 2, 1, 256), 33, 1, 8, 8, False, "tma",
     lambda p, P, G, T: _has(p["tma"], kernel="tma", n_chunks=1, chunk_elems=8)),
    ("fallback: T % 4 != 0", K(2, 8, 8192, 3, 2, 128), 41, 3, 37, 37, True, "tma,u8",
     lambda p, P, G, T: _has(p["tma"], kernel="ldg", fallback="alignment")),
    ("fallback: misaligned base", K(3, 4, 2048, 2, 1, 64), 50, 2, 64, 64, True, "tma,tma+1",
     lambda p, P, G, T: _has(p["tma+1"], kernel="ldg", fallback="alignment") and _has(p["tma"], kernel="tma")),
    ("fallback: shared memory over budget", K(1, 32, 8192, 3, 2, 256), 9, 2, 2048, 2048, True, "tma",
     lambda p, P, G, T: _has(p["tma"], kernel="ldg", fallback="smem")),
    ("fold of 3+ rounds", K(1, 8, 512, 2, 1, 64), 799, 1, 12, 12, True, "ldg,tma",
     lambda p, P, G, T: p["ldg"]["fold_rounds"] >= 3 and p["ldg"]["fold_grid"] == 1),
    ("fold of 3+ rounds", K(2, 16, 2048, 1, 2, 128), 2090, 1, 4, 4, False, "ldg,u8",
     lambda p, P, G, T: p["ldg"]["fold_rounds"] >= 3 and p["ldg"]["grid"] == 4),
    ("fold of 3+ rounds", K(3, 4, 8192, 3, 1, 256), 6170, 1, 4, 4, False, "tma",
     lambda p, P, G, T: p["tma"]["fold_rounds"] >= 3 and p["tma"]["fold_grid"] == 3),
    ("fold of 3+ rounds", K(7, 32, 512, 1, 2, 64), 3601, 1, 4, 4, True, "ldg",
     lambda p, P, G, T: p["ldg"]["fold_rounds"] >= 3 and p["ldg"]["fold_grid"] == 7 and p["ldg"]["grid"] == 14),
    ("G >= 33", K(2, 16, 512, 2, 1, 128), 9, 40, 132, 132, True, "ldg,tma,u8",
     lambda p, P, G, T: G >= 33 and p["tma"]["kernel"] == "tma" and p["tma"]["n_chunks"] == 2),
    ("G >= 33", K(1, 32, 2048, 3, 2, 256), 4, 65, 20, 21, True, "ldg,ldg+1,tma",
     lambda p, P, G, T: G >= 33 and _has(p["tma"], kernel="ldg", fallback="alignment")),
]
REGIMES = {"depth 1", "fewer chunks than stages", "4-element last chunk", "T smaller than one chunk",
           "fallback: T % 4 != 0", "fallback: misaligned base", "fallback: shared memory over budget",
           "fold of 3+ rounds", "G >= 33"}


def _write_knobs(d, knobs, labels):
    with open(os.path.join(d, "knobs.txt"), "w") as f:
        f.write(f"{knobs.sm_count} {knobs.tma_warps} {knobs.tma_chunk} {knobs.tma_depth} {knobs.ldg_ctas} "
                f"{knobs.fold_threads} {labels}\n")


def test_matrix_covers_every_knob_value():
    ks = [c[1] for c in CASES]
    assert {k.sm_count for k in ks} == {1, 2, 3, 7}
    assert {k.tma_warps for k in ks} == {4, 8, 16, 32}
    assert {k.tma_chunk for k in ks} == {512, 2048, 8192}
    assert {k.tma_depth for k in ks} == {1, 2, 3}
    assert {k.ldg_ctas for k in ks} == {1, 2}
    assert {k.fold_threads for k in ks} == {64, 128, 256}
    assert {c[0] for c in CASES} == REGIMES
    assert any(c[2] % 32 for c in CASES) and any(c[4] % 4 for c in CASES)


def test_every_geometry_equals_the_oracle(emul, tmp_path, oracle_np):
    rng = np.random.default_rng(20261015)
    dirs, data = [], []
    for i, (regime, knobs, P, G, T, ld, power, labels, check) in enumerate(CASES):
        util, kw, elig, created = _window(rng, P, G, T, power)
        d = tmp_path / f"g{i}"
        _write_case(str(d), util, kw.get("power"), kw.get("thr", 0.0), elig if i % 2 else None,
                    created if i % 3 == 0 else None, 1_700_000_000 - 2500, ld)
        _write_knobs(str(d), knobs, labels)
        dirs.append(d)
        data.append((util, kw, elig if i % 2 else None, created if i % 3 == 0 else None))
    res = _run_with_plans(emul, dirs)
    hit = set()
    tma_warps_ran, ldg_ctas_ran = set(), set()
    for (regime, knobs, P, G, T, ld, power, labels, check), d, (util, kw, elig, created) in zip(CASES, dirs, data):
        runs = res[str(d)]
        want_labels = set(labels.split(","))
        if "u8" in want_labels and not os.path.exists(d / "util.u8"):
            want_labels.discard("u8")
        assert {r["variant"] for r in runs} == want_labels | {l + "#2" for l in want_labels}, (regime, d)
        want = oracle_np.decide(util, kw.get("power"), elig, created, 1_700_000_000 - 2500, kw.get("thr", 0.0))
        for r in runs:
            tag = (regime, knobs, r["variant"])
            assert r["clean"], tag
            assert np.array_equal(r["d"], want["decision_bits"]), tag
            assert np.array_equal(r["c"], want["candidate_bits"]), tag
            assert np.array_equal(r["v"], want["veto_bits"]), tag
            assert r["counts"] == (want["n_series"], want["n_candidates"], want["n_decisions"]), tag
            assert KAT.smax_equal(r["smax"].reshape(want["series_max"].shape), want["series_max"]), tag
            assert r["plan"]["fold_threads"] == knobs.fold_threads
            if r["plan"]["kernel"] == "tma":
                tma_warps_ran.add(r["plan"]["block"] // 32)
            if r["plan"]["kernel"] == "ldg":
                ldg_ctas_ran.add((knobs.ldg_ctas, r["plan"]["grid"] == knobs.ldg_ctas * knobs.sm_count))
        plans = {r["variant"]: r["plan"] for r in runs if "#" not in r["variant"]}
        assert check(plans, P, G, T), (regime, knobs, plans)
        if P % 32:
            hit.add("P % 32 != 0")
        hit.add(regime)
    assert hit == REGIMES | {"P % 32 != 0"}
    assert tma_warps_ran == {4, 8, 16, 32}                      # every warp count ran the TMA kernel itself
    assert {(1, True), (2, True)} <= ldg_ctas_ran               # and both LDG grids were the full sm_count * ctas


def test_plan_tool_agrees_with_the_emulator(emul, tmp_path):
    """the helper the GPU tests ask for the geometry reports what the emulated launches used"""
    exe = geometry.build(tmp_path)
    knobs = K(3, 4, 512, 2, 1, 64)
    P, G, T = 70, 3, 260
    util = np.zeros((P, G, T), np.float32)
    d = tmp_path / "c"
    _write_case(str(d), util)
    _write_knobs(str(d), knobs, "ldg,tma,tma+1")
    runs = {r["variant"]: r["plan"] for r in _run_with_plans(emul, [d])[str(d)]}
    for label, variant, ok in (("ldg", "ldg", True), ("tma", "tma", True), ("tma+1", "tma", False)):
        p = geometry.plan(exe, knobs, variant, T, P * G, tma_ok=ok, P=P)
        got = runs[label]
        assert (p.kernel, p.fallback, p.grid, p.block, p.fold_grid, p.fold_rounds) == \
            (got["kernel"], got["fallback"], got["grid"], got["block"], got["fold_grid"], got["fold_rounds"]), label
        if p.kernel == "tma":
            assert (p.depth, p.chunk_elems, p.n_chunks, p.smem) == \
                (got["depth"], got["chunk_elems"], got["n_chunks"], got["smem"])


GRIDS = [1, 132, 264, 1056]


@pytest.mark.parametrize("grid", GRIDS)
def test_row_split_at_the_series_limit(emul, grid):
    """cta_row_count: CTA b owns rows b, b + grid, ...  For every total up to the 2^32 - 2 rows of a window at the
    series limit with a power plane, the shares add up to the total and differ by at most one row."""
    totals = sorted({0, 1, grid - 1, grid, grid + 1, 2**31 - 1, 2**32 - grid, 0xFFFFFFFE})
    r = subprocess.run([emul, "--rowsplit", str(grid)] + [str(t) for t in totals], capture_output=True, text=True,
                       check=True, timeout=60)
    lines = r.stdout.split("\n")[:len(totals)]
    for t, l in zip(totals, lines):
        g, total, s, lo, hi = (int(x) for x in l.split())
        assert (g, total) == (grid, t)
        assert s == t and hi - lo <= 1, (grid, t, s, lo, hi)


def test_multi_round_fold_under_thread_sanitizer(tmp_path):
    """a fold grid that loops (4 rounds on 2 SMs with 64-thread CTAs) and an LDG grid of full width, under
    ThreadSanitizer: the fold's per-round clears of the masks, the ticket, the counters"""
    exe = _build(tmp_path, sanitize="thread")
    rng = np.random.default_rng(5)
    P, G, T = 1555, 1, 8
    util, kw, elig, _ = _window(rng, P, G, T, True)
    d = tmp_path / "fold4"
    _write_case(str(d), util, kw["power"], kw["thr"], elig)
    knobs = K(2, 4, 512, 2, 2, 64)
    _write_knobs(str(d), knobs, "ldg,tma")
    env = dict(os.environ, TSAN_OPTIONS="halt_on_error=1")
    r = subprocess.run([exe, str(d)], capture_output=True, text=True, timeout=1800, env=env)
    assert r.returncode == 0 and "ThreadSanitizer" not in r.stderr, r.stderr[-3000:]
    lines = r.stdout.splitlines()
    assert len(lines) == 4
    assert all(_plan_of(l.split()[-1])["fold_rounds"] >= 4 for l in lines)
    assert all(l.split()[2] == "clean" for l in lines)


def test_both_tma_layout_definitions_are_the_same():
    """TmaLayout is defined in gpr_launch.h and, under the same guard, in gpr_kernels.cuh's namespace body (which the
    emulation compiles alone): the two must not drift apart"""
    import re
    csrc = os.path.join(ROOT, "gpu-pruner_b200", "csrc")
    blocks = []
    for name in ("gpr_launch.h", "gpr_kernels.cuh"):
        m = re.search(r"#ifndef GPR_TMA_LAYOUT_DEFINED\n.*?#endif\n", open(os.path.join(csrc, name)).read(), re.S)
        assert m, name
        blocks.append(m.group(0))
    assert blocks[0] == blocks[1]
