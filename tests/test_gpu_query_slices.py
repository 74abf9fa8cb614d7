"""GPU: `gpu-pruner --query-slice S` — ranges longer than S seconds asked as consecutive queries and merged into the
resident window on the GPU (DESIGN.md §8e).  The scenarios of tests/test_gpu_daemon.py and of the churn run of
tests/test_gpu_daemon_reshape.py, recorded also as slices, run through the binary at two slice lengths: every verdict
line equals the oracle's on a fresh full-range ingest of its tick and the line of the unsliced run, and each run takes
the unsliced run's path.  The CPU run of the same rule on an emulated device is tests/test_query_slices.py."""
import json
import subprocess

import pytest

import hostlib as H
import slice_ticks as ST
import test_gpu_daemon as D
import test_gpu_daemon_reshape as R
import ticks as TK

pytestmark = pytest.mark.gpu


def _recorded(monkeypatch, S, make, *args):
    """make(*args) with every range also recorded as the slices --query-slice S asks for"""
    with monkeypatch.context() as m:
        m.setattr(TK, "write_ticks", lambda root, store_at, times, N, step, **kw:
                  ST.write_sliced_ticks(root, store_at, times, N, step, S, **kw))
        return make(*args)


def _run(root, n, dur, *extra):
    cmd = [H.BIN, "--prometheus-url", f"file://{root}", "-d", "-c", "0", "--max-ticks", str(n), "-t", str(dur),
           "-l", "json", *extra]
    p = subprocess.run(cmd, capture_output=True, text=True, timeout=900)
    assert p.returncode == 0, p.stderr[-3000:]
    return [json.loads(l)["fields"]["message"] for l in p.stderr.splitlines() if l.startswith("{")]


def _check(root, n, dur, thr, oracle_np, S, *extra):
    plain = _run(root, n, dur, *extra)
    sliced = _run(root, n, dur, *extra, "--query-slice", str(S))
    v = lambda ms: [m for m in ms if m.startswith("Query returned")]
    assert v(sliced) == v(plain) and len(v(plain)) == n
    for k, line in enumerate(v(sliced)):
        n_series, n_pods = D._expected(root, k, dur, thr, oracle_np)
        assert line == f"Query returned {n_series} series across {n_pods} unique pods", (k, line)
    assert any("query slices" in m for m in sliced if m.startswith("Device ingest")), sliced
    assert not any(m.startswith("Failed") or "query_failures" in m for m in sliced)
    # the same path: a tick that rebuilt unsliced rebuilds sliced, and the other way round
    rebuilt = lambda ms: [m.split(": ", 1)[1] for m in ms if m.startswith("Resident window rebuilt")]
    assert rebuilt(sliced) == rebuilt(plain)
    return sliced


@pytest.mark.parametrize("S", [10, 34])
@pytest.mark.parametrize("power", [False, True], ids=["util", "util+power"])
def test_daemon_scenario_sliced(tmp_path, monkeypatch, power, S, oracle_np):
    root, n, dur = _recorded(monkeypatch, S, D._scenario, tmp_path, 4 + power, power)
    extra = ("--power-threshold", "150") if power else ()
    msgs = _check(root, n, dur, 150.0 if power else None, oracle_np, S, *extra)
    notes = [m for m in msgs if m.startswith("Device ingest")]
    assert sum(f"{-(-120 // S)} query slices" in m for m in notes) == 3, notes   # ticks 0, 6 and 7 take the full range


@pytest.mark.parametrize("S", [10, 34])
def test_churn_scenario_sliced_with_reshape(tmp_path, monkeypatch, S, oracle_np):
    root, n, dur = _recorded(monkeypatch, S, R._churn, tmp_path)
    _check(root, n, dur, None, oracle_np, S, "--reshape-ring")
    _check(root, n, dur, None, oracle_np, S)


def test_one_shot_sliced(tmp_path, monkeypatch, oracle_np):
    """one-shot mode (no -d): the full range asked as slices and decided on the resident ring"""
    root, n, dur = _recorded(monkeypatch, 20, D._scenario, tmp_path, 4, False)
    cmd = [H.BIN, "--prometheus-url", f"file://{root}", "-t", str(dur), "-l", "json"]
    out = []
    for extra in ((), ("--query-slice", "20")):
        p = subprocess.run(cmd + list(extra), capture_output=True, text=True, timeout=600)
        assert p.returncode == 0, p.stderr[-3000:]
        out.append([json.loads(l)["fields"]["message"] for l in p.stderr.splitlines() if l.startswith("{")])
    v = lambda ms: [m for m in ms if m.startswith("Query returned")]
    assert v(out[0]) == v(out[1]) and len(v(out[1])) == 1
    n_series, n_pods = D._expected(root, 0, dur, None, oracle_np)
    assert v(out[1])[0] == f"Query returned {n_series} series across {n_pods} unique pods"
    assert any("6 query slices" in m for m in out[1]), out[1]


# ---- snapshots after a sliced cold start, a restore followed by a long sliced delta, a declined row in a middle slice
def _gap_scenario(root, S):
    """tests/test_gpu_daemon.py's cluster with a power plane, a PROF series that shadows its UTIL series, a series whose
    values the device declines (1e+23) only in the middle of the window, and 100 s without a tick after tick 1"""
    import random
    from test_resident_ticks import _series
    rng = random.Random(61)
    N, step, dur = 120, 2, 2
    t0 = 1_700_000_000
    times = [t0 + N, t0 + N + 30, t0 + N + 130, t0 + N + 160, t0 + N + 190]
    horizon = times[-1] + 5
    store = [_series(rng, f"pod-{p}", g, t0, horizon, step, rng.choice(["idle", "idle", "busy"])) for p in range(40)
             for g in range(2)]
    store.append(("DCGM_FI_PROF_GR_ENGINE_ACTIVE", store[0][1], [(t, 0.0) for t in range(t0, horizon, step)]))
    store.append(("DCGM_FI_DEV_GPU_UTIL", TK.labels("odd", 0),
                  [(t, 1e23 if times[0] - 70 < t <= times[0] - 40 else 0) for t in range(t0, horizon, step)]))
    store += [_series(rng, f"pod-{p}", 0, t0, horizon, step, "x", metric="DCGM_FI_DEV_POWER_USAGE") for p in range(40)]
    ST.write_sliced_ticks(str(root), lambda k: store, times, N, step, S, with_power=True)
    return str(root), len(times), dur


def test_snapshot_after_a_sliced_cold_start_and_a_restore(tmp_path, oracle_np):
    """the snapshot after a sliced cold start holds the unsliced run's ring and session by series identity (the row the
    device declined in a middle slice included: it is patched in that slice's buckets); a process restarted from it
    asks its first, 100 s delta as slices and decides as the uninterrupted unsliced run does"""
    import snapshot_identity as SI
    from test_gpu_daemon_snapshot import _renumbered
    S, thr = 10, ("--power-threshold", "150")
    root, n, dur = _gap_scenario(tmp_path / "ticks", S)
    full = _run(root, n, dur, *thr)
    v = lambda ms: [m for m in ms if m.startswith("Query returned")]
    for k, line in enumerate(v(full)):
        assert line == "Query returned %d series across %d unique pods" % D._expected(root, k, dur, 150.0, oracle_np)
    one = _run(root, 1, dur, *thr, "--snapshot-file", str(tmp_path / "snap-one"))
    sl = _run(root, 1, dur, *thr, "--query-slice", str(S), "--snapshot-file", str(tmp_path / "snap-sliced"))
    note = [m for m in sl if m.startswith("Device ingest")][0]
    assert "12 query slices" in note and " 0 re-parsed on the CPU" not in note, note
    assert v(one) == v(sl) == v(full)[:1]
    assert SI.mismatch(open(tmp_path / "snap-one", "rb").read(), open(tmp_path / "snap-sliced", "rb").read()) == ""
    for cut in (1, 2):
        broot, nb = _renumbered(root, cut, tmp_path / f"b{cut}")
        snap = tmp_path / f"snap-{cut}"
        _run(root, cut, dur, *thr, "--query-slice", str(S), "--snapshot-file", str(snap))
        b = _run(broot, nb, dur, *thr, "--query-slice", str(S), "--snapshot-file", str(snap))
        assert any(m.startswith("Snapshot restored from") for m in b)
        assert v(b) == v(full)[cut:]
        first = [m for m in b if m.startswith("Device ingest")][0]
        if cut == 2:   # saved after tick 1, restarted at tick 2: the 100 s gap, 10 slices into the restored ring
            assert "10 query slices over the last 100 s" in first, first
        else:          # saved after tick 0: tick 1's 30 s delta is three 10 s slices
            assert "3 query slices over the last 30 s" in first, first


def test_c2_cold_start_sliced_at_180s_equals_one_query(tmp_path):
    """10,000 pods x 4 GPUs x 1,800 s: the cold start as one query and as ten 180 s slices leave the same ring and
    session (their snapshots compared by series identity) and the same verdict"""
    import ctypes as C
    import os
    import sys
    import snapshot_identity as SI
    sys.path.insert(0, os.path.join(H.ROOT, "tools"))
    import slice_bench as SB
    lib = H.lib()
    lib.gph_synth_response.restype = C.c_longlong
    q = SB.fixtures(lib, str(tmp_path / "c2"), 10000, 4, 1800, 180)
    assert q["slices"] == 10 and q["largest_slice"]["samples"] == 7_200_000
    one = SB.binary(H, str(tmp_path / "c2"), 1800, 0, str(tmp_path / "snap-one"))
    sl = SB.binary(H, str(tmp_path / "c2"), 1800, 180, str(tmp_path / "snap-sliced"))
    assert one["verdict"] == sl["verdict"] and len(one["verdict"]) == 1
    assert any("10 query slices" in m for m in sl["ingest"]), sl["ingest"]
    assert SI.mismatch(open(tmp_path / "snap-one", "rb").read(), open(tmp_path / "snap-sliced", "rb").read()) == ""
