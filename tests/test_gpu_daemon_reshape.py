"""GPU: `gpu-pruner -d --reshape-ring` — daemon mode whose resident window is reshaped on the GPU (gpr_resident_live_rows +
gpr_resident_remap) when pods outgrow its rows or a pod gains a series slot beyond its G, instead of being rebuilt from
the full range.  The scenario of tests/test_gpu_daemon.py with the flag: the third-slot tick (6) is appended to the
resident window after a reshape, and only the tick without a slice (7) rebuilds.  Every verdict line equals the
oracle's on a fresh full-range ingest of its tick and the line of the same run without the flag.  A churn scenario that
used to run out of rows every few ticks never rebuilds, and a --snapshot-file run cut right after one of its reshaping
ticks resumes onto the uninterrupted run's path, verdicts, ring and session.  The CPU run of the same rule on an emulated device is
tests/test_resident_reshape.py."""
import json
import random
import subprocess

import numpy as np
import pytest

import hostlib as H
import snapshot_ref as SR
import ticks as TK
from test_gpu_daemon import _expected, _scenario
from test_gpu_daemon_snapshot import _renumbered
from test_resident_ticks import _series

pytestmark = pytest.mark.gpu


def _run(root, n_ticks, duration_min, *extra):
    cmd = [H.BIN, "--prometheus-url", f"file://{root}", "-d", "-c", "0", "--max-ticks", str(n_ticks), "-t",
           str(duration_min), "-l", "json", *extra]
    p = subprocess.run(cmd, capture_output=True, text=True, timeout=900)
    assert p.returncode == 0, p.stderr[-3000:]
    return [json.loads(l)["fields"] for l in p.stderr.splitlines() if l.startswith("{")]


def _check(root, n, dur, thr, oracle_np, *extra):
    """runs the binary with and without --reshape-ring: every verdict line equals the oracle's and the other run's.
    Returns (the flagged run's log fields, its per-tick "appended to the resident" list)."""
    plain = _run(root, n, dur, *extra)
    fields = _run(root, n, dur, *extra, "--reshape-ring")
    verdicts = [f["message"] for f in fields if f["message"].startswith("Query returned")]
    assert verdicts == [f["message"] for f in plain if f["message"].startswith("Query returned")]
    assert len(verdicts) == n
    for k, v in enumerate(verdicts):
        n_series, n_pods = _expected(root, k, dur, thr, oracle_np)
        assert v == f"Query returned {n_series} series across {n_pods} unique pods", (k, v)
    ingests = [f["message"] for f in fields if f["message"].startswith("Device ingest")]
    return fields, ["appended to the resident" in m for m in ingests]


@pytest.mark.parametrize("power", [False, True], ids=["util", "util+power"])
def test_third_slot_tick_is_appended_after_a_reshape(tmp_path, power, oracle_np):
    root, n, dur = _scenario(tmp_path, 4 + power, power)
    thr = 150.0 if power else None
    extra = ("--power-threshold", "150") if power else ()
    fields, appended = _check(root, n, dur, thr, oracle_np, *extra)
    assert appended == [False, True, True, True, True, True, True, False, True]
    shaped = [f for f in fields if f["message"].startswith("Resident window reshaped on the GPU:")]
    assert len(shaped) == 1 and ", 2 -> 3, " in shaped[0]["message"], shaped
    assert shaped[0].get("monotonic_counter.ring_reshapes") == "1"
    rebuilt = [f["message"] for f in fields if f["message"].startswith("Resident window rebuilt from the full range")]
    assert len(rebuilt) == 0   # tick 7 has no slice at all: it takes the full range without a delta attempt


def _churn(root):
    """40 pods x 2 GPUs that stay, and 30 short-lived pods per tick: 300 names over a cluster of about 100 pods"""
    rng = random.Random(8)
    N, step, interval, dur = 120, 2, 30, 2
    t0 = 1_700_000_000
    times = [t0 + N + k * interval for k in range(10)]
    horizon = times[-1] + 5
    store = [_series(rng, f"stay-{p}", g, t0, horizon, step, rng.choice(["idle", "busy"])) for p in range(40)
             for g in range(2)]
    for k, t in enumerate(times):
        store += [_series(rng, f"nb-{k}-{j}", 0, t - interval + 1, t + 2, step, rng.choice(["idle", "busy"]))
                  for j in range(30)]
    TK.write_ticks(str(root), lambda k: store, times, N, step)
    return str(root), len(times), dur


def test_churn_that_used_to_exhaust_the_rows_never_rebuilds(tmp_path, oracle_np):
    root, n, dur = _churn(tmp_path)
    plain = _run(root, n, dur)
    assert any(f["message"].startswith("Resident window rebuilt from the full range: more pods") for f in plain)
    fields, appended = _check(root, n, dur, None, oracle_np)
    assert appended == [False] + [True] * (n - 1)
    shaped = [f["message"] for f in fields if f["message"].startswith("Resident window reshaped on the GPU:")]
    assert shaped and any(int(m.split(", ")[2].split()[0]) > 0 for m in shaped), shaped


def _same_snapshot(a, b):
    """two snapshots hold the same window and session: every field, the known series in any order (the file lists them
    in the order of the session's hash table), the planes' chunks byte for byte"""
    x, y = (SR.read(open(p, "rb").read()) for p in (a, b))
    for k in x:
        if k in ("sections", "planes"):
            continue
        assert (sorted(x[k]) if k in ("known", "prof_sigs") else x[k]) == \
            (sorted(y[k]) if k in ("known", "prof_sigs") else y[k]), k
    assert len(x["planes"]) == len(y["planes"])
    for p, q in zip(x["planes"], y["planes"]):
        for k in ("series_chunks", "rows", "chunk_bytes", "data"):
            assert np.array_equal(p[k], q[k]), k


def test_snapshot_cut_right_after_a_reshaping_tick(tmp_path):
    """--snapshot-file after a tick that reshaped and dropped pods stores the new shape in the unchanged format; a process
    restarted on the next ticks restores it (its checks hold for the compacted session), takes the uninterrupted run's
    path and verdicts, and ends with the same ring and session in its snapshot"""
    root, n, dur = _churn(tmp_path / "ticks")
    u = _run(root, n, dur, "--reshape-ring", "--snapshot-file", str(tmp_path / "snap-u"))
    tick, cut = 0, None
    for f in u:
        m = f["message"]
        if m.startswith("Query returned"):
            tick += 1
        elif m.startswith("Resident window reshaped on the GPU:") and int(m.split(", ")[2].split()[0]) > 0:
            cut = tick + 1          # the snapshot written after this tick
            break
    assert cut is not None and cut < n, [f["message"] for f in u if "reshaped" in f["message"]]
    a = _run(root, cut, dur, "--reshape-ring", "--snapshot-file", str(tmp_path / "snap"))
    assert sum(f["message"].startswith("Resident window reshaped on the GPU:") for f in a) >= 1
    doc = SR.read(open(tmp_path / "snap", "rb").read())
    assert doc["pods_cap"] >= len(doc["pods"]) and doc["G"] >= 1
    broot, nb = _renumbered(root, cut, tmp_path / "b")
    b = _run(broot, nb, dur, "--reshape-ring", "--snapshot-file", str(tmp_path / "snap"))
    assert any(f["message"].startswith("Snapshot restored from") for f in b)
    verdicts = lambda fs: [f["message"] for f in fs if f["message"].startswith("Query returned")]
    assert verdicts(b) == verdicts(u)[cut:]
    ingests = [f["message"] for f in b if f["message"].startswith("Device ingest")]
    assert all("appended to the resident" in m for m in ingests), ingests
    _same_snapshot(tmp_path / "snap", tmp_path / "snap-u")
