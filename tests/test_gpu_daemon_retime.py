"""GPU: `gpu-pruner -d --retime-ring` — daemon mode whose resident window is retimed on the GPU (gpr_resident_retime) when
the query step doubles at one tick, or when a process restarts from the --snapshot-file of a longer window into a
shorter --duration, instead of being rebuilt from the full range.  Plain, with --query-slice and with --late-seconds.
Every verdict line equals the oracle's on a fresh full-range ingest of its tick at that tick's step and duration, and
the line of the same run without the flag; the retime's log line and counter appear.  The CPU run of the same rule on an
emulated device is tests/test_resident_retime.py."""
import json
import random
import subprocess

import pytest

import hostlib as H
import retime_ticks as RT
from test_gpu_daemon import _expected
from test_gpu_daemon_snapshot import _renumbered
from test_resident_ticks import _series

pytestmark = pytest.mark.gpu

T0 = 1_700_000_000
RETIMED = "Resident window retimed on the GPU:"
MODES = [((), 0, 0), (("--query-slice", "20"), 20, 0), (("--late-seconds", "15"), 0, 15)]
IDS = ["plain", "query-slice", "late-seconds"]


def _run(root, n_ticks, duration_min, *extra):
    cmd = [H.BIN, "--prometheus-url", f"file://{root}", "-d", "-c", "0", "--max-ticks", str(n_ticks), "-t",
           str(duration_min), "-l", "json", *extra]
    p = subprocess.run(cmd, capture_output=True, text=True, timeout=900)
    assert p.returncode == 0, p.stderr[-3000:]
    return [json.loads(l)["fields"] for l in p.stderr.splitlines() if l.startswith("{")]


def _verdicts(fields):
    return [f["message"] for f in fields if f["message"].startswith("Query returned")]


def _want(root, ticks, durations, oracle_np, thr=150.0):
    return ["Query returned %d series across %d unique pods" % _expected(root, k, durations[k], thr, oracle_np)
            for k in ticks]


def _timeline(root, steps, durations, L, S):
    rng = random.Random(17)
    times = [T0 + 120 + k * 40 for k in range(len(steps))]
    horizon = times[-1] + 5
    store = [_series(rng, f"pod-{p}", g, T0 - 50, horizon, 5, rng.choice(["idle", "busy"]))
             for p in range(12) for g in range(1 + p % 2)]
    store += [_series(rng, f"pod-{p}", 0, T0 - 50, horizon, 5, "x", metric="DCGM_FI_DEV_POWER_USAGE") for p in range(12)]
    RT.write_retime_ticks(str(root), store, times, steps, durations, L=L, S=S, power=True)
    return str(root)


@pytest.mark.parametrize("extra,S,L", MODES, ids=IDS)
def test_step_doubled_at_one_tick(tmp_path, oracle_np, extra, S, L):
    steps, durations = [5, 5, 5, 10, 10, 10], [2] * 6
    root = _timeline(tmp_path, steps, durations, L, S)
    n = len(steps)
    common = ("--power-threshold", "150") + extra
    plain = _run(root, n, 2, *common)
    fields = _run(root, n, 2, *common, "--retime-ring")
    assert _verdicts(fields) == _verdicts(plain) == _want(root, range(n), durations, oracle_np)
    retimed = [f for f in fields if f["message"].startswith(RETIMED)]
    assert len(retimed) == 1 and retimed[0]["message"].startswith(RT.retime_line(24, 5, 120, 10, 120)), retimed
    assert retimed[0].get("monotonic_counter.ring_retimes") == "1"
    assert not any(f["message"].startswith(RETIMED) for f in plain)
    assert any("step / window length changed" in f["message"] for f in plain)
    assert not any("Resident window rebuilt from the full range" in f["message"] for f in fields)


@pytest.mark.parametrize("extra,S,L", MODES, ids=IDS)
def test_restart_into_a_shorter_duration(tmp_path, oracle_np, extra, S, L):
    """a process at --duration 2 writes its snapshot after tick 2; the next one starts at --duration 1 on ticks 3..: with
    the flag it restores the longer window and its first delta retimes it, without it the snapshot is refused"""
    steps, durations, cut = [5] * 6, [2, 2, 2, 1, 1, 1], 3
    root = _timeline(tmp_path / "ticks", steps, durations, L, S)
    common = ("--power-threshold", "150") + extra
    for flag in ((), ("--retime-ring",)):
        snap = str(tmp_path / ("snap" + "".join(flag)))
        a = _run(root, cut, 2, *common, *flag, "--snapshot-file", snap)
        assert _verdicts(a) == _want(root, range(cut), durations, oracle_np)
        broot, nb = _renumbered(root, cut, tmp_path / ("b" + "".join(flag)))
        b = _run(broot, nb, 1, *common, *flag, "--snapshot-file", snap)
        assert _verdicts(b) == _want(root, range(cut, cut + nb), durations, oracle_np)
        msgs = [f["message"] for f in b]
        if flag:
            assert any(m.startswith("Snapshot restored from") for m in msgs), [m for m in msgs if "Snapshot" in m]
            retimed = [f for f in b if f["message"].startswith(RETIMED)]
            assert len(retimed) == 1 and retimed[0]["message"].startswith(RT.retime_line(24, 5, 120, 5, 60))
            assert retimed[0].get("monotonic_counter.ring_retimes") == "1"
            assert not any("Resident window rebuilt from the full range" in m for m in msgs)
        else:
            assert any("fingerprint mismatch: window of 120 s, now 60 s" in m for m in msgs), msgs
            assert not any(m.startswith(RETIMED) for m in msgs)
