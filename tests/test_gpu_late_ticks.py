"""GPU: `gpu-pruner -d --late-seconds L` on a server whose samples arrive late (tests/late_ticks.py).  Some pods' only busy
sample reaches the server up to 75 s after its timestamp (step 30 s, a tick every 60 s): it lands behind the previous
tick's query, so a delta that starts where the resident window ends never sees it and the pod reads idle.
  * with --late-seconds 90 every verdict line equals the oracle's on that tick's full/ window, and the late-cell lines
    match the model — plain, with --query-slice, with --reshape-ring (a pod gains a slot on the way), and cut by a
    snapshot at a tick and resumed;
  * with --late-seconds 0 at least one verdict differs, on a tick where the model loses a busy sample;
  * with --late-seconds 45 (not a multiple of the step) and samples lagged 30-40 s every verdict still equals the
    oracle's."""
import random
import re

import pytest

import late_ticks as LT
import ticks as TK
from test_gpu_daemon import _expected, _run

pytestmark = pytest.mark.gpu

STEP, INTERVAL, DUR = 30, 60, 10
WINDOW = DUR * 60
T0 = 1_700_000_000
TIMES = [T0 + WINDOW + k * INTERVAL for k in range(9)]


def _scenario(seed, lag_lo, lag_hi, d_hi, grow=False):
    """16 pods: 6 whose only busy sample is late (one per delta tick, lagged lag_lo..lag_hi s, d s before the previous
    tick), 8 idle, 2 busy on time; every other sample lags 0-10 s.  grow: pod-15 gains a second GPU at tick 5."""
    rng = random.Random(seed)
    series = []
    horizon = TIMES[-1]
    late_ticks = {}
    for p in range(16):
        samples = []
        t = T0 + rng.randrange(1, 15)
        while t <= horizon:
            samples.append([t, 40 if p >= 14 else 0, rng.uniform(0, 10)])
            t += 15
        if p < 6:
            k = 1 + p
            d = rng.randrange(5, d_hi)
            ts = TIMES[k - 1] - d
            samples.append([ts, 60, rng.uniform(max(lag_lo, d + 1), lag_hi)])
            samples.sort()
            late_ticks[p] = k
        series.append(("DCGM_FI_DEV_GPU_UTIL", TK.labels(f"pod-{p}", 0), [tuple(s) for s in samples]))
    if grow:
        extra = [(t, 0, 0.0) for t in range(TIMES[4] + 7, horizon + 1, 15)]
        series.append(("DCGM_FI_DEV_GPU_UTIL", TK.labels("pod-15", 1), extra))
    return LT.LateStore(series), late_ticks


def _verdicts(msgs):
    return [m for m in msgs if m.startswith("Query returned")]


def _late_lines(msgs):
    pat = re.compile(r"Late samples raised (\d+) util cells and (\d+) power cells in the re-asked (\d+) s")
    return [tuple(int(x) for x in m.groups()) for m in map(pat.match, msgs) if m]


def _check_run(root, late, msgs, L, oracle_np, first=0, check_cells=True):
    verdicts = _verdicts(msgs)
    assert len(verdicts) == len(TIMES) - first
    for k, v in enumerate(verdicts):
        n_series, n_pods = _expected(root, k, DUR, None, oracle_np)
        assert v == f"Query returned {n_series} series across {n_pods} unique pods", (k, v)
    assert not any("does not continue" in m or "rebuilt from the full range" in m for m in msgs), msgs
    if check_cells:
        want = [n for n in LT.late_cells(late, TIMES, WINDOW, STEP, L)[first:] if n]
        assert _late_lines(msgs) == [(n, 0, L) for n in want]
        assert want


@pytest.mark.parametrize("extra", [(), ("--query-slice", "120"), ("--reshape-ring",)], ids=["plain", "slices", "reshape"])
def test_late_seconds_90_equals_fresh_queries(tmp_path, extra, oracle_np):
    late, _ = _scenario(11, 60, 75, 50, grow=extra == ("--reshape-ring",))
    S = int(extra[1]) if extra and extra[0] == "--query-slice" else 0
    root = LT.write_late_ticks(str(tmp_path), late, TIMES, WINDOW, STEP, 90, S=S)
    msgs = _run(root, len(TIMES), DUR, "--late-seconds", "90", *extra)
    _check_run(root, late, msgs, 90, oracle_np)
    ingests = [m for m in msgs if m.startswith("Device ingest")]
    assert all("re-asked the newest 90 s" in m for m in ingests[1:]), ingests
    if extra == ("--reshape-ring",):
        assert any(m.startswith("Resident window reshaped on the GPU") for m in msgs)


def test_late_seconds_90_across_a_snapshot(tmp_path, oracle_np):
    late, _ = _scenario(12, 60, 75, 50)
    cut = 4
    a = LT.write_late_ticks(str(tmp_path / "a"), late, TIMES[:cut], WINDOW, STEP, 90)
    b = LT.write_late_ticks(str(tmp_path / "b"), late, TIMES[cut:], WINDOW, STEP, 90, prev=TIMES[cut - 1])
    snap = str(tmp_path / "snap")
    m1 = _run(a, cut, DUR, "--late-seconds", "90", "--snapshot-file", snap)
    m2 = _run(b, len(TIMES) - cut, DUR, "--late-seconds", "90", "--snapshot-file", snap)
    assert any(m.startswith("Snapshot restored") for m in m2), m2
    for root, msgs, first in ((a, m1, 0), (b, m2, cut)):
        verdicts = _verdicts(msgs)
        for k, v in enumerate(verdicts):
            n_series, n_pods = _expected(root, k, DUR, None, oracle_np)
            assert v == f"Query returned {n_series} series across {n_pods} unique pods", (first + k, v)
    want = [n for n in LT.late_cells(late, TIMES, WINDOW, STEP, 90) if n]
    assert _late_lines(m1) + _late_lines(m2) == [(n, 0, 90) for n in want] and want


def test_late_seconds_0_misses_late_samples(tmp_path, oracle_np):
    late, late_ticks = _scenario(11, 60, 75, 50)
    root = LT.write_late_ticks(str(tmp_path), late, TIMES, WINDOW, STEP, 0)
    msgs = _run(root, len(TIMES), DUR, "--late-seconds", "0")
    verdicts = _verdicts(msgs)
    differ = [k for k, v in enumerate(verdicts)
              if v != "Query returned %d series across %d unique pods" % _expected(root, k, DUR, None, oracle_np)]
    assert differ and set(differ) <= set(range(min(late_ticks.values()), len(TIMES))), differ
    assert not _late_lines(msgs) and not any("re-asked" in m for m in msgs)


def test_late_seconds_45_not_a_multiple_of_the_step(tmp_path, oracle_np):
    late, _ = _scenario(13, 30, 40, 25)
    root = LT.write_late_ticks(str(tmp_path), late, TIMES, WINDOW, STEP, 45)
    msgs = _run(root, len(TIMES), DUR, "--late-seconds", "45")
    _check_run(root, late, msgs, 45, oracle_np)
