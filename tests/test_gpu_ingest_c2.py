"""GPU, slow: the `gpu-pruner` binary in daemon mode on a C2-sized response, its verdicts checked tick by tick.

tests/cpp/c2_response.cpp renders DESIGN.md §7's synthetic universe (10,000 pods x 4 GPUs, the oracle's own cells) as
Prometheus' compact matrix JSON, util and power: tick 0 is the full 30-minute range (about 1.25 GB per response,
40,000 series, some 600 upload chunks), ticks 1-3 the 180 s scraped since the tick before.  This is the run bench.py
times (tools/daemon_ticks_bench.py); here each tick's `Query returned` line and the set of pods it would scale must
equal oracle_c on the matching 1,800 columns of the universe, and every tick must stay on the device."""
import json
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

import hostlib as H

pytestmark = [pytest.mark.gpu, pytest.mark.slow]

torch = pytest.importorskip("torch")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GB = 1 << 30
SEED, P, G, W, NEW, TICKS = 0x5EED0002, 10000, 4, 1800, 180, 4
T_TOTAL = W + NEW * (TICKS - 1)
NOW = 1_700_000_000
T0 = NOW - T_TOTAL - 600           # column c is unix time T0 + c
THR = 150.0


def _build(out_dir):
    exe = os.path.join(str(out_dir), "c2_response")
    oracle = os.path.join(ROOT, "oracle")
    subprocess.check_call(["g++", "-O2", "-std=c++17", os.path.join(ROOT, "tests", "cpp", "c2_response.cpp"),
                           "-L", oracle, "-lgpr_oracle", "-Wl,-rpath," + oracle, "-o", exe])
    return exe


def _fixtures(exe, root):
    """tick-%04d/{full,delta}/{util,power,query}.json; -> the end time of every tick"""
    ends = []
    for k in range(TICKS):
        hi = W + NEW * k                    # columns [hi - W, hi) are tick k's window
        t_end = T0 + hi - 1
        ends.append(t_end)
        kind, lo = ("full", hi - W) if k == 0 else ("delta", hi - NEW)
        d = os.path.join(root, "tick-%04d" % k, kind)
        os.makedirs(d)
        for name, plane in (("util.json", 0), ("power.json", 1)):
            subprocess.check_call([exe, os.path.join(d, name), str(plane), str(SEED), str(P), str(G), str(T_TOTAL),
                                   str(T0), str(lo), str(hi)])
        q = {"end": t_end, "step": 1}
        if kind == "delta":
            q["start"] = t_end - NEW
        with open(os.path.join(d, "query.json"), "w") as f:
            json.dump(q, f)
    return ends


def _expected(oracle_c, u, w, k):
    """oracle_c on tick k's 1,800 columns, each series its own `sum by` element: (n_series, idle pod names)"""
    cols = slice(NEW * k, NEW * k + W)
    r = oracle_c.decide(u[:, :, cols], w[:, :, cols], power_threshold=THR, n_threads=os.cpu_count() or 1)
    cand = np.unpackbits(r["candidate_bits"].view(np.uint8), bitorder="little")[:P].astype(bool)
    return r["n_series"], {(f"pod-{p}", f"ns-{p % 64}") for p in np.flatnonzero(cand)}


def test_c2_daemon_ticks_decide_like_the_oracle(tmp_path, oracle_c):
    from test_gpu_promql import _kube
    free_disk = shutil.disk_usage(str(tmp_path)).free
    if free_disk < 4 * GB:
        pytest.skip(f"the fixtures need about 3 GB of disk, {free_disk / GB:.1f} GB free")
    free, _ = torch.cuda.mem_get_info()
    if free < 8 * GB:
        pytest.skip(f"needs 8 GB of device memory, {free / GB:.1f} GB free")
    exe = _build(tmp_path)
    root = tmp_path / "prom"
    ends = _fixtures(exe, str(root))
    full = os.path.getsize(root / "tick-0000" / "full" / "util.json")
    assert full > 1.1e9, full
    _kube(tmp_path / "kube", [(f"pod-{p}", f"ns-{p % 64}") for p in range(P)])
    cmd = [H.BIN, "--prometheus-url", f"file://{root}", "--kube-fixture", str(tmp_path / "kube"), "-d", "-c", "0",
           "--max-ticks", str(TICKS), "-t", str(W // 60), "-g", "300", "--now", str(NOW), "-l", "json",
           "--power-threshold", "150"]
    p = subprocess.run(cmd, capture_output=True, text=True, timeout=3000)
    assert p.returncode == 0, p.stderr[-3000:]
    msgs = [json.loads(l)["fields"]["message"] for l in p.stderr.splitlines() if l.startswith("{")]
    # the messages of each tick: from its ingest note to the next one
    starts = [i for i, m in enumerate(msgs) if m.startswith("Device ingest")]
    assert len(starts) == TICKS, [m for m in msgs if m.startswith("Device ingest")]
    u = oracle_c.synth_fill(SEED, 0, 0, P, G, T_TOTAL)
    w = oracle_c.synth_fill(SEED, 1, 0, P, G, T_TOTAL)
    assert np.isnan(u).any() and (np.nan_to_num(u) == 0).all(axis=2).any()
    for k in range(TICKS):
        tick = msgs[starts[k]:starts[k + 1] if k + 1 < TICKS else len(msgs)]
        note = tick[0]
        assert note.startswith("Device ingest: ") and "(0 re-parsed on the CPU, 0 rows patched" in note, (k, note)
        if k == 0:
            assert "parsed on the GPU into a resident" in note, note
        else:
            assert "of the last 180 s appended to the resident 10000x4x1800 window" in note, (k, note)
        n_series, pods = _expected(oracle_c, u, w, k)
        verdict = [m for m in tick if m.startswith("Query returned")]
        assert verdict == [f"Query returned {n_series} series across {len(pods)} unique pods"], (k, verdict)
        sent = {(m.group(2), m.group(1)) for m in (re.match(r"Dry-run: Would have sent \[Deployment\] ([^:]+):dep-(\S+) for scaledown", x)
                                                   for x in tick) if m}
        assert sent == pods, (k, len(sent), len(pods), sorted(sent ^ pods)[:8])
        print(f"\n[c2 tick {k}] t_end {ends[k]}: {n_series} idle series, {len(pods)} pods would be scaled; {note[:120]}")
