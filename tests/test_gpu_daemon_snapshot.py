"""GPU: `gpu-pruner -d --snapshot-file` across a restart (DESIGN.md §8i), on the scenario of tests/test_gpu_daemon.py.
Process A runs ticks 0..k-1 and snapshots the resident window after every tick; process B, started on the ticks k..
(renumbered from tick-0000), restores it and asks only for the slice since the snapshot.  B's verdicts must equal the
uninterrupted run's and the oracle's on a fresh full-range query.  A snapshot that is damaged or missing costs the
full range, never a verdict; a snapshot that cannot be written costs nothing but an error line."""
import json
import os
import shutil
import subprocess

import numpy as np
import pytest

import export_ref as XR
import hostlib as H
import snapshot_ref as SR
from test_gpu_daemon import _expected, _run, _scenario

pytestmark = pytest.mark.gpu

CUTS = (1, 3, 5, 8)


def _verdicts(msgs):
    return [m for m in msgs if m.startswith("Query returned")]


def _renumbered(root, k, dest):
    """the ticks k.. of `root` as tick-0000.. of `dest`: what a restarted process is asked next"""
    n = 0
    while os.path.exists(os.path.join(root, "tick-%04d" % (k + n))):
        shutil.copytree(os.path.join(root, "tick-%04d" % (k + n)), os.path.join(dest, "tick-%04d" % n))
        n += 1
    return str(dest), n


@pytest.fixture(scope="module", params=[False, True], ids=["util", "util+power"])
def timeline(request, tmp_path_factory, oracle_np):
    power = request.param
    d = tmp_path_factory.mktemp("snap_" + ("power" if power else "util"))
    root, n, dur = _scenario(d / "ticks", 4 + power, power)
    extra = ("--power-threshold", "150") if power else ()
    full = _verdicts(_run(root, n, dur, *extra))
    thr = 150.0 if power else None
    want = ["Query returned %d series across %d unique pods" % _expected(root, k, dur, thr, oracle_np) for k in range(n)]
    assert full == want
    return d, root, n, dur, extra, full, power


@pytest.mark.parametrize("k", CUTS)
def test_restart_resumes_from_the_snapshot(timeline, k):
    d, root, n, dur, extra, full, _ = timeline
    snap = d / ("snap-%d" % k)
    a = _run(root, k, dur, *extra, "--snapshot-file", str(snap))
    assert _verdicts(a) == full[:k]
    assert sum(m.startswith("Snapshot written to") for m in a) == k, [m for m in a if "napshot" in m]
    assert any(m.startswith("Snapshot not restored (no snapshot file") for m in a)
    broot, nb = _renumbered(root, k, d / ("b-%d" % k))
    b = _run(broot, nb, dur, *extra, "--snapshot-file", str(snap))
    assert any(m.startswith("Snapshot restored from") for m in b), [m for m in b if "napshot" in m]
    assert _verdicts(b) == full[k:]
    ingests = [m for m in b if m.startswith("Device ingest")]
    # the scenario forces the full range at ticks 6 (a third GPU slot) and 7 (no slice): no cut lands there
    assert "appended to the resident" in ingests[0], ingests[0]


def test_snapshot_file_holds_the_window_of_a_fresh_ingest(timeline):
    """the file read by tests/snapshot_ref.py (written from DESIGN.md §8i): its CRC checks, and its chunks, decoded by
    tests/chunks_ref.py, give back the window a fresh CPU ingest of that tick yields"""
    d, root, n, dur, extra, _, power = timeline
    k = 3
    snap = d / "snap-file-check"
    _run(root, k, dur, *extra, "--snapshot-file", str(snap))
    doc = SR.read(open(snap, "rb").read())
    fd = os.path.join(root, "tick-%04d" % (k - 1), "full")
    q = json.load(open(os.path.join(fd, "query.json")))
    load = lambda f: json.load(open(os.path.join(fd, f))) if os.path.exists(os.path.join(fd, f)) else None
    u, w, meta = H.ingest(load("util.json"), load("prof.json"), load("power.json") if power else None,
                          duration_min=dur, step=q["step"], t_end=q["end"], power_threshold=150.0 if power else None)
    assert doc["t_end"] == q["end"] and doc["step"] == q["step"] and doc["power"] == power
    G, T = doc["G"], doc["T"]
    assert T == u.shape[2]
    rows = doc["pods_cap"] * G
    planes = [XR.restore(p["series_chunks"], p["rows"], p["chunk_bytes"], p["data"], rows, T, doc["t_end"], doc["step"])
              for p in doc["planes"]]
    fresh = [u] + ([w] if power else [])
    used = [np.zeros(rows, bool) for _ in planes]
    for pf, pod in enumerate(meta["pods"]):
        pr = [i for i, p in enumerate(doc["pods"]) if (p["name"], p["ns"]) == (pod["name"], pod["namespace"])]
        assert len(pr) == 1, pod["name"]
        for plane, n_slots in ((0, len(pod["slots"])), (1, pod["power_slots"] if power else 0)):
            for sf in range(n_slots):
                want = XR.canonical(fresh[plane][pf, sf].view(np.uint32))
                hit = [r for r in range(pr[0] * G, pr[0] * G + G) if not used[plane][r] and (planes[plane][r] == want).all()]
                assert hit, (pod["name"], plane, sf)
                used[plane][hit[0]] = True
    for plane, pl in enumerate(planes):
        assert (pl[~used[plane]] == XR.FILL).all()   # nothing but "no sample" elsewhere


@pytest.mark.parametrize("damage", ["flip", "truncate"])
def test_damaged_snapshot_rebuilds_from_the_full_range(timeline, damage):
    d, root, n, dur, extra, full, _ = timeline
    k = 3
    snap = d / ("snap-" + damage)
    _run(root, k, dur, *extra, "--snapshot-file", str(snap))
    blob = bytearray(open(snap, "rb").read())
    if damage == "flip":
        p = SR.read(bytes(blob))["planes"][0]
        blob[p["data_at"] + len(p["data"]) // 2] ^= 0x10
    else:
        blob = blob[:len(blob) // 2]
    open(snap, "wb").write(bytes(blob))
    broot, nb = _renumbered(root, k, d / ("b-" + damage))
    b = _run(broot, nb, dur, *extra, "--snapshot-file", str(snap))
    why = [m for m in b if m.startswith("Snapshot not restored")]
    assert why and ("checksum" in why[0] if damage == "flip" else "truncated" in why[0]), why
    assert _verdicts(b) == full[k:]
    assert "into a resident" in [m for m in b if m.startswith("Device ingest")][0]


def test_missing_snapshot_directory_changes_nothing(timeline, tmp_path):
    d, root, n, dur, extra, full, _ = timeline
    cmd = [H.BIN, "--prometheus-url", f"file://{root}", "-d", "-c", "0", "--max-ticks", str(n), "-t", str(dur), "-l",
           "json", *extra, "--snapshot-file", str(tmp_path / "no" / "such" / "dir" / "snap")]
    p = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    assert p.returncode == 0, p.stderr[-3000:]
    logs = [json.loads(l) for l in p.stderr.splitlines() if l.startswith("{")]
    msgs = [l["fields"]["message"] for l in logs]
    assert _verdicts(msgs) == full
    errors = [l for l in logs if l["level"] == "ERROR" and l["fields"]["message"].startswith("Snapshot not written")]
    assert len(errors) == n and all(l["fields"].get("monotonic_counter.snapshot_failures") == "1" for l in errors)
    assert not any("query_failures" in json.dumps(l["fields"]) for l in logs)


def test_cpu_ingest_ignores_the_flag(timeline, tmp_path):
    d, root, n, dur, extra, _, _ = timeline
    runs = []
    for flag in ((), ("--snapshot-file", str(tmp_path / "snap"))):
        cmd = [H.BIN, "--prometheus-url", f"file://{root}", "-d", "-c", "0", "--max-ticks", str(n), "-t", str(dur), "-l",
               "json", *extra, *flag]
        p = subprocess.run(cmd, capture_output=True, text=True, timeout=600, env=dict(os.environ, GPR_INGEST="cpu"))
        assert p.returncode == 0
        runs.append([json.loads(l)["fields"]["message"] for l in p.stderr.splitlines() if l.startswith("{")])
    assert _verdicts(runs[1]) == _verdicts(runs[0]) and len(_verdicts(runs[0])) == n
    assert sum("snapshots need the device ingest" in m for m in runs[1]) == 1
    assert not os.path.exists(tmp_path / "snap")
