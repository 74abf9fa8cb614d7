"""--query-slice (DESIGN.md §8e) at C2 size: the cold start of `gpu-pruner -d` asked as one query against the same range
asked as slices of --slice seconds, through the PRODUCT BINARY.

  fixtures  10,000 pods x 4 GPUs x 1,800 s (the engine's synthetic response): tick-0000/full/util.json for the one
            query, and tick-0000/full/slice-%04d/ with each slice's response (the synthetic response of that slice's
            (start, end]) for the sliced run.  The largest query's sample count and text bytes are read from them.
  times     per run, the device ingest's time from the binary's log; the sliced run reads each slice between merges, so
            the reads it logs are taken off: the engine time of the cold start.  The tick's "window ready" time is kept
            beside it (it also holds the fixture reads and the context's creation).
  ring      both runs write --snapshot-file after the tick; the two files must hold the same ring and session by series
            identity (tests/snapshot_identity.py).
  memory    peak device memory of the binary's process is not measured (no read-only per-process query is used here).

    python tools/slice_bench.py [--pods 10000 --gpus 4 --samples 1800 --slice 180 --repeats 3]"""
import argparse
import ctypes as C
import json
import os
import re
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))
from reshape_bench import T0, TICK, series_of, write  # noqa: E402


def fixtures(lib, root, pods, gpus, samples, S):
    full = os.path.join(root, "tick-0000", "full")
    write(full, series_of(lib, pods, gpus, samples, T0), T0)
    n = -(-samples // S)
    sizes = []
    for j in range(n):
        a, b = max(T0 - samples, T0 - (n - j) * S), T0 - (n - 1 - j) * S
        d = os.path.join(full, "slice-%04d" % j)
        write(d, series_of(lib, pods, gpus, b - a, b), b, start=a)
        sizes.append({"start": a, "end": b, "samples": pods * gpus * (b - a),
                      "bytes": os.path.getsize(os.path.join(d, "util.json"))})
    return {"one_query": {"samples": pods * gpus * samples, "bytes": os.path.getsize(os.path.join(full, "util.json"))},
            "largest_slice": max(sizes, key=lambda s: s["bytes"]), "slices": len(sizes)}


def binary(H, root, samples, S, snapshot=None):
    cmd = [H.BIN, "--prometheus-url", f"file://{root}", "-d", "-c", "0", "--max-ticks", "1", "-t", str(samples // 60),
           "-l", "json", "--now", str(T0)] + (["--query-slice", str(S)] if S else []) + \
          (["--snapshot-file", snapshot] if snapshot else [])
    p = subprocess.run(cmd, capture_output=True, text=True, timeout=1800)
    assert p.returncode == 0, p.stderr[-2000:]
    msgs = [json.loads(l)["fields"]["message"] for l in p.stderr.splitlines() if l.startswith("{")]
    reads = [float(m.group(1)) for m in (re.search(r" in ([\d.]+) ms$", x) for x in msgs
                                          if x.startswith("Recorded responses read")) if m]
    t = [TICK.match(m) for m in msgs if TICK.match(m)][0]
    ingest = [m for m in msgs if m.startswith("Device ingest")]
    ingest_ms = float(re.search(r" in ([\d.]+) ms \(", ingest[0]).group(1))
    return {"verdict": [m for m in msgs if m.startswith("Query returned")], "ingest": ingest,
            "window_ready_ms": float(t.group(2)), "read_ms": sum(reads), "ingest_ms": ingest_ms,
            # the sliced ingest reads each slice between merges: its reads are inside ingest_ms
            "engine_ms": round(ingest_ms - (sum(reads) if S else 0), 3), "decide_ms": float(t.group(3))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pods", type=int, default=10000)
    ap.add_argument("--gpus", type=int, default=4)
    ap.add_argument("--samples", type=int, default=1800)
    ap.add_argument("--slice", type=int, default=180)
    ap.add_argument("--repeats", type=int, default=3)
    a = ap.parse_args()
    import hostlib as H
    lib = H.lib()
    lib.gph_synth_response.restype = C.c_longlong
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    out = {"gpu": gpu, "config": f"{a.pods} pods x {a.gpus} GPUs x {a.samples} s, slices of {a.slice} s"}
    with tempfile.TemporaryDirectory() as d:
        out["queries"] = fixtures(lib, d, a.pods, a.gpus, a.samples, a.slice)
        out["runs"] = []
        for i in range(a.repeats):
            snaps = [os.path.join(d, "snap-one"), os.path.join(d, "snap-sliced")] if i == 0 else [None, None]
            one, sl = binary(H, d, a.samples, 0, snaps[0]), binary(H, d, a.samples, a.slice, snaps[1])
            out["runs"].append({"one_query": one, "sliced": sl, "same_verdict": one["verdict"] == sl["verdict"]})
            if i == 0:
                import snapshot_identity as SI
                out["same_ring_and_session"] = SI.mismatch(open(snaps[0], "rb").read(), open(snaps[1], "rb").read()) or True
    print(json.dumps(out))


if __name__ == "__main__":
    main()
