"""--reshape-ring (DESIGN.md §8e) at C2 size: the reshaping tick against the full-range rebuild tick it replaces, through
the PRODUCT BINARY, and gpr_resident_live_rows alone.

  tick  tick 0 = the full range of 10,000 pods x 4 GPUs x 1,800 s (the engine's synthetic response, 1.25 GB), in which
        a fifth of the pods (pod % 5 == 0) have samples only in the oldest --new seconds: they depart.  Tick 1 is a --new
        second slice in which every remaining pod reports a fifth GPU (G 4 -> 5) and 2,500 new pods (+25 %) join with 5
        GPUs each.  With --reshape-ring the binary reshapes: the departed pods are dropped, the ring remapped to
        [10,500 + 2,625 + 64][5]; without it the same tick throws NeedFullWindow and rebuilds from tick 1's full range
        (what a server would answer: the kept series' samples still in the window and their slice; the series new in
        the slice with the slice alone), so both paths must reach the same verdict.  Engine time = tick time minus the fixture read (the
        file:// mechanism).  The two runs alternate --repeats times; each is a fresh process with the same fixtures.
  live  gpr_resident_live_rows alone on a [10,000][4][1,800] ring, with and without the power plane, every row live
        (a sample in the first cell: one load per row) and every row dead (the fill: both planes read whole); host
        clock around the blocking call, median of 50 after 5 warm-up calls.

    python tools/reshape_bench.py [--pods 10000 --gpus 4 --samples 1800 --new 180 --repeats 3]"""
import argparse
import ctypes as C
import json
import os
import re
import statistics
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
T0 = 1_700_000_000
SEP = b',{"metric":'
TICK = re.compile(r"Tick (\d+): window ready in ([\d.]+) ms, verdict and gates in ([\d.]+) ms")
SHAPED = re.compile(r"Resident window reshaped on the GPU: .*\(live rows ([\d.]+) ms, remap ([\d.]+) ms\)")


def series_of(lib, P, G, n, t_end):
    """the synthetic response's series objects, in (pod, gpu) order, each as b'{"metric":...]}'"""
    need = -lib.gph_synth_response(P, G, n, C.c_longlong(t_end), C.c_ulonglong(7), None, C.c_longlong(0))
    buf = C.create_string_buffer(need)
    k = lib.gph_synth_response(P, G, n, C.c_longlong(t_end), C.c_ulonglong(7), buf, C.c_longlong(need))
    body = buf.raw[:k]
    head = body.index(b"[{") + 1
    parts = body[head:body.rindex(b"]}}")].split(SEP)
    return [p if i == 0 else b'{"metric":' + p for i, p in enumerate(parts[:-1])] + [b'{"metric":' + parts[-1]]


def write(d, parts, t_end, start=None):
    os.makedirs(d)
    with open(os.path.join(d, "util.json"), "wb") as f:
        f.write(b'{"status":"success","data":{"resultType":"matrix","result":[')
        f.write(b",".join(parts))
        f.write(b"]}}")
    q = {"end": t_end, "step": 1}
    if start is not None:
        q["start"] = start
    json.dump(q, open(os.path.join(d, "query.json"), "w"))


def tick_fixtures(lib, root, pods, gpus, samples, new):
    G2, P2 = gpus + 1, pods + pods // 4
    gone = lambda p: p < pods and p % 5 == 0
    full0 = series_of(lib, pods, gpus, samples, T0)
    old0 = series_of(lib, pods, gpus, new, T0 - samples + new)       # the departed pods' oldest --new seconds
    write(os.path.join(root, "tick-0000", "full"),
          [(old0 if gone(i // gpus) else full0)[i] for i in range(pods * gpus)], T0)
    del full0, old0
    sl = series_of(lib, P2, G2, new, T0 + new)
    write(os.path.join(root, "tick-0001", "delta"), [s for i, s in enumerate(sl) if not gone(i // G2)], T0 + new, start=T0)
    # tick 1's full range is what a server would answer: a kept series' samples of tick 0 that are still in the window,
    # then its slice; the series new in the slice (fifth GPUs, new pods) with the slice alone
    full0 = series_of(lib, pods, gpus, samples, T0)
    first = b"[%d," % (T0 - samples + new + 1)
    parts = []
    for p in range(P2):
        if gone(p):
            continue
        for g in range(G2):
            s = sl[p * G2 + g]
            if p < pods and g < gpus:
                o = full0[p * gpus + g]
                s = o[:o.index(b'"values":[') + 10] + o[o.index(first):-2] + b"," + s[s.index(b'"values":[') + 10:]
            parts.append(s)
    write(os.path.join(root, "tick-0001", "full"), parts, T0 + new)


def binary(H, root, samples, reshape):
    cmd = [H.BIN, "--prometheus-url", f"file://{root}", "-d", "-c", "0", "--max-ticks", "2", "-t", str(samples // 60),
           "-l", "json", "--now", str(T0)] + (["--reshape-ring"] if reshape else [])
    p = subprocess.run(cmd, capture_output=True, text=True, timeout=1800)
    assert p.returncode == 0, p.stderr[-2000:]
    msgs = [json.loads(l)["fields"]["message"] for l in p.stderr.splitlines() if l.startswith("{")]
    reads = [float(re.search(r" in ([\d.]+) ms$", m).group(1)) for m in msgs if m.startswith("Recorded responses read")]
    # tick 0 reads one fixture; tick 1 the delta and, when it rebuilds, the full range as well
    r = {"verdicts": [m for m in msgs if m.startswith("Query returned")],
         "ingest": [m for m in msgs if m.startswith("Device ingest")],
         "reshaped": [m for m in msgs if m.startswith("Resident window reshaped")],
         "rebuilt": [m for m in msgs if m.startswith("Resident window rebuilt")],
         "reads_ms": reads}
    tk = [float(t.group(2)) + float(t.group(3)) for t in map(TICK.match, msgs) if t]
    r["tick_ms"] = tk
    r["tick1_engine_ms"] = round(tk[1] - sum(reads[1:]), 3)
    s = [SHAPED.match(m) for m in r["reshaped"]]
    if s and s[0]:
        r["live_rows_ms"], r["remap_ms"] = float(s[0].group(1)), float(s[0].group(2))
    return r


def live_rows(pods, gpus, samples):
    import numpy as np
    import gpu_pruner_b200 as g
    from gpu_pruner_b200 import ffi
    out = {}
    eng = g.IdleEngine(device=0)
    try:
        for power in (False, True):
            eng.resident_init(pods, gpus, samples, power_plane=power)
            rows = pods * gpus
            for kind in ("dead", "live"):
                if kind == "live":   # one sample in the first cell of every row of the util plane
                    u, _, _ = eng.resident_planes()
                    a = np.full((rows, samples), 0xFFFFFFFF, np.uint32)
                    a[:, 0] = np.float32(5.0).view(np.uint32)
                    eng.memcpy(u, a, a.nbytes, ffi.GPR_MEM_DEVICE, ffi.GPR_MEM_HOST)
                    del a
                for _ in range(5):
                    bits = eng.resident_live_rows()
                assert bits.all() if kind == "live" else not bits.any()
                ts = []
                for _ in range(50):
                    t0 = time.perf_counter()
                    eng.resident_live_rows()
                    ts.append((time.perf_counter() - t0) * 1e3)
                # what the call has to read: a live row's first 16-byte load per lane (512 B), a dead row whole in every plane
                read = rows * 512 if kind == "live" else rows * samples * 4 * (2 if power else 1)
                out[f"{'power' if power else 'util'}_{kind}"] = {
                    "median_ms": round(statistics.median(ts), 4), "min_ms": round(min(ts), 4),
                    "bytes_needed": read, "GB_per_s_at_median": round(read / statistics.median(ts) / 1e6, 1)}
    finally:
        eng.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pods", type=int, default=10000)
    ap.add_argument("--gpus", type=int, default=4)
    ap.add_argument("--samples", type=int, default=1800)
    ap.add_argument("--new", type=int, default=180)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--skip-live", action="store_true")
    a = ap.parse_args()
    import hostlib as H
    lib = H.lib()
    lib.gph_synth_response.restype = C.c_longlong
    out = {"config": f"{a.pods} pods x {a.gpus} GPUs x {a.samples} s, a {a.new} s tick: 20 % depart, +25 % join, G -> "
                     f"{a.gpus + 1}"}
    with tempfile.TemporaryDirectory() as d:
        tick_fixtures(lib, d, a.pods, a.gpus, a.samples, a.new)
        out["fixture_bytes"] = {k: os.path.getsize(os.path.join(d, k, "util.json"))
                                for k in ("tick-0000/full", "tick-0001/delta", "tick-0001/full")}
        out["runs"] = []
        for _ in range(a.repeats):
            rs = binary(H, d, a.samples, True)
            rb = binary(H, d, a.samples, False)
            out["runs"].append({"reshape": rs, "rebuild": rb, "same_verdicts": rs["verdicts"] == rb["verdicts"]})
    if not a.skip_live:
        out["live_rows"] = live_rows(a.pods, a.gpus, a.samples)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
