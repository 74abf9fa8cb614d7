"""Daemon-mode snapshots (--snapshot-file, DESIGN.md §8i) through the PRODUCT BINARY at C2 size, with the power plane:
the C2 tick fixtures of tools/daemon_ticks_bench.py (the engine's synthetic response, 1.25 GB per full range).

  A     tick 0 = the full range, tick 1 = a 180 s slice, each followed by the snapshot: its size and the binary's own
        breakdown (export, copy, checksum, write) from its log lines.  The first snapshot of a process also sizes and
        allocates the export buffers; the second is the steady state of a running daemon
  B     a restarted process on the next tick: the restore (read, checksum, restore) from its log line, and the engine
        time of its first tick, which appends only the 180 s slice
  cold  the same next tick without the flag: the full range rebuilt from the text
B and cold alternate --repeats times.  Engine time = tick time minus the fixture read (the file:// mechanism).

    python tools/snapshot_bench.py [--pods 10000 --gpus 4 --samples 1800 --new 180 --power-threshold 150 --repeats 3]"""
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
T0 = 1_700_000_000

WRITE = re.compile(r"Snapshot written to .*: (\d+) bytes in ([\d.]+) ms \(export ([\d.]+), copy ([\d.]+), checksum ([\d.]+), "
                   r"write ([\d.]+) ms\)")
READ = re.compile(r"Snapshot restored from .*: (\d+) bytes in ([\d.]+) ms \(read ([\d.]+), checksum ([\d.]+), restore ([\d.]+) ms\)")
TICK = re.compile(r"Tick (\d+): window ready in ([\d.]+) ms, verdict and gates in ([\d.]+) ms")


def run(pods, gpus, samples, new, power_threshold, repeats):
    import hostlib as H
    lib = H.lib()
    lib.gph_synth_response.restype = C.c_longlong

    def response(n, t_end):
        need = -lib.gph_synth_response(pods, gpus, n, C.c_longlong(t_end), C.c_ulonglong(7), None, C.c_longlong(0))
        buf = C.create_string_buffer(need)
        k = lib.gph_synth_response(pods, gpus, n, C.c_longlong(t_end), C.c_ulonglong(7), buf, C.c_longlong(need))
        return buf.raw[:k]

    out = {"config": f"{pods} pods x {gpus} GPUs x {samples} samples, {new} new per tick, power {power_threshold}"}
    with tempfile.TemporaryDirectory() as d:
        def fixture(dd, n, t_end, start=None):
            os.makedirs(dd)
            text = response(n, t_end)
            with open(os.path.join(dd, "util.json"), "wb") as f:
                f.write(text)
            if power_threshold:     # as tools/daemon_ticks_bench.py: the same series as watts, 37 -> 137.37
                with open(os.path.join(dd, "power.json"), "wb") as f:
                    f.write(re.sub(rb',"(\d+)"\]', rb',"1\1.37"]', text))
            q = {"end": t_end, "step": 1}
            if start is not None:
                q["start"] = start
            json.dump(q, open(os.path.join(dd, "query.json"), "w"))

        a_root, b_root = os.path.join(d, "a"), os.path.join(d, "b")
        fixture(os.path.join(a_root, "tick-0000", "full"), samples, T0)
        fixture(os.path.join(a_root, "tick-0001", "delta"), new, T0 + new, start=T0)
        fixture(os.path.join(b_root, "tick-0000", "full"), samples, T0 + 2 * new)
        fixture(os.path.join(b_root, "tick-0000", "delta"), new, T0 + 2 * new, start=T0 + new)
        snap = os.path.join(d, "snapshot")

        def binary(root, flag, n_ticks=1):
            extra = ["--power-threshold", repr(power_threshold)] if power_threshold else []
            if flag:
                extra += ["--snapshot-file", snap]
            p = subprocess.run([H.BIN, "--prometheus-url", f"file://{root}", "-d", "-c", "0", "--max-ticks", str(n_ticks), "-t",
                                str(samples // 60), "-l", "json", "--now", str(T0)] + extra, capture_output=True, text=True,
                               timeout=1800)
            assert p.returncode == 0, p.stderr[-2000:]
            msgs = [json.loads(l)["fields"]["message"] for l in p.stderr.splitlines() if l.startswith("{")]
            r = {"verdicts": [m for m in msgs if m.startswith("Query returned")],
                 "ingest": [m for m in msgs if m.startswith("Device ingest")]}
            reads = [float(re.search(r" in ([\d.]+) ms$", m).group(1)) for m in msgs if m.startswith("Recorded responses read")]
            r["ticks"], r["writes"] = [], []
            for m in msgs:
                t = TICK.match(m)
                if t:
                    tick_ms = float(t.group(2)) + float(t.group(3))
                    r["ticks"].append({"tick_ms": tick_ms, "engine_ms": round(tick_ms - reads[len(r["ticks"])], 3)})
                w = WRITE.match(m)
                if w:
                    r["writes"].append(dict(zip(("bytes", "total_ms", "export_ms", "copy_ms", "checksum_ms", "write_ms"),
                                          [int(w.group(1))] + [float(x) for x in w.groups()[1:]])))
                g = READ.match(m)
                if g:
                    r["restore"] = dict(zip(("bytes", "total_ms", "read_ms", "checksum_ms", "restore_ms"),
                                            [int(g.group(1))] + [float(x) for x in g.groups()[1:]]))
            return r

        out["snapshot"] = binary(a_root, True, 2)
        saved = open(snap, "rb").read()
        out["runs"] = []
        for _ in range(repeats):
            with open(snap, "wb") as f:        # B writes its own snapshot: every B restores the one A wrote
                f.write(saved)
            b = binary(b_root, True)
            cold = binary(b_root, False)
            out["runs"].append({"resumed": b, "cold": cold, "same_verdicts": b["verdicts"] == cold["verdicts"]})
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pods", type=int, default=10000)
    ap.add_argument("--gpus", type=int, default=4)
    ap.add_argument("--samples", type=int, default=1800)
    ap.add_argument("--new", type=int, default=180)
    ap.add_argument("--power-threshold", type=float, default=150.0)
    ap.add_argument("--repeats", type=int, default=3)
    a = ap.parse_args()
    print(json.dumps(run(a.pods, a.gpus, a.samples, a.new, a.power_threshold, a.repeats)))


if __name__ == "__main__":
    main()
