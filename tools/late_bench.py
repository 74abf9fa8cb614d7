"""What `gpu-pruner -d --late-seconds L` costs a steady daemon tick at C2, through the PRODUCT BINARY: tick 0 = the full
30-minute range (10,000 pods x 4 GPUs x 1,800 samples at a 1 s step), ticks 1.. = the 180 s scraped since the previous
tick plus the re-asked L seconds, parsed into the resident ring.  Runs L = 0, 60 and 180 alternately, `--repeats`
rounds, and reports per run the median steady tick's engine time (window + verdict, file reads taken off), the device
ingest time, the text bytes of a steady tick, and the band read and compare time the binary logs.

    python tools/late_bench.py [--pods 10000 --gpus 4 --samples 1800 --new 180 --ticks 5 --late 0,60,180 --repeats 3]
                               [--power-threshold 150]

The synthetic responses (gph_synth_response) give a sample the same value whenever it is asked, so no cell changes and
no late-cell line is logged: this measures the cost of re-asking, not late samples."""
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


def _median(xs):
    xs = sorted(x for x in xs if x is not None)
    return xs[len(xs) // 2] if xs else None


def run(pods, gpus, samples, new, ticks, lates, repeats, power_threshold):
    import hostlib as H
    lib = H.lib()
    lib.gph_synth_response.restype = C.c_longlong

    def response(n, t_end):
        need = -lib.gph_synth_response(pods, gpus, n, C.c_longlong(t_end), C.c_ulonglong(7), None, C.c_longlong(0))
        buf = C.create_string_buffer(need)
        k = lib.gph_synth_response(pods, gpus, n, C.c_longlong(t_end), C.c_ulonglong(7), buf, C.c_longlong(need))
        return buf.raw[:k]

    def write(dd, text, q):
        os.makedirs(dd)
        with open(os.path.join(dd, "util.json"), "wb") as f:
            f.write(text)
        if power_threshold:     # the same series as watts with a fractional part: 37 -> 137.37
            with open(os.path.join(dd, "power.json"), "wb") as f:
                f.write(re.sub(rb',"(\d+)"\]', rb',"1\1.37"]', text))
        json.dump(q, open(os.path.join(dd, "query.json"), "w"))

    out = {"config": f"{pods} pods x {gpus} GPUs x {samples} samples at 1 s, {new} s per tick", "runs": []}
    with tempfile.TemporaryDirectory() as d:
        roots, text_bytes = {}, {}
        for L in lates:
            root = os.path.join(d, f"L{L}")
            for k in range(ticks):
                t_end = T0 + k * new
                if k == 0 and roots:       # the same full range for every L
                    os.makedirs(root)
                    os.symlink(os.path.join(next(iter(roots.values())), "tick-0000"), os.path.join(root, "tick-0000"))
                elif k == 0:
                    write(os.path.join(root, "tick-0000", "full"), response(samples, t_end), {"end": t_end, "step": 1})
                else:
                    text = response(new + L, t_end)
                    text_bytes[L] = len(text)
                    write(os.path.join(root, "tick-%04d" % k, "delta"), text,
                          {"end": t_end, "step": 1, "start": t_end - new - L})
            roots[L] = root
        out["steady_text_bytes"] = text_bytes

        def run_binary(L):
            extra = ["--power-threshold", repr(power_threshold)] if power_threshold else []
            p = subprocess.run([H.BIN, "--prometheus-url", f"file://{roots[L]}", "-d", "-c", "0", "--max-ticks", str(ticks),
                                "-t", str(samples // 60), "-l", "json", "--now", str(T0), "--late-seconds", str(L)] + extra,
                               capture_output=True, text=True, timeout=1800)
            assert p.returncode == 0, p.stderr[-2000:]
            msgs = [json.loads(l)["fields"]["message"] for l in p.stderr.splitlines() if l.startswith("{")]
            tk = []
            for m in msgs:
                r = re.match(r"Tick (\d+): window ready in ([\d.]+) ms, verdict and gates in ([\d.]+) ms", m)
                if r:
                    tk.append({"window_ms": float(r.group(2)), "verdict_ms": float(r.group(3))})
            reads = [float(re.search(r" in ([\d.]+) ms$", m).group(1)) for m in msgs if m.startswith("Recorded responses read")]
            for t, r in zip(tk, reads):
                t["engine_ms"] = t["window_ms"] + t["verdict_ms"] - r
            notes = [m for m in msgs if m.startswith("Device ingest")]
            ingest = [float(re.search(r"window in ([\d.]+) ms", m).group(1)) for m in notes]
            band = [float(b.group(1)) if (b := re.search(r"band read and compare ([\d.]+) ms", m)) else None for m in notes]
            assert all("appended to the resident" in m for m in notes[1:]), notes
            assert not any(m.startswith("Resident window rebuilt") for m in msgs)
            return {"L": L, "steady_engine_ms_median": _median([t["engine_ms"] for t in tk[1:]]),
                    "steady_ingest_ms_median": _median(ingest[1:]), "band_ms_median": _median(band[1:]),
                    "steady_ticks": len(tk) - 1, "late_lines": sum(m.startswith("Late samples") for m in msgs),
                    "verdicts": sorted(set(m for m in msgs if m.startswith("Query returned")))}

        for rep in range(repeats):
            for L in lates:
                r = run_binary(L)
                r["round"] = rep
                out["runs"].append(r)
                print(json.dumps(r), file=sys.stderr, flush=True)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pods", type=int, default=10000)
    ap.add_argument("--gpus", type=int, default=4)
    ap.add_argument("--samples", type=int, default=1800)
    ap.add_argument("--new", type=int, default=180)
    ap.add_argument("--ticks", type=int, default=5)
    ap.add_argument("--late", default="0,60,180")
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--power-threshold", type=float, default=0.0)
    a = ap.parse_args()
    print(json.dumps(run(a.pods, a.gpus, a.samples, a.new, a.ticks, [int(x) for x in a.late.split(",")], a.repeats,
                         a.power_threshold)))


if __name__ == "__main__":
    main()
