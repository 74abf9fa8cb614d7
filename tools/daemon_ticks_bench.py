"""Daemon mode through the PRODUCT BINARY at C2 size (BASELINE configs[1] shape, config #5 cadence): tick 0 = the full
30-minute range query (1.25 GB of response text) parsed on the GPU into the resident ring; ticks 1.. = only the 180 s
scraped since the previous tick (125 MB), parsed into the ring, rescan.  Reports what the binary logs per tick.
Also runs the same fixtures with GPR_INGEST=cpu (full range + CPU text parser every tick) for comparison.

    python tools/daemon_ticks_bench.py [--pods 10000 --gpus 4 --samples 1800 --new 180 --ticks 6]
                                       [--power-threshold 150] [--bins A,B --repeats 3]

--power-threshold adds a DCGM_FI_DEV_POWER_USAGE response (decimal watts, so every sample takes the float path of
the device parser and its snap to the threshold) and turns the veto clause on.  --bins times several builds of the
binary on the same fixtures, alternating them run by run; each run reports its median steady-state tick."""
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


def run(pods=10000, gpus=4, samples=1800, new=180, ticks=6, cpu_ticks=2, power_threshold=0.0, bins=None, repeats=1):
    import hostlib as H
    lib = H.lib()
    lib.gph_synth_response.restype = C.c_longlong

    def response(n, t_end):
        need = -lib.gph_synth_response(pods, gpus, n, C.c_longlong(t_end), C.c_ulonglong(7), None, C.c_longlong(0))
        buf = C.create_string_buffer(need)
        k = lib.gph_synth_response(pods, gpus, n, C.c_longlong(t_end), C.c_ulonglong(7), buf, C.c_longlong(need))
        return buf.raw[:k]

    out = {"config": f"{pods} pods x {gpus} GPUs x {samples} samples, {new} new per tick"}
    with tempfile.TemporaryDirectory() as d:
        sizes = {}
        for k in range(ticks):
            t_end = T0 + k * new
            for kind, n in (("full", samples), ("delta", new)):
                if kind == "delta" and k == 0:
                    continue
                if kind == "full" and k >= max(1, cpu_ticks):
                    continue          # only the first ticks carry the full range (enough for the CPU comparison)
                dd = os.path.join(d, "tick-%04d" % k, kind)
                os.makedirs(dd)
                text = response(n, t_end)
                sizes[kind] = len(text)
                with open(os.path.join(dd, "util.json"), "wb") as f:
                    f.write(text)
                if power_threshold:     # the same series as watts with a fractional part: 37 -> 137.37
                    with open(os.path.join(dd, "power.json"), "wb") as f:
                        f.write(re.sub(rb',"(\d+)"\]', rb',"1\1.37"]', text))
                q = {"end": t_end, "step": 1}
                if kind == "delta":
                    q["start"] = t_end - new
                json.dump(q, open(os.path.join(dd, "query.json"), "w"))
        out["text_bytes"] = sizes

        def run_binary(n_ticks, env, binary=H.BIN):
            extra = ["--power-threshold", repr(power_threshold)] if power_threshold else []
            p = subprocess.run([binary, "--prometheus-url", f"file://{d}", "-d", "-c", "0", "--max-ticks", str(n_ticks), "-t",
                                str(samples // 60), "-l", "json", "--now", str(T0)] + extra, capture_output=True, text=True,
                               timeout=1800, env=dict(os.environ, **env))
            msgs = [json.loads(l)["fields"]["message"] for l in p.stderr.splitlines() if l.startswith("{")]
            tk = []
            for m in msgs:
                r = re.match(r"Tick (\d+): window ready in ([\d.]+) ms, verdict and gates in ([\d.]+) ms \(decision kernels ([\d.]+) ms\)", m)
                if r:
                    tk.append({"tick": int(r.group(1)), "window_ms": float(r.group(2)), "verdict_ms": float(r.group(3)),
                               "kernel_ms": float(r.group(4)), "total_ms": float(r.group(2)) + float(r.group(3))})
            reads = [float(re.search(r" in ([\d.]+) ms$", m).group(1)) for m in msgs if m.startswith("Recorded responses read")]
            for t, r in zip(tk, reads):     # one read per tick in these fixtures: the file:// fixture mechanism, not the engine
                t["file_read_ms"] = r
                t["engine_ms"] = round(t["total_ms"] - r, 3)
            return tk, [m for m in msgs if m.startswith("Device ingest")], [m for m in msgs if m.startswith("Query returned")]

        if bins:
            runs = {b: [] for b in bins}
            for _ in range(repeats):
                for b in bins:
                    tk_b, _, verdicts_b = run_binary(ticks, {}, b)
                    st = sorted(t.get("engine_ms", t["total_ms"]) for t in tk_b[1:])
                    runs[b].append({"steady_tick_ms_median": st[len(st) // 2] if st else None, "verdicts": verdicts_b})
            out["alternating"] = runs
            return out
        tk, notes, verdicts = run_binary(ticks, {})
        out["resident"] = {"ticks": tk, "first_note": notes[0] if notes else None, "steady_note": notes[-1] if notes else None,
                           "verdicts": verdicts}
        steady = sorted(t.get("engine_ms", t["total_ms"]) for t in tk[1:])
        if steady:
            out["resident"]["steady_tick_ms_median"] = steady[len(steady) // 2]
            out["resident"]["samples_per_s_at_median_tick"] = pods * gpus * samples / (steady[len(steady) // 2] * 1e-3)
        if cpu_ticks > 0:
            tk_c, notes_c, verdicts_c = run_binary(cpu_ticks, {"GPR_INGEST": "cpu"})
            out["cpu_ingest_full_range"] = {"ticks": tk_c, "note": notes_c[-1] if notes_c else None, "verdicts": verdicts_c}
            out["same_verdicts"] = verdicts[:len(verdicts_c)] == verdicts_c
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pods", type=int, default=10000)
    ap.add_argument("--gpus", type=int, default=4)
    ap.add_argument("--samples", type=int, default=1800)
    ap.add_argument("--new", type=int, default=180)
    ap.add_argument("--ticks", type=int, default=6)
    ap.add_argument("--cpu-ticks", type=int, default=2)
    ap.add_argument("--power-threshold", type=float, default=0.0)
    ap.add_argument("--bins", default="", help="comma-separated gpu-pruner binaries to alternate")
    ap.add_argument("--repeats", type=int, default=1)
    a = ap.parse_args()
    bins = [b for b in a.bins.split(",") if b]
    print(json.dumps(run(a.pods, a.gpus, a.samples, a.new, a.ticks, a.cpu_ticks, a.power_threshold, bins, a.repeats)))


if __name__ == "__main__":
    main()
