"""Developer micro-benchmark: device-resident windows, back-to-back async decides, CUDA events.
Not the judged benchmark (that is bench.py); used to compare kernel variants and tunables."""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

import gpu_pruner_b200 as g  # noqa: E402


# Windows other than the synthetic ones bound what a row costs: `idle` (all zeros) and `late` (zeros, one busy sample
# in the last column: the same bytes, another verdict) are read to the end of every row, `busy` (all ones) is
# settled by every row's first sample.  The power plane gets the same pattern, scaled past the 150 W threshold.
FILLS = ("synthetic", "idle", "late", "busy")


def window(eng, fill, seed, plane, P, G, T):
    x = torch.empty((P, G, T), dtype=torch.float32, device="cuda:0")
    if fill == "synthetic":
        eng.synth_fill(seed, plane, x, 0, P, G, T)
        return x
    x.zero_()
    hot = 1000.0 if plane else 1.0
    if fill == "late":
        x[:, :, T - 1] = hot
    elif fill == "busy":
        x.fill_(hot)
    return x


def run(variant, P, G, T, iters, rot, power=False, u8=False, fill="synthetic", smax=False):
    eng = g.IdleEngine(device=0, kernel=variant)
    wins = []
    for i in range(rot):
        u = window(eng, fill, 0x5EED0002 + i, 0, P, G, T)
        w = window(eng, fill, 0x5EED0002 + i, 1, P, G, T) if power else None
        if u8:   # GPR_FMT_U8B: 0 = no sample, b = value + 1
            u = torch.where(torch.isnan(u), torch.zeros_like(u), u + 1).to(torch.uint8)
        wins.append((u, w))
    fmt = g.ffi.GPR_FMT_U8B if u8 else g.ffi.GPR_FMT_F32
    db = torch.zeros((P + 31) // 32, dtype=torch.int32, device="cuda:0")
    sm = torch.empty((P, G), dtype=torch.float32, device="cuda:0") if smax else None   # asks for every row whole
    torch.cuda.synchronize()
    for i in range(5):
        eng.decide_ptr(wins[i % rot][0], P, G, T, db, power=wins[i % rot][1], power_threshold=150.0 if power else 0.0,
                       blocking=False, util_format=fmt, series_max=sm)
    eng.sync()
    best = 1e9
    tot = 0.0
    reps = 3
    for _ in range(reps):
        eng.timer_begin()
        for i in range(iters):
            eng.decide_ptr(wins[i % rot][0], P, G, T, db, power=wins[i % rot][1],
                           power_threshold=150.0 if power else 0.0, blocking=False, util_format=fmt, series_max=sm)
        ms = eng.timer_end()
        eng.sync()
        best = min(best, ms / iters)
        tot += ms / iters
    nbytes = (1.0 if u8 else 4.0) * P * G * T + (4.0 * P * G * T if power else 0.0)
    print(f"{'u8' if u8 else variant:4s} P={P} G={G} T={T} power={int(power)} rot={rot} fill={fill}"
          f"{' series_max' if smax else ''}: best {best*1e3:8.2f} us/step  "
          f"avg {tot/reps*1e3:8.2f} us  -> {nbytes/best/1e6:8.1f} GB/s (best)  "
          f"{P/best/1e3:8.2f} Mdecisions/s", flush=True)
    eng.close()


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", default="c2,c3")
    ap.add_argument("--variants", default="ldg,tma")
    ap.add_argument("--iters", type=int, default=100)
    ap.add_argument("--shape", default="", help="P,G,T,rot (overrides --configs)")
    ap.add_argument("--power", action="store_true")
    ap.add_argument("--u8", action="store_true", help="windows in the biased-byte format (one kernel, --variants ignored)")
    ap.add_argument("--fill", default="synthetic", choices=FILLS, help="window contents (see FILLS)")
    ap.add_argument("--series-max", action="store_true", help="ask for series_max: every row is read whole")
    ap.add_argument("--no-power-row", action="store_true", help="skip the C2 power-plane row of --configs c2")
    a = ap.parse_args()
    kw = {"fill": a.fill, "smax": a.series_max}
    shapes = {"c2": (10000, 4, 1800, 6), "c3": (100000, 8, 3600, 2), "c4": (250000, 4, 1800, 2),
              "c5s": (312500, 4, 7200, 1)}
    if a.u8:
        for c in a.configs.split(","):
            P, G, T, rot = shapes[c]
            run("auto", P, G, T, a.iters if c == "c2" else max(10, a.iters // 5), rot * 3, u8=True)
        sys.exit(0)
    if a.shape:
        P, G, T, rot = map(int, a.shape.split(","))
        for v in a.variants.split(","):
            run(v, P, G, T, a.iters, rot, power=a.power, **kw)
        sys.exit(0)
    for c in a.configs.split(","):
        P, G, T, rot = shapes[c]
        for v in a.variants.split(","):
            run(v, P, G, T, a.iters if c == "c2" else max(10, a.iters // 5), rot, **kw)
    if "c2" in a.configs.split(",") and not a.no_power_row:
        for v in a.variants.split(","):
            run(v, 10000, 4, 1800, a.iters, 4, power=True, **kw)
