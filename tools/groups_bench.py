"""Developer benchmark of `sum by` group tables (gpr_window.groups) on a C2 window (10,000 pods x 4 x 1800, the
synthetic generator of bench.py): both f32 kernels, five variants —
  none      no table (what bench.py runs)
  slots     no table, idle_slots requested (what the gpu-pruner binary runs for a window without groups)
  lone      a table in which every series leads itself (the group kernels run, nothing is read whole)
  grouped   15 % of the pods with a group of 2-3 series (their rows are read whole and summed)
  smax      no table, series_max requested (what the gpu-pruner binary asked for before the table existed)
— each as pipelined async batches (CUDA events around `iters` back-to-back decisions) and as one isolated blocking
decision, with the modelled bytes read (the early-exit rule of gpr_kernels.cuh per row; 4 T for a grouped row or any
row under series_max).  The card name and power limit are read in the same run."""
import argparse
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402

import gpu_pruner_b200 as g  # noqa: E402

P, G, T = 10000, 4, 1800
SEED = 0x5EED0002
HEAD, LDG_UNROLL = 128, 8


def tables(rng):
    lone = np.tile(np.arange(G, dtype=np.uint32), (P, 1))
    grouped = lone.copy()
    for p in np.flatnonzero(rng.random(P) < 0.15):
        grouped[p, 1:int(rng.integers(2, 4))] = 0
        grouped[p] |= np.where(rng.random(G) < 0.5, 0x100, 0).astype(np.uint32)
    return lone, grouped


def modelled_bytes(first, full, kernel):
    """first settling sample of each row (T = none); full = rows read whole"""
    if kernel == "tma":   # head, then the rest in one chunk (T 1800 at the default 8 KB chunk)
        n = np.where(first < HEAD, HEAD, T)
    else:                 # aligned rows: 32 float4 per warp, then batches of 8 x 32 float4
        stops = [HEAD]
        while stops[-1] < T:
            stops.append(min(stops[-1] + 4 * 32 * LDG_UNROLL, T))
        stops = np.array(stops)
        n = np.where(first < T, stops[np.minimum(np.searchsorted(stops, first, side="right"), len(stops) - 1)], T)
    return int((4 * np.where(full, T, n)).sum())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    try:
        smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        smi = f"nvidia-smi unavailable ({e})"
    print(f"# card: {smi}")
    rng = np.random.default_rng(1)
    lone, grouped = tables(rng)
    dev = "cuda:0"
    for kernel in ("tma", "ldg"):
        eng = g.IdleEngine(device=0, kernel=kernel)
        u = torch.empty((P, G, T), dtype=torch.float32, device=dev)
        eng.synth_fill(SEED, 0, u, 0, P, G, T)
        torch.cuda.synchronize()
        x = u.cpu().numpy().reshape(P * G, T)
        pos = x > 0
        first = np.where(pos.any(1), pos.argmax(1), T)
        db = torch.zeros((P + 31) // 32, dtype=torch.int32, device=dev)
        isl = torch.zeros(P, dtype=torch.int32, device=dev)
        sm = torch.empty((P, G), dtype=torch.float32, device=dev)
        lone_t = torch.from_numpy(lone.astype(np.int32)).to(dev)
        grouped_t = torch.from_numpy(grouped.astype(np.int32)).to(dev)
        lead = grouped & 0xFF
        full_grouped = np.array([np.bincount(r, minlength=G)[r] > 1 for r in lead]).ravel()
        variants = {
            "none": (dict(), np.zeros(P * G, bool)),
            "slots": (dict(idle_slots=isl), np.zeros(P * G, bool)),
            "lone": (dict(groups=lone_t, idle_slots=isl), np.zeros(P * G, bool)),
            "grouped": (dict(groups=grouped_t, idle_slots=isl), full_grouped),
            "smax": (dict(series_max=sm), np.ones(P * G, bool)),
        }
        for name, (kw, full) in variants.items():
            for _ in range(5):
                eng.decide_ptr(u, P, G, T, db, blocking=False, **kw)
            eng.sync()
            best = 1e9
            for _ in range(args.reps):
                eng.timer_begin()
                for _ in range(args.iters):
                    eng.decide_ptr(u, P, G, T, db, blocking=False, **kw)
                ms = eng.timer_end()
                eng.sync()
                best = min(best, ms / args.iters)
            iso = 1e9
            for _ in range(args.reps):
                eng.flush_l2()
                r = eng.decide_ptr(u, P, G, T, db, **kw)
                iso = min(iso, r.kernel_ms)
            mb = modelled_bytes(first, full, kernel) / 1e6
            print(f"{kernel:4s} {name:8s} pipelined {best * 1e3:8.1f} us   isolated {iso * 1e3:8.1f} us   "
                  f"modelled {mb:7.1f} MB of {4 * P * G * T / 1e6:.0f}")
            time.sleep(0.2)
        eng.close()


if __name__ == "__main__":
    main()
