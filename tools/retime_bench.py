"""--retime-ring (DESIGN.md §8e) at C2 size: gpr_resident_retime alone on a [10,000][4][1,800] ring with the power
plane and the block index (the ring of tools/remap_bench.py and tools/export_bench.py).

  (a) factor 2 (the query step doubled), (b) n_keep 900, factor 1 (--duration halved), (c) both.
For each: the kernels' time (k_retime_rows, one per plane, from torch.profiler's CUDA activity: the median over the
calls of the per-call sum), the whole call (host clock around the blocking call: allocation, gathers, wait, free), both
medians of --calls calls after 3 warm-up calls, and the bytes the gathers must move (every kept cell read once, every new
cell written once, in both planes) over the kernel time.  Every call starts from the same ring, copied in from a device
tensor between calls.  The card's name and power limit are read in the same run.

    python tools/retime_bench.py [--pods 10000 --gpus 4 --samples 1800 --calls 50]"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=60).stdout.strip()
    except OSError as e:
        q = f"nvidia-smi not run: {e}"
    return q


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pods", type=int, default=10000)
    ap.add_argument("--gpus", type=int, default=4)
    ap.add_argument("--samples", type=int, default=1800)
    ap.add_argument("--calls", type=int, default=50)
    a = ap.parse_args()
    import torch
    import gpu_pruner_b200 as g
    from gpu_pruner_b200 import ffi
    P, G, T = a.pods, a.gpus, a.samples
    rows = P * G
    out = {"card": card(), "config": f"{P} pods x {G} GPUs x {T} samples, power plane and block index"}
    gen = torch.Generator(device="cuda").manual_seed(3)
    src = [torch.rand((rows, T), device="cuda", generator=gen) * 100 for _ in range(2)]
    for s in src:
        s[torch.rand((rows, T), device="cuda", generator=gen) < 0.3] = float("nan")
    eng = g.IdleEngine(device=0)
    try:
        def fresh():
            eng.resident_init(P, G, T, power_plane=True, block_index=True)
            u, p, _ = eng.resident_planes()
            for ptr, s in ((u, src[0]), (p, src[1])):
                eng.memcpy(ptr, s.data_ptr(), s.numel() * 4, ffi.GPR_MEM_DEVICE, ffi.GPR_MEM_DEVICE)
            eng.resident_reindex()
            torch.cuda.synchronize()

        for name, n_keep, factor in (("a_factor2", T, 2), ("b_keep_half", T // 2, 1), ("c_both", T // 2, 2)):
            T2 = -(-n_keep // factor)
            for _ in range(3):
                fresh()
                eng.resident_retime(n_keep, factor)
            call_ms = []
            with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                for _ in range(a.calls):
                    fresh()
                    t0 = time.perf_counter()
                    eng.resident_retime(n_keep, factor)
                    call_ms.append((time.perf_counter() - t0) * 1e3)
            kern = [e.device_time / 1e3 if hasattr(e, "device_time") else e.cuda_time / 1e3
                    for e in prof.events() if "k_retime_rows" in e.name]
            per_call = [kern[i] + kern[i + 1] for i in range(0, len(kern) - 1, 2)]   # util, then power
            moved = 2 * rows * (n_keep + T2) * 4
            k_med = statistics.median(per_call) if per_call else float("nan")
            out[name] = {"n_keep": n_keep, "factor": factor, "T_new": T2, "kernel_launches": len(kern),
                         "kernel_ms_median": round(k_med, 4), "kernel_ms_min": round(min(per_call), 4) if per_call else None,
                         "call_ms_median": round(statistics.median(call_ms), 3), "call_ms_min": round(min(call_ms), 3),
                         "bytes_moved": moved, "GB_per_s_kernel": round(moved / k_med / 1e6, 1),
                         "share_of_3_35_TB_s": round(moved / k_med / 1e6 / 3350, 3)}
    finally:
        eng.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
