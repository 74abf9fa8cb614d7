"""gpr_resident_export at C2 size: the ring of 10,000 pods x 4 GPUs x 1,800 samples of the synthetic universe (DESIGN.md
§7) with the power plane, encoded as XOR chunks, and restored from them into a fresh context.

    python tools/export_bench.py [--reps 30]

Prints the card (nvidia-smi, read-only query) and then, per plane:
  * the export into device outputs and into pinned host outputs, alternated: the host clock around the blocking call
    (median and spread over --reps), and the three kernels' times from a torch.profiler run of its own;
  * its size: samples, series, chunks, bytes, bytes per sample against the 4 B per cell of the raw plane;
  * the restore the export is for: gpr_resident_init, gpr_chunks_scatter(GPR_TEXT_RESIDENT) of the device chunks for
    both planes, gpr_resident_reindex (host clock, median), and whether the restored planes equal the exported ring
    unrolled (every NaN as the fill), bit for bit.
"""
import argparse
import ctypes as C
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
SEED, P, G, T = 0x5EED0002, 10000, 4, 1800
T_END, STEP = 1_700_000_000 + T - 1, 1
THR = 150.0
KERNELS = ("k_export_size", "k_export_scan", "k_export_write")


def export_raw(eng, plane, arrays, mem_kind):
    from gpu_pruner_b200 import ffi
    g = ffi.gpr_text_grid()
    g.struct_size = C.sizeof(ffi.gpr_text_grid)
    g.t_end, g.step, g.window_seconds, g.n_samples = T_END, STEP, T * STEP, T
    g.power_threshold = THR if plane else 0.0
    o = ffi.gpr_chunk_export()
    o.struct_size = C.sizeof(ffi.gpr_chunk_export)
    o.mem_kind = mem_kind
    ptrs = [a.data_ptr() if hasattr(a, "data_ptr") else a.ctypes.data for a in arrays]
    o.series_chunks, o.rows, o.chunk_bytes, o.data = ptrs
    o.cap_series, o.cap_chunks, o.cap_bytes = arrays[1].shape[0], arrays[2].shape[0] - 1, arrays[3].shape[0]
    rc = eng._lib.gpr_resident_export(eng._h, C.byref(g), plane, 120, C.byref(o))
    eng._check(rc)
    return o


def med(xs):
    xs = sorted(xs)
    return xs[len(xs) // 2], xs[0], xs[-1]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=30)
    args = ap.parse_args()
    print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv"],
                         capture_output=True, text=True).stdout.strip(), flush=True)
    import torch
    import gpu_pruner_b200 as g
    from gpu_pruner_b200 import ffi
    eng = g.IdleEngine(device=0)
    eng.resident_init(P, G, T, power_plane=True)
    u, p, _ = eng.resident_planes()
    eng.synth_fill(SEED, 0, u, 0, P, G, T)
    eng.synth_fill(SEED, 1, p, 0, P, G, T)
    rows = P * G
    ring = []
    for ptr in (u, p):
        a = np.empty((rows, T), np.uint32)
        eng.memcpy(a, ptr, a.nbytes, ffi.GPR_MEM_HOST, ffi.GPR_MEM_DEVICE)
        ring.append(a)
    print(f"ring [{P}][{G}][{T}] util + power, {2 * rows * T * 4 / 1e6:.0f} MB; head {eng.resident_head()}", flush=True)

    outs = {}
    for pl in (0, 1):
        ex = eng.resident_export(T_END, STEP, plane=pl, power_threshold=THR if pl else 0.0)   # sizes, and warm-up
        ns, nc, nb = ex["rows"].size, ex["chunk_bytes"].size - 1, ex["data"].size
        dev = (torch.empty(ns + 1, dtype=torch.int64, device="cuda"), torch.empty(ns, dtype=torch.int32, device="cuda"),
               torch.empty(nc + 1, dtype=torch.int64, device="cuda"), torch.empty(nb, dtype=torch.uint8, device="cuda"))
        pin = (eng.host_array((ns + 1,), np.uint64), eng.host_array((ns,), np.uint32),
               eng.host_array((nc + 1,), np.uint64), eng.host_array((nb,), np.uint8))
        torch.cuda.synchronize()
        times = {"device": [], "pinned": []}
        for _ in range(args.reps):
            for kind, arrs, mk in (("device", dev, ffi.GPR_MEM_DEVICE), ("pinned", pin, ffi.GPR_MEM_HOST)):
                t0 = time.perf_counter()
                o = export_raw(eng, pl, arrs, mk)
                times[kind].append((time.perf_counter() - t0) * 1e3)
        assert np.array_equal(pin[3], ex["data"]) and np.array_equal(dev[3].cpu().numpy(), ex["data"])
        name = ("util", "power")[pl]
        n = o.n_samples
        print(f"[{name}] {n} samples in {ns} series, {nc} chunks, {nb} bytes: {nb / n:.3f} B per sample "
              f"({nb / (rows * T):.3f} B per cell; the raw plane is 4 B per cell, {rows * T * 4} bytes)")
        for kind in ("device", "pinned"):
            m, lo, hi = med(times[kind])
            print(f"[{name}] export call, {kind} outputs: median {m:.3f} ms (min {lo:.3f}, max {hi:.3f}, "
                  f"{args.reps} calls)", flush=True)
        outs[pl] = (ex, dev)

    # the kernels, in a profiled run of their own
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(10):
            for pl in (0, 1):
                export_raw(eng, pl, outs[pl][1], ffi.GPR_MEM_DEVICE)
        torch.cuda.synchronize()
    per = {k: [] for k in KERNELS}
    for ev in prof.events():
        for k in KERNELS:
            if k in ev.name and ev.device_type.name == "CUDA":
                per[k].append(ev.device_time_total / 1e3 if hasattr(ev, "device_time_total") else ev.cuda_time_total / 1e3)
    tot = 0.0
    for k in KERNELS:
        m = med(per[k])[0] if per[k] else float("nan")
        tot += m
        print(f"kernel {k}: median {m:.3f} ms over {len(per[k])} launches (both planes)")
    print(f"kernels per export: {tot:.3f} ms", flush=True)

    # the restore: a fresh context, both planes from the device chunks, reindexed
    res = g.IdleEngine(device=0)
    rt = []
    for r in range(max(3, args.reps // 5)):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        res.resident_init(P, G, T, power_plane=True, block_index=True)
        for pl in (0, 1):
            ex, dev = outs[pl]
            res.chunks_scatter(dev[0], dev[1], dev[2], dev[3], T_END, STEP, T, rows, plane=pl, resident=True,
                               window_seconds=T * STEP, power_threshold=THR if pl else 0.0,
                               mem_kind=ffi.GPR_MEM_DEVICE, n_series=ex["rows"].size)
        res.resident_reindex()
        rt.append((time.perf_counter() - t0) * 1e3)
    m, lo, hi = med(rt)
    print(f"restore (init with index + chunks_scatter of both planes from device chunks + reindex): median {m:.3f} ms "
          f"(min {lo:.3f}, max {hi:.3f}, {len(rt)} runs)")
    ru, rp, _ = res.resident_planes()
    same = True
    for pl, ptr in enumerate((ru, rp)):
        a = np.empty((rows, T), np.uint32)
        res.memcpy(a, ptr, a.nbytes, ffi.GPR_MEM_HOST, ffi.GPR_MEM_DEVICE)
        want = ring[pl].copy()
        want[(want & 0x7FFFFFFF) > 0x7F800000] = 0xFFFFFFFF
        same = same and np.array_equal(a, want)     # head 0 in both: the synthetic ring is already unrolled
    print(f"restored ring equals the exported one bit for bit: {same}")
    res.close()
    eng.close()


if __name__ == "__main__":
    main()
