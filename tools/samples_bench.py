"""gpr_samples_scatter at C2 size (10,000 pods x 4 GPUs x 1,800 samples of the synthetic universe, DESIGN.md §7): every
present util cell one sample at its bucket's timestamp.

    python tools/samples_bench.py [--reps 50] [--out DIR]

Prints the card (nvidia-smi, read-only query) and then:
  * device batch: k_samples_scatter kernel time (torch.profiler CUDA activity, summed over --reps calls after a warm-up)
    and the modelled bytes over it — 16 B read per sample + 4 B merged per in-window sample — as a share of the H100
    SXM data sheet's 3.35 TB/s; and the whole blocking call (check kernel, fill, read-back) by host clock;
  * pinned host batch: the blocking call against one pinned cudaMemcpy of the same 16 B per sample (PCIe-bound);
  * the text path on the same samples: the compact matrix JSON of tests/cpp/c2_response.cpp, pinned, through
    gpr_text_scan + gpr_text_parse — and whether both paths leave the same plane.
"""
import argparse
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
SEED, P, G, T = 0x5EED0002, 10000, 4, 1800
T0 = 1_700_000_000
T_END = T0 + T - 1
HBM = 3.35e12


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--host-reps", type=int, default=5)
    args = ap.parse_args()
    print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv"],
                         capture_output=True, text=True).stdout.strip(), flush=True)
    import torch
    import gpu_pruner_b200 as g
    eng = g.IdleEngine(device=0)
    rows = P * G
    util = torch.empty((rows, T), dtype=torch.float32, device="cuda")
    eng.synth_fill(SEED, 0, util, 0, P, G, T)
    present = ~torch.isnan(util)
    counts = present.sum(1)
    offsets = torch.zeros(rows + 1, dtype=torch.int64, device="cuda")
    offsets[1:] = torch.cumsum(counts, 0)
    r_idx, c_idx = present.nonzero(as_tuple=True)
    ts = (T_END - (T - 1 - c_idx).to(torch.int64)) * 1000
    vals = util[r_idx, c_idx].to(torch.float64)
    r_ids = torch.arange(rows, dtype=torch.int32, device="cuda")
    n = int(offsets[-1])
    del r_idx, c_idx, present
    torch.cuda.synchronize()   # the context's stream is not ordered with torch's
    print(f"batch: {rows} series, {n} samples, {16 * n / 1e9:.3f} GB of timestamps + values", flush=True)

    def scatter(o, r, t, v, kind):
        return eng.samples_scatter(o, r, t, v, T_END, 1, T, rows, mem_kind=kind, n_series=rows)

    # ---- device batch
    dev = g.ffi.GPR_MEM_DEVICE
    for _ in range(5):
        st = scatter(offsets, r_ids, ts, vals, dev)
    assert st["n_oow"] == 0 and st["n_in"] == n
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(args.reps):
            scatter(offsets, r_ids, ts, vals, dev)
        torch.cuda.synchronize()
    k_us = [e.device_time for e in prof.events() if "k_samples_scatter" in e.name]
    assert len(k_us) == args.reps, len(k_us)
    k_ms = float(np.median(k_us)) / 1e3
    bytes_model = 16 * n + 4 * n
    print(f"device batch: k_samples_scatter median {k_ms:.3f} ms over {args.reps} calls (min {min(k_us) / 1e3:.3f}, "
          f"max {max(k_us) / 1e3:.3f}); modelled {bytes_model / 1e9:.3f} GB -> {bytes_model / k_ms / 1e6:.0f} GB/s = "
          f"{bytes_model / k_ms * 1e3 / HBM:.2f} of 3.35 TB/s", flush=True)
    t = []
    for _ in range(10):
        t0 = time.perf_counter()
        scatter(offsets, r_ids, ts, vals, dev)
        t.append(time.perf_counter() - t0)
    print(f"device batch: whole blocking call median {np.median(t) * 1e3:.3f} ms (check kernel, fill, scatter, "
          f"read-back)", flush=True)
    plane_dev = np.empty((rows, T), np.uint32)
    eng.memcpy(plane_dev, eng.text_planes()[0], plane_dev.nbytes, 0, 1)

    # ---- pinned host batch
    h_off, h_rows = offsets.cpu().numpy().view(np.uint64), r_ids.cpu().numpy().view(np.uint32)
    h_ts, h_vals = eng.host_array(n, np.int64), eng.host_array(n, np.float64)
    h_ts[:], h_vals[:] = ts.cpu().numpy(), vals.cpu().numpy()
    host = g.ffi.GPR_MEM_HOST
    scatter(h_off, h_rows, h_ts, h_vals, host)
    t = []
    for _ in range(args.host_reps):
        t0 = time.perf_counter()
        scatter(h_off, h_rows, h_ts, h_vals, host)
        t.append(time.perf_counter() - t0)
    plane_host = np.empty((rows, T), np.uint32)
    eng.memcpy(plane_host, eng.text_planes()[0], plane_host.nbytes, 0, 1)
    d_buf = torch.empty(16 * n, dtype=torch.uint8, device="cuda")
    h_buf = eng.host_array(16 * n, np.uint8)
    c = []
    for _ in range(args.host_reps):
        t0 = time.perf_counter()
        eng.memcpy(d_buf.data_ptr(), h_buf, 16 * n, dev, host)
        c.append(time.perf_counter() - t0)
    print(f"pinned host batch: blocking call median {np.median(t) * 1e3:.1f} ms ({16 * n / np.median(t) / 1e9:.1f} GB/s "
          f"of samples); one pinned cudaMemcpy of the same {16 * n / 1e9:.3f} GB: {np.median(c) * 1e3:.1f} ms "
          f"({16 * n / np.median(c) / 1e9:.1f} GB/s)", flush=True)
    del d_buf

    # ---- the text path on the same samples
    with tempfile.TemporaryDirectory() as d:
        exe = os.path.join(d, "c2_response")
        oracle = os.path.join(ROOT, "oracle")
        subprocess.check_call(["g++", "-O2", "-std=c++17", os.path.join(ROOT, "tests", "cpp", "c2_response.cpp"),
                               "-L", oracle, "-lgpr_oracle", "-Wl,-rpath," + oracle, "-o", exe])
        path = os.path.join(d, "util.json")
        subprocess.check_call([exe, path, "0", str(SEED), str(P), str(G), str(T), str(T0), "0", str(T)])
        size = os.path.getsize(path)
        text = eng.host_array(size, np.uint8)
        with open(path, "rb") as f:
            f.readinto(memoryview(text))
    order = torch.nonzero(counts > 0).flatten().cpu().numpy()
    t_scan, t_parse = [], []
    for _ in range(args.host_reps + 1):
        t0 = time.perf_counter()
        opens, closes = eng.text_scan(text, slot=0)
        t1 = time.perf_counter()
        sp = np.zeros(len(opens), g.IdleEngine.SPAN_DTYPE)
        sp["begin"] = opens + 12
        sp["end"] = closes[np.searchsorted(closes, opens + 12)] + 2
        sp["row"] = order
        t2 = time.perf_counter()
        out = eng.text_parse(sp, T_END, 1, T, rows, slot=0)
        t3 = time.perf_counter()
        t_scan.append(t1 - t0)
        t_parse.append(t3 - t2)
    assert len(opens) == len(order) and not (out["flags"] & 2).any()
    plane_text = np.empty((rows, T), np.uint32)
    eng.memcpy(plane_text, eng.text_planes()[0], plane_text.nbytes, 0, 1)
    ts_, tp_ = np.median(t_scan[1:]), np.median(t_parse[1:])
    print(f"text path, same samples ({size / 1e9:.3f} GB of pinned JSON): gpr_text_scan median {ts_ * 1e3:.1f} ms + "
          f"gpr_text_parse median {tp_ * 1e3:.1f} ms = {(ts_ + tp_) * 1e3:.1f} ms", flush=True)
    print(f"planes identical: device vs text {np.array_equal(plane_dev, plane_text)}, "
          f"pinned host vs text {np.array_equal(plane_host, plane_text)}", flush=True)
    eng.close()


if __name__ == "__main__":
    main()
