"""gpr_chunks_scatter at C2 size (10,000 pods x 4 GPUs x 1,800 samples of the synthetic universe, DESIGN.md §7): every
present util cell one sample at its bucket's timestamp, each series cut into Prometheus XOR chunks of 120 samples by
the encoder of tests/cpp/chunks_encode.cpp.

    python tools/chunks_bench.py [--reps 50]

Prints the card (nvidia-smi, read-only query) and then:
  * bytes per sample of the chunks (counted on the CPU), against 16 B for decoded samples and the text's bytes;
  * device batch: k_chunks_scatter kernel time (torch.profiler CUDA activity, median of --reps calls) and its modelled
    bytes per second (chunk bytes + 16 B of offsets per chunk + 4 B merged per in-window sample); the whole blocking
    call (check kernel, fill, scatter, read-back) by host clock;
  * pinned host batch: the blocking call against one pinned cudaMemcpy of the same chunk bytes;
  * the same samples through gpr_samples_scatter (pinned) and through the text path (pinned JSON, scan + parse), in
    the same run, and whether all paths leave identical planes.
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
sys.path.insert(0, os.path.join(ROOT, "tests"))
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
    import chunks_ref
    eng = g.IdleEngine(device=0)
    rows = P * G
    util = torch.empty((rows, T), dtype=torch.float32, device="cuda")
    eng.synth_fill(SEED, 0, util, 0, P, G, T)
    present = ~torch.isnan(util)
    counts = present.sum(1)
    r_idx, c_idx = present.nonzero(as_tuple=True)
    ts = ((T_END - (T - 1 - c_idx).to(torch.int64)) * 1000).cpu().numpy()
    vals = util[r_idx, c_idx].to(torch.float64).cpu().numpy()
    offsets = np.zeros(rows + 1, np.uint64)
    offsets[1:] = np.cumsum(counts.cpu().numpy())
    n = int(offsets[-1])
    del r_idx, c_idx, present
    t0 = time.perf_counter()
    sc, cb, data = chunks_ref.encode_native(offsets, ts, vals.view(np.uint64), 120)
    n_chunks, n_bytes = len(cb) - 1, len(data)
    print(f"batch: {rows} series, {n} samples, {n_chunks} chunks of up to 120 samples; encoded on the CPU in "
          f"{time.perf_counter() - t0:.1f} s", flush=True)
    print(f"bytes per sample: chunk data {n_bytes / n:.3f} B ({n_bytes / 1e6:.1f} MB); with chunk_bytes and "
          f"series_chunks {(n_bytes + 8 * (n_chunks + 1) + 12 * rows) / n:.3f} B; decoded samples 16 B", flush=True)
    r_ids = np.arange(rows, dtype=np.uint32)

    def chunks(s, r, c, d, kind):
        return eng.chunks_scatter(s, r, c, d, T_END, 1, T, rows, mem_kind=kind, n_series=rows)

    def plane():
        out = np.empty((rows, T), np.uint32)
        eng.memcpy(out, eng.text_planes()[0], out.nbytes, 0, 1)
        return out

    # ---- device batch
    dev, host = g.ffi.GPR_MEM_DEVICE, g.ffi.GPR_MEM_HOST
    d_sc, d_rows = torch.from_numpy(sc.view(np.int64)).cuda(), torch.from_numpy(r_ids.view(np.int32)).cuda()
    d_cb, d_data = torch.from_numpy(cb.view(np.int64)).cuda(), torch.from_numpy(data).cuda()
    torch.cuda.synchronize()   # the context's stream is not ordered with torch's
    for _ in range(5):
        st = chunks(d_sc, d_rows, d_cb, d_data, dev)
    assert st["n_oow"] == 0 and st["n_in"] == n, st
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(args.reps):
            chunks(d_sc, d_rows, d_cb, d_data, dev)
        torch.cuda.synchronize()
    k_us = [e.device_time for e in prof.events() if "k_chunks_scatter" in e.name]
    c_us = [e.device_time for e in prof.events() if "k_chunks_check" in e.name]
    assert len(k_us) == args.reps, len(k_us)
    k_ms = float(np.median(k_us)) / 1e3
    bytes_model = n_bytes + 16 * n_chunks + 4 * n
    print(f"device batch: k_chunks_scatter median {k_ms:.3f} ms over {args.reps} calls (min {min(k_us) / 1e3:.3f}, "
          f"max {max(k_us) / 1e3:.3f}); modelled {bytes_model / 1e9:.3f} GB -> {bytes_model / k_ms / 1e6:.0f} GB/s = "
          f"{bytes_model / k_ms * 1e3 / HBM:.3f} of 3.35 TB/s; {n / k_ms / 1e6:.2f} G samples/s; k_chunks_check "
          f"median {np.median(c_us) / 1e3:.3f} ms", flush=True)
    t = []
    for _ in range(10):
        t0 = time.perf_counter()
        chunks(d_sc, d_rows, d_cb, d_data, dev)
        t.append(time.perf_counter() - t0)
    print(f"device batch: whole blocking call median {np.median(t) * 1e3:.3f} ms (series check, chunk check, fill, "
          f"scatter, read-backs)", flush=True)
    plane_dev = plane()

    # ---- pinned host batch
    h_data = eng.host_array(n_bytes, np.uint8)
    h_data[:] = data
    chunks(sc, r_ids, cb, h_data, host)
    t = []
    for _ in range(args.host_reps):
        t0 = time.perf_counter()
        chunks(sc, r_ids, cb, h_data, host)
        t.append(time.perf_counter() - t0)
    plane_host = plane()
    c = []
    for _ in range(args.host_reps):
        t0 = time.perf_counter()
        eng.memcpy(d_data.data_ptr(), h_data, n_bytes, dev, host)
        c.append(time.perf_counter() - t0)
    pieces = -(-n_bytes // (32 << 20))
    print(f"pinned host batch: blocking call median {np.median(t) * 1e3:.2f} ms ({pieces} pieces of <= 32 MB, "
          f"{'checked and merged from the staging' if pieces <= 2 else 'uploaded twice: checked, then merged'}); "
          f"one pinned cudaMemcpy of the same {n_bytes / 1e6:.1f} MB: {np.median(c) * 1e3:.2f} ms", flush=True)

    # ---- the same samples through gpr_samples_scatter and the text path
    h_ts, h_vals = eng.host_array(n, np.int64), eng.host_array(n, np.float64)
    h_ts[:], h_vals[:] = ts, vals
    eng.samples_scatter(offsets, r_ids, h_ts, h_vals, T_END, 1, T, rows)
    t = []
    for _ in range(args.host_reps):
        t0 = time.perf_counter()
        eng.samples_scatter(offsets, r_ids, h_ts, h_vals, T_END, 1, T, rows)
        t.append(time.perf_counter() - t0)
    plane_samples = plane()
    print(f"same samples, pinned, gpr_samples_scatter: median {np.median(t) * 1e3:.1f} ms ({16 * n / 1e9:.3f} GB)",
          flush=True)
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
    order = np.flatnonzero(counts.cpu().numpy() > 0)
    t_all = []
    for _ in range(args.host_reps + 1):
        t0 = time.perf_counter()
        opens, closes = eng.text_scan(text, slot=0)
        sp = np.zeros(len(opens), g.IdleEngine.SPAN_DTYPE)
        sp["begin"] = opens + 12
        sp["end"] = closes[np.searchsorted(closes, opens + 12)] + 2
        sp["row"] = order
        out = eng.text_parse(sp, T_END, 1, T, rows, slot=0)
        t_all.append(time.perf_counter() - t0)
    assert len(opens) == len(order) and not (out["flags"] & 2).any()
    plane_text = plane()
    print(f"same samples as text ({size / 1e9:.3f} GB of pinned JSON, {size / n:.2f} B per sample): scan + span "
          f"table + parse median {np.median(t_all[1:]) * 1e3:.1f} ms", flush=True)
    print(f"planes identical: chunks device vs text {np.array_equal(plane_dev, plane_text)}, chunks pinned vs text "
          f"{np.array_equal(plane_host, plane_text)}, samples vs text {np.array_equal(plane_samples, plane_text)}",
          flush=True)
    eng.close()


if __name__ == "__main__":
    main()
