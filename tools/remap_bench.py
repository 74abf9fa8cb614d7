"""gpr_resident_remap at C2 size: the ring of 10,000 pods x 4 GPUs x 1,800 samples of the synthetic universe (DESIGN.md
§7) with the power plane and the block index (0.6 GB), widened to G = 5 and grown by 25 % to 12,500 pods, against
rebuilding that ring from the full range as text.

    python tools/remap_bench.py [--reps 50]

Prints the card (nvidia-smi, read-only query) and then:
  * the remap: each timed call takes [10,000][4] to [12,500][5] (old pods keep their slots, in shuffled order; the new
    slot and the new pods have no source), and an untimed call takes it back.  The context runs on a caller-owned
    stream, so CUDA events recorded on it before and after the call time the whole call as the GPU sees it (the
    allocation of the new ring included); the host clock times the blocking call; torch.profiler gives the four
    k_remap_rows gathers per call.  Bytes moved: every live new row read and written, every new row without a source
    written, the map read; as a rate and as a share of the H100 SXM data sheet's 3.35 TB/s;
  * the rebuild the remap replaces: gpr_resident_init of the new shape, then the util and the power range-query
    responses of the same window (compact matrix JSON of tests/cpp/c2_response.cpp, pinned) through gpr_text_scan +
    gpr_text_parse(GPR_TEXT_RESIDENT), then gpr_resident_reindex; and whether its util plane equals the remapped one.
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
SEED, P0, G0, T = 0x5EED0002, 10000, 4, 1800
P1, G1 = 12500, 5
T0 = 1_700_000_000
T_END = T0 + T - 1
HBM = 3.35e12
NONE = 0xFFFFFFFF


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--text-reps", type=int, default=3)
    args = ap.parse_args()
    print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv"],
                         capture_output=True, text=True).stdout.strip(), flush=True)
    import torch
    import gpu_pruner_b200 as g
    stream = torch.cuda.Stream()
    eng = g.IdleEngine(device=0, stream=stream.cuda_stream)
    eng.resident_init(P0, G0, T, power_plane=True, block_index=True)
    u, p, _ = eng.resident_planes()
    eng.synth_fill(SEED, 0, u, 0, P0, G0, T)
    eng.synth_fill(SEED, 1, p, 0, P0, G0, T)
    eng.resident_reindex()

    rng = np.random.default_rng(1)
    fwd = np.full((P1, G1), NONE, np.uint32)
    fwd[rng.permutation(P0), :G0] = np.arange(P0 * G0, dtype=np.uint32).reshape(P0, G0)
    fwd = fwd.ravel()
    back = np.full(P0 * G0, NONE, np.uint32)
    live = fwd != NONE
    back[fwd[live]] = np.flatnonzero(live).astype(np.uint32)
    d_fwd = torch.from_numpy(fwd.view(np.int32)).cuda()
    d_back = torch.from_numpy(back.view(np.int32)).cuda()
    torch.cuda.synchronize()
    idx_ld = ((T + 63) // 64 + 3) // 4 * 4
    n_live, n_new = int(live.sum()), P1 * G1
    bytes_moved = 2 * (2 * n_live * T * 4 + (n_new - n_live) * T * 4) + \
        2 * (2 * n_live * idx_ld * 4 + (n_new - n_live) * idx_ld * 4) + n_new * 4
    old_bytes = 2 * P0 * G0 * (T + idx_ld) * 4
    new_bytes = 2 * n_new * (T + idx_ld) * 4
    print(f"ring: [{P0}][{G0}][{T}] util + power + index = {old_bytes / 1e9:.3f} GB -> [{P1}][{G1}][{T}] = "
          f"{new_bytes / 1e9:.3f} GB; {n_live} live rows of {n_new}; {bytes_moved / 1e9:.3f} GB moved per remap",
          flush=True)

    def remap(P, G, m):
        eng.resident_remap(P, G, m)

    for _ in range(3):
        remap(P1, G1, d_fwd)
        remap(P0, G0, d_back)
    ev_ms, host_ms = [], []
    for _ in range(args.reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(stream)
        t0 = time.perf_counter()
        remap(P1, G1, d_fwd)
        t1 = time.perf_counter()
        b.record(stream)
        b.synchronize()
        ev_ms.append(a.elapsed_time(b))
        host_ms.append((t1 - t0) * 1e3)
        remap(P0, G0, d_back)
    ev, hm = float(np.median(ev_ms)), float(np.median(host_ms))
    print(f"remap, whole call: CUDA events median {ev:.3f} ms over {args.reps} calls (min {min(ev_ms):.3f}, max "
          f"{max(ev_ms):.3f}); host clock median {hm:.3f} ms; {bytes_moved / ev / 1e6:.0f} GB/s = "
          f"{bytes_moved / ev * 1e3 / HBM:.2f} of 3.35 TB/s", flush=True)
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA], acc_events=True) as prof:
        for _ in range(10):
            remap(P1, G1, d_fwd)
            remap(P0, G0, d_back)
        torch.cuda.synchronize()
    k = [e.device_time for e in prof.events() if "k_remap_rows" in e.name]
    assert len(k) == 80, len(k)
    k_fwd = [sum(k[i:i + 4]) / 1e3 for i in range(0, 80, 8)]    # the four gathers of each forward call
    kf = float(np.median(k_fwd))
    print(f"remap, the four k_remap_rows gathers of a forward call: median {kf:.3f} ms; "
          f"{bytes_moved / kf / 1e6:.0f} GB/s = {bytes_moved / kf * 1e3 / HBM:.2f} of 3.35 TB/s", flush=True)
    remap(P1, G1, d_fwd)
    u, _, _ = eng.resident_planes()
    remapped = np.empty((n_new, T), np.uint32)
    eng.memcpy(remapped, u, remapped.nbytes, 0, 1)

    # ---- the rebuild from the full range, as text
    with tempfile.TemporaryDirectory() as d:
        exe = os.path.join(d, "c2_response")
        oracle = os.path.join(ROOT, "oracle")
        subprocess.check_call(["g++", "-O2", "-std=c++17", os.path.join(ROOT, "tests", "cpp", "c2_response.cpp"),
                               "-L", oracle, "-lgpr_oracle", "-Wl,-rpath," + oracle, "-o", exe])
        texts = []
        for plane in (0, 1):
            path = os.path.join(d, f"plane{plane}.json")
            subprocess.check_call([exe, path, str(plane), str(SEED), str(P0), str(G0), str(T), str(T0), "0", str(T)])
            size = os.path.getsize(path)
            text = eng.host_array(size, np.uint8)
            with open(path, "rb") as f:
                f.readinto(memoryview(text))
            texts.append(text)
    print(f"text: util {texts[0].size / 1e9:.3f} GB + power {texts[1].size / 1e9:.3f} GB of pinned JSON", flush=True)
    counts = []
    for plane in (0, 1):
        tmp = torch.empty((P0 * G0, T), dtype=torch.float32, device="cuda")
        eng.synth_fill(SEED, plane, tmp, 0, P0, G0, T)
        torch.cuda.synchronize()
        counts.append((~torch.isnan(tmp)).sum(1).cpu().numpy())
        del tmp
    t_all = []
    for _ in range(args.text_reps + 1):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        eng.resident_init(P1, G1, T, power_plane=True, block_index=True)
        for plane in (0, 1):
            opens, closes = eng.text_scan(texts[plane], slot=plane)
            sp = np.zeros(len(opens), g.IdleEngine.SPAN_DTYPE)
            sp["begin"] = opens + 12
            sp["end"] = closes[np.searchsorted(closes, opens + 12)] + 2
            sp["row"] = back[np.flatnonzero(counts[plane] > 0)]
            eng.text_parse(sp, T_END, 1, T, n_new, slot=plane, plane=plane, resident=True,
                           power_threshold=150.0 if plane else 0.0)
        eng.resident_reindex()
        t_all.append(time.perf_counter() - t0)
    tr = float(np.median(t_all[1:])) * 1e3
    u, _, _ = eng.resident_planes()
    rebuilt = np.empty((n_new, T), np.uint32)
    eng.memcpy(rebuilt, u, rebuilt.nbytes, 0, 1)
    print(f"rebuild from the full range (init + util and power text scan and parse + reindex): median {tr:.1f} ms "
          f"over {args.text_reps} runs; {tr / ev:.0f}x the remap's CUDA-event time", flush=True)
    # an absent sample is 0xFFFFFFFF in the rebuilt ring and whatever NaN the synthetic generator wrote in the remapped
    # one: the planes agree when every cell has the same bits or both cells are NaN
    fa, fb = rebuilt.view(np.float32), remapped.view(np.float32)
    differ = int((~((rebuilt == remapped) | (np.isnan(fa) & np.isnan(fb)))).sum())
    print(f"util plane of the rebuild vs the remap: {differ} cells differ (NaN = no sample in both counts as equal)",
          flush=True)
    eng.close()


if __name__ == "__main__":
    main()
