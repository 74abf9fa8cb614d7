"""CPU: `gpu-pruner --query-slice S` (DESIGN.md §8e) on the EMULATED device (tests/cpp/slice_emul.cpp: text_emul.cpp's
device with the source of k_remap_rows, ASan/UBSan), through the binary's FileSource.
A range longer than S seconds is asked as consecutive queries of at most S seconds and merged into the resident ring:
PROF slices first, then UTIL, then POWER, the ring grown when a later slice brings more pods or slots.  Every timeline
runs unsliced and sliced: at every tick of both runs the ring holds exactly the window a fresh full-range ingest yields
(by series identity, every other row empty), a full fetch leaves the one-query shape, and the per-series maxima the
verdict is made of are the same in both runs.  The GPU run through the binary is tests/test_gpu_query_slices.py."""
import json
import os
import random
import subprocess

import pytest

import hostlib as H
import slice_ticks as ST
import ticks as TK
from test_resident_ticks import _series


def build_emul(out_dir, sanitize="address,undefined"):
    import emul_build
    from test_hotpath_emul import _extract
    from test_ring_emul import _extract_ring
    d = str(out_dir)
    for name, body in (("text_kernel_extract.inc", emul_build.extract_parse_kernel()),
                       ("hotpath_extract.inc", _extract()), ("ring_extract.inc", _extract_ring())):
        with open(os.path.join(d, name), "w") as f:
            f.write(body)
    out = os.path.join(d, "slice_emul")
    host = os.path.join(H.ROOT, "gpu-pruner_b200", "host")
    cmd = ["g++", "-O1", "-g", "-std=c++20", "-fsanitize=" + sanitize, "-fno-omit-frame-pointer",
           "-fno-sanitize-recover=all", "-DEMUL_PARSE_KERNEL", "-Wno-unknown-pragmas", "-I", host,
           "-I", os.path.join(H.ROOT, "tests", "cpp"), "-I", d, os.path.join(H.ROOT, "tests", "cpp", "slice_emul.cpp")]
    cmd += [os.path.join(host, f) for f in ("ingest.cpp", "ingest_device.cpp", "json.cpp", "controller.cpp", "cli.cpp",
                                            "kube.cpp", "promql.cpp", "snapshot.cpp")]
    subprocess.check_call(cmd + ["-o", out, "-lpthread"])
    return out


@pytest.fixture(scope="module")
def driver(tmp_path_factory):
    return build_emul(tmp_path_factory.mktemp("emul_slices"))


def _run(driver, root, S, duration_min, thr=0, reshape=False, ok=True, **env):
    e = dict(os.environ, ASAN_OPTIONS="detect_leaks=0:abort_on_error=1", **env)
    r = subprocess.run([driver] + (["--reshape"] if reshape else []) + [str(S), str(duration_min), str(thr), str(root)],
                       capture_output=True, text=True, timeout=900, env=e)
    lines = r.stdout.splitlines()
    ticks = [l for l in lines if l.startswith(("OK ", "MISMATCH "))]
    if ok:
        assert r.returncode == 0 and ticks and all(l.startswith("OK ") for l in ticks), (r.stdout[-3000:], r.stderr[-2000:])
    modes = [dict(kv.split("=", 1) for kv in l.split()[1:4]) | {"why": " ".join(l.split()[4:])} for l in ticks]
    total = dict(kv.split("=") for kv in [l for l in lines if l.startswith("TOTAL ")][0].split()[1:])
    return modes, [l for l in lines if l.startswith("MAXIMA ")], {k: int(v) for k, v in total.items()}, r.stderr


def _both(driver, root, S, duration_min, thr=0, reshape=False, **env):
    """the timeline unsliced and sliced at S: the same maxima at every tick, and without --reshape-ring the same path
    (with it, a long delta grows the ring where the unsliced tick reshapes and drops pods: the shapes, and so later
    paths, may differ)"""
    plain, m_plain, _, _ = _run(driver, root, 0, duration_min, thr, reshape, **env)
    sliced, m_sliced, total, err = _run(driver, root, S, duration_min, thr, reshape, **env)
    if not reshape:
        assert [t["mode"] for t in sliced] == [t["mode"] for t in plain]
    assert m_sliced == m_plain
    assert all(t["slices"] == "1" for t in plain)
    return sliced, total


def _lengths(step, duration_min):
    """S = one step, a few steps, a length that does not divide the window, and one at least as long as the window"""
    N = duration_min * 60
    odd = next(k * step for k in range(7, 1000) if N % (k * step))
    return [step, 3 * step, odd, N] if N // step <= 60 else [odd, N]


@pytest.mark.parametrize("step,interval,duration_min", [(1, 20, 1), (5, 45, 2), (15, 180, 30)])
def test_steady_state(driver, tmp_path, step, interval, duration_min):
    rng = random.Random(step * 1000 + interval)
    N = duration_min * 60
    t0 = 1_700_000_000
    times = [t0 + N + k * interval for k in range(5)]
    store = [_series(rng, f"pod-{p}", g, t0 - 50, times[-1] + 10, step, rng.choice(["idle", "busy"]), jitter=step > 1)
             for p in range(6) for g in range(rng.randrange(1, 4))]
    for S in _lengths(step, duration_min):
        root = tmp_path / f"S{S}"
        ST.write_sliced_ticks(str(root), lambda k: store, times, N, step, S)
        sliced, _ = _both(driver, root, S, duration_min)
        assert [t["mode"] for t in sliced] == ["full"] + ["delta"] * 4
        assert int(sliced[0]["slices"]) == -(-N // S)
        assert all(int(t["slices"]) == -(-interval // S) for t in sliced[1:])


def test_series_come_and_go_and_a_late_slot(driver, tmp_path):
    """tests/test_resident_ticks.py's store: the late duplicate needs a third slot, which the unsliced run takes from the
    full range at tick 5; the sliced full range meets it only in its newest slices and grows the ring"""
    rng = random.Random(5)
    N, step, interval = 120, 2, 30
    t0 = 1_700_000_000
    times = [t0 + N + k * interval for k in range(10)]
    horizon = times[-1] + 5
    base = [_series(rng, f"pod-{p}", g, t0, horizon, step, "busy") for p in range(4) for g in range(2)]
    leaves = _series(rng, "leaver", 0, t0, times[2] - 3, step, "idle")
    joins = _series(rng, "joiner", 0, times[3] + 1, horizon, step, "idle")
    second = _series(rng, "pod-0", 1, times[4] + 1, horizon, step, "idle", UUID="GPU-late")
    store = base + [leaves, joins, second]
    for S in (step, 34, 120):
        root = tmp_path / f"S{S}"
        ST.write_sliced_ticks(str(root), lambda k: store, times, N, step, S)
        sliced, total = _both(driver, root, S, 2)
        assert [t["mode"] for t in sliced] == ["full"] + ["delta"] * 4 + ["full"] + ["delta"] * 4
        if S < 120:
            assert total["growths"] > 0   # the leaver lives only in the oldest slices, the joiner in the newest


def test_prof_only_in_older_slices_still_shadows(driver, tmp_path):
    """a PROF series whose samples end early shadows its UTIL series over the whole window (`A or B` looks at the
    whole range); a PROF series that starts late does the same from the newest slices"""
    rng = random.Random(9)
    N, step, interval = 60, 1, 15
    t0 = 1_700_000_000
    times = [t0 + N + k * interval for k in range(4)]
    horizon = times[-1] + 5
    util = [_series(rng, f"pod-{p}", 0, t0, horizon, step, "busy") for p in range(4)]
    early = ("DCGM_FI_PROF_GR_ENGINE_ACTIVE", util[0][1], [(t, 0.0) for t in range(t0, times[0] - 40)])
    late = ("DCGM_FI_PROF_GR_ENGINE_ACTIVE", util[1][1], [(t, 0.0) for t in range(times[0] - 5, horizon)])
    store = util + [early, late]
    for S in (2, 25):
        root = tmp_path / f"S{S}"
        ST.write_sliced_ticks(str(root), lambda k: store, times, N, step, S)
        sliced, _ = _both(driver, root, S, 1)
        assert sliced[0]["mode"] == "full" and int(sliced[0]["slices"]) > 1


def test_oldest_slice_pods_sum_by_groups_and_power(driver, tmp_path):
    """pods that report only in the oldest slice, a `sum by` group whose two members report in different slices, and a
    power plane, with the power threshold the samples are snapped to"""
    rng = random.Random(17)
    N, step, interval = 120, 2, 30
    t0 = 1_700_000_000
    times = [t0 + N + k * interval for k in range(3)]
    horizon = times[-1] + 5
    store = [_series(rng, f"pod-{p}", 0, t0, horizon, step, rng.choice(["idle", "busy"])) for p in range(5)]
    store += [_series(rng, f"old-{p}", 0, times[0] - N + 1, times[0] - N + 20, step, "idle") for p in range(6)]
    store.append(_series(rng, "grp", 0, t0, times[0] - 70, step, "idle", UUID="GPU-a"))
    store.append(_series(rng, "grp", 0, times[0] - 30, horizon, step, "busy", UUID="GPU-b"))
    store += [_series(rng, f"pod-{p}", 0, t0, horizon, step, "x", metric="DCGM_FI_DEV_POWER_USAGE") for p in range(5)]
    for S in (4, 50):
        root = tmp_path / f"S{S}"
        ST.write_sliced_ticks(str(root), lambda k: store, times, N, step, S, with_power=True)
        _both(driver, root, S, 2, thr=150)


def test_hard_span_in_a_middle_slice(driver, tmp_path):
    """values the strict device parser declines (18 digits) only in the middle of the window: the row is re-parsed
    on the CPU and written back in its slice's buckets, which are not the newest"""
    rng = random.Random(23)
    N, step, interval = 60, 1, 15
    t0 = 1_700_000_000
    times = [t0 + N + k * interval for k in range(3)]
    horizon = times[-1] + 5
    store = [_series(rng, f"pod-{p}", 0, t0, horizon, step, "busy") for p in range(3)]
    store.append(("DCGM_FI_DEV_GPU_UTIL", TK.labels("odd", 0),
                  [(t, "123456789012345678" if times[0] - 40 < t <= times[0] - 20 else (1e23 if t % 3 else 0))
                   for t in range(t0, horizon)]))
    root = tmp_path / "S10"
    ST.write_sliced_ticks(str(root), lambda k: store, times, N, step, 10)
    _, total = _both(driver, root, 10, 1)
    assert total["older_patches"] > 0


def test_restore_then_a_delta_longer_than_the_slice(driver, tmp_path):
    """a restart with the window saved after tick 1 (save_state, the ring kept aside, restore_state into a new session),
    down for 100 s: the first delta after the restore is asked as five slices and merged into the restored ring, with
    the restored pods, known series, PROF rows and head-room; a pod that joined while the process was down gets a row"""
    rng = random.Random(31)
    N, step = 120, 2
    t0 = 1_700_000_000
    times = [t0 + N, t0 + N + 30, t0 + N + 30 + 100, t0 + N + 160]
    horizon = times[-1] + 5
    store = [_series(rng, f"pod-{p}", g, t0, horizon, step, rng.choice(["idle", "busy"])) for p in range(4) for g in range(2)]
    store.append(("DCGM_FI_PROF_GR_ENGINE_ACTIVE", store[0][1], [(t, 0.0) for t in range(t0, horizon, step)]))
    store.append(_series(rng, "during", 0, times[1] + 10, times[1] + 40, step, "idle"))   # joins while "down"
    store += [_series(rng, f"pod-{p}", 0, t0, horizon, step, "x", metric="DCGM_FI_DEV_POWER_USAGE") for p in range(4)]
    root = tmp_path / "S20"
    ST.write_sliced_ticks(str(root), lambda k: store, times, N, step, 20, with_power=True)
    sliced, total = _both(driver, root, 20, 2, thr=150, EMUL_RESTORE_BEFORE="2")
    assert total["restores"] == 1
    assert [t["mode"] for t in sliced] == ["full", "delta", "delta", "delta"]
    assert sliced[2]["slices"] == "5"


def test_a_recorded_slice_for_another_range_fails_the_tick(driver, tmp_path):
    rng = random.Random(41)
    N, step, interval = 60, 1, 15
    t0 = 1_700_000_000
    times = [t0 + N + k * interval for k in range(4)]
    store = [_series(rng, f"pod-{p}", 0, t0, times[-1] + 5, step, "busy") for p in range(3)]
    ST.write_sliced_ticks(str(tmp_path), lambda k: store, times, N, step, 5)
    q = tmp_path / "tick-0002" / "delta" / "slice-0001" / "query.json"
    meta = json.loads(q.read_text())
    q.write_text(json.dumps(dict(meta, start=meta["start"] - 1)))
    modes, _, _, _ = _run(driver, tmp_path, 5, 1)
    assert [t["mode"] for t in modes] == ["full", "delta", "failed", "full"]
    a, b = meta["start"], meta["end"]
    assert f"answers ({a - 1}, {b}], the query asks for ({a}, {b}]" in modes[2]["why"], modes[2]


def test_a_slice_that_is_not_a_whole_number_of_steps_fails_the_tick(driver, tmp_path):
    rng = random.Random(43)
    N, step, interval = 60, 5, 15
    t0 = 1_700_000_000
    times = [t0 + N + k * interval for k in range(2)]
    store = [_series(rng, f"pod-{p}", 0, t0, times[-1] + 5, step, "busy") for p in range(3)]
    ST.write_sliced_ticks(str(tmp_path), lambda k: store, times, N, step, 7)
    modes, _, _, _ = _run(driver, tmp_path, 7, 1)
    assert [t["mode"] for t in modes] == ["failed", "failed"]
    assert "--query-slice 7 s is not a whole number of the query step (5 s)" in modes[0]["why"]


def test_fuzz_timelines(driver, tmp_path):
    """random clusters with PROF and power series, gaps, waves of short-lived pods and late slots, sliced at a random
    multiple of the step, with and without --reshape-ring"""
    for seed in range(8):
        rng = random.Random(3000 + seed)
        step = rng.choice([1, 2, 10])
        duration_min = rng.choice([1, 2])
        N = duration_min * 60
        interval = step * rng.randrange(2, 12)
        t0 = 1_700_000_000 + rng.randrange(1000)
        times = [t0 + N + k * interval for k in range(rng.randrange(4, 8))]
        horizon = times[-1] + 5
        store = []
        for p in range(rng.randrange(2, 7)):
            for g in range(rng.randrange(1, 4)):
                a = rng.choice([t0, t0, rng.randrange(t0, horizon)])
                b = rng.choice([horizon, horizon, rng.randrange(a, horizon + 1)])
                store.append(_series(rng, f"p{p}", g, a, b, step, rng.choice(["idle", "busy"]), jitter=rng.random() < 0.5))
                if rng.random() < 0.2:
                    store.append(_series(rng, f"p{p}", g, a, b, step, "busy", metric="DCGM_FI_PROF_GR_ENGINE_ACTIVE"))
                if rng.random() < 0.5:
                    store.append(_series(rng, f"p{p}", g, a, b, step, "x", metric="DCGM_FI_DEV_POWER_USAGE"))
        for w in range(rng.randrange(0, 3)):
            at = rng.randrange(t0, horizon)
            store += [_series(rng, f"w{w}-{j}", rng.randrange(3), at, at + interval, step, "idle")
                      for j in range(rng.randrange(20, 90))]
        if rng.random() < 0.5:
            store.append(_series(rng, "p0", 7, rng.randrange(t0, horizon), horizon, step, "idle", UUID="GPU-late"))
        S = step * rng.choice([1, 2, 3, 7, 11])
        d = tmp_path / f"s{seed}"
        ST.write_sliced_ticks(str(d), lambda k: store, times, N, step, S, with_power=True,
                              skip_delta={rng.randrange(1, len(times))} if rng.random() < 0.3 else ())
        _both(driver, d, S, duration_min, thr=150, reshape=rng.random() < 0.5)


# ---- CLI ---------------------------------------------------------------------------------------------------------------
def test_cli_query_slice():
    assert H.parse_cli(["--prometheus-url", "file:///x", "--query-slice", "180"])["ok"]
    assert H.parse_cli(["--prometheus-url", "file:///x", "-d", "--query-slice=60"])["ok"]
    for bad in ("-5", "1.5", "x", ""):
        r = H.parse_cli(["--prometheus-url", "file:///x", "--query-slice", bad])
        assert not r["ok"] and r["exit_code"] == 2 and "--query-slice" in r["message"], bad
    r = H.parse_cli(["--prometheus-url", "file:///x", "--query-slice"])
    assert not r["ok"] and r["exit_code"] == 2
    assert "--query-slice <SECONDS>" in H.parse_cli(["--help"])["message"]


def test_cli_query_slice_leaves_the_query_alone():
    base = ["--prometheus-url", "file:///x", "-d", "-t", "5", "--power-threshold", "150"]
    assert H.render_selectors(base + ["--query-slice", "60"]) == H.render_selectors(base)
    assert H.render_query(base + ["--query-slice", "60"]) == H.render_query(base)


def test_binary_query_slice_flag():
    if not os.path.exists(H.BIN):
        pytest.skip("gpu-pruner binary not built")
    p = subprocess.run([H.BIN, "--help"], capture_output=True, text=True)
    assert p.returncode == 0 and "--query-slice" in p.stdout
    p = subprocess.run([H.BIN, "--prometheus-url", "file:///x", "--query-slice", "-1"], capture_output=True, text=True)
    assert p.returncode == 2 and "--query-slice" in p.stderr
