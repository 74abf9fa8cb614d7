"""CPU: `gpu-pruner -d --retime-ring` (IngestOptions::retime, DESIGN.md §8e) on the EMULATED device
(tests/cpp/retime_ticks_emul.cpp: text_emul.cpp's device with the sources of k_retime_rows, k_live_rows, k_remap_rows and
k_ring_cols under the CPU shim, ASan/UBSan), through the binary's FileSource (controller.cpp).
A delta tick whose query step grew by a whole factor, or whose --duration got shorter on an edge of the old step's
buckets, retimes the ring on the GPU instead of fetching the full range; every other change of step or window takes the
full range as before, and says why.

Every timeline runs twice, with and without the option.  At every tick of both runs the ring holds exactly the window of
a fresh full-range ingest at that tick's step and duration (the driver compares every series' row by identity and
requires every other row to be empty), the per-series maxima (MAXIMA lines) are the same in both runs, and the retime
log lines are the ones the plan gives.  The C ABI on the GPU is tests/test_gpu_resident_retime.py."""
import os
import random
import subprocess

import pytest

import hostlib as H
import retime_ticks as RT
import ticks as TK
from test_resident_ticks import _series

T0 = 1_700_000_000
RETIMED = "Resident window retimed on the GPU: "
REBUILT = "Resident window rebuilt from the full range: "


def build_emul(out_dir, sanitize="address,undefined"):
    import emul_build
    from test_hotpath_emul import _extract
    from test_ring_emul import _extract_ring
    d = str(out_dir)
    for name, body in (("text_kernel_extract.inc", emul_build.extract_parse_kernel()),
                       ("hotpath_extract.inc", _extract()), ("ring_extract.inc", _extract_ring())):
        with open(os.path.join(d, name), "w") as f:
            f.write(body)
    out = os.path.join(d, "retime_ticks_emul")
    host = os.path.join(H.ROOT, "gpu-pruner_b200", "host")
    cmd = ["g++", "-O1", "-g", "-std=c++20", "-fsanitize=" + sanitize, "-fno-omit-frame-pointer",
           "-fno-sanitize-recover=all", "-DEMUL_PARSE_KERNEL", "-Wno-unknown-pragmas", "-I", host,
           "-I", os.path.join(H.ROOT, "tests", "cpp"), "-I", d,
           os.path.join(H.ROOT, "tests", "cpp", "retime_ticks_emul.cpp")]
    cmd += [os.path.join(host, f) for f in ("ingest.cpp", "ingest_device.cpp", "json.cpp", "controller.cpp", "cli.cpp",
                                            "kube.cpp", "promql.cpp", "snapshot.cpp")]
    subprocess.check_call(cmd + ["-o", out, "-lpthread"])
    return out


@pytest.fixture(scope="module")
def driver(tmp_path_factory):
    return build_emul(tmp_path_factory.mktemp("emul_retime"))


def _run(driver, root, duration_min, retime, L=0, S=0, thr=0, **env):
    e = dict(os.environ, ASAN_OPTIONS="detect_leaks=0:abort_on_error=1", **env)
    r = subprocess.run([driver] + (["--retime"] if retime else []) + [str(L), str(S), str(duration_min), str(thr),
                                                                        str(root)],
                       capture_output=True, text=True, timeout=900, env=e)
    lines = r.stdout.splitlines()
    ticks = [l for l in lines if l.startswith(("OK ", "MISMATCH "))]
    assert r.returncode == 0 and ticks and all(l.startswith("OK ") for l in ticks), (r.stdout[-3000:], r.stderr[-2000:])
    modes = [dict(kv.split("=", 1) for kv in l.split()[1:4]) for l in ticks]
    log = r.stderr.splitlines()
    retimes = [l[l.index(RETIMED):] for l in log if RETIMED in l]
    rebuilt = [l[l.index(REBUILT) + len(REBUILT):] for l in log if REBUILT in l]
    return modes, [l for l in lines if l.startswith("MAXIMA ")], retimes, rebuilt


def _both(driver, root, duration_min, L=0, S=0, thr=0, **env):
    """the timeline with and without --retime-ring: the same maxima at every tick, no retime without the option"""
    plain, m_plain, r_plain, _ = _run(driver, root, duration_min, False, L, S, thr, **env)
    res, m_res, retimes, rebuilt = _run(driver, root, duration_min, True, L, S, thr, **env)
    assert m_res == m_plain
    assert r_plain == [] and len(res) == len(plain) and res[0]["mode"] == "full"
    return res, plain, retimes, rebuilt


def _store(rng, t1, step, n_pods=5, power=False, prof_pod=None, prof_until=None):
    store = [_series(rng, f"pod-{p}", g, T0 - 50, t1, step, rng.choice(["idle", "busy"]), jitter=step > 1)
             for p in range(n_pods) for g in range(1 + p % 2)]
    if power:
        store += [_series(rng, f"pod-{p}", 0, T0 - 50, t1, step, "x", metric="DCGM_FI_DEV_POWER_USAGE")
                  for p in range(n_pods)]
    if prof_pod is not None:
        store.append(_series(rng, f"pod-{prof_pod}", 0, T0 - 50, prof_until or t1, step, "busy",
                             metric="DCGM_FI_PROF_GR_ENGINE_ACTIVE"))
    return store


def _timeline(tmp_path, name, steps, durations, interval, L=0, S=0, power=False, seed=1, n_pods=5, **kw):
    rng = random.Random(seed)
    times = [T0 + 120 + k * interval for k in range(len(steps))]
    store = kw.pop("store", None) or _store(rng, times[-1] + 5, min(steps), n_pods, power, **kw)
    root = tmp_path / name
    RT.write_retime_ticks(str(root), store, times, steps, durations, L=L, S=S, power=power)
    return root


@pytest.mark.parametrize("k", [2, 3])
def test_step_grows_by_a_whole_factor(driver, tmp_path, k):
    steps = [5] * 3 + [5 * k] * 4
    root = _timeline(tmp_path, f"x{k}", steps, [2] * 7, 30)
    res, plain, retimes, _ = _both(driver, root, 2)
    assert [t["mode"] for t in plain] == ["full"] * 1 + ["delta"] * 2 + ["full"] + ["delta"] * 3
    assert [t["mode"] for t in res] == ["full"] + ["delta"] * 6
    assert len(retimes) == 1 and retimes[0].startswith(RT.retime_line(24, 5, 120, 5 * k, 120))
    assert res[3]["T"] == str(-(-120 // (5 * k)))


def test_step_x2_with_query_slices(driver, tmp_path):
    root = _timeline(tmp_path, "slices", [5, 5, 10, 10, 10], [2] * 5, 40, S=20)
    res, _, retimes, _ = _both(driver, root, 2, S=20)
    assert [t["mode"] for t in res] == ["full"] + ["delta"] * 4 and len(retimes) == 1


@pytest.mark.parametrize("L", [15, 20])
def test_step_x2_with_late_seconds(driver, tmp_path, L):
    root = _timeline(tmp_path, f"late{L}", [5, 5, 10, 10, 10], [2] * 5, 30, L=L)
    res, _, retimes, _ = _both(driver, root, 2, L=L)
    assert [t["mode"] for t in res] == ["full"] + ["delta"] * 4 and len(retimes) == 1


def test_step_x2_with_a_reshape_in_the_same_tick(driver, tmp_path):
    rng = random.Random(9)
    times = [T0 + 120 + k * 30 for k in range(5)]
    store = _store(rng, times[-1] + 5, 5, n_pods=3)
    store += [_series(rng, f"new-{p}", 0, times[1] + 1, times[-1] + 5, 5, "idle") for p in range(80)]   # joins at 2
    root = tmp_path / "reshape"
    RT.write_retime_ticks(str(root), store, times, [5, 5, 10, 10, 10], [2] * 5)
    res, _, retimes, _ = _both(driver, root, 2, EMUL_RESHAPE="1")
    assert [t["mode"] for t in res] == ["full"] + ["delta"] * 4 and len(retimes) == 1


def test_step_x2_with_the_power_plane(driver, tmp_path):
    root = _timeline(tmp_path, "power", [5, 5, 10, 10], [2] * 4, 30, power=True)
    res, _, retimes, _ = _both(driver, root, 2, thr=150)
    assert [t["mode"] for t in res] == ["full"] + ["delta"] * 3 and len(retimes) == 1


@pytest.mark.parametrize("steps,why", [([10, 10, 5, 5], "the step got finer"),
                                       ([10, 10, 15, 15], "not a whole multiple")])
def test_finer_and_fractional_steps_take_the_full_range(driver, tmp_path, steps, why):
    root = _timeline(tmp_path, "s%d" % steps[2], steps, [2] * 4, 30)
    res, _, retimes, rebuilt = _both(driver, root, 2)
    assert [t["mode"] for t in res] == ["full", "delta", "full", "delta"] and retimes == []
    assert rebuilt == ["step / window length changed (%s)" % why] or why in rebuilt[0], rebuilt


def test_prof_series_only_in_the_dropped_part_takes_the_full_range(driver, tmp_path):
    """--duration 2 -> 1 at tick 2: pod-0's PROF series stopped reporting 90 s before it, so it has samples in the old
    window and none in the new one.  (Tick 1 already rebuilds: the series is missing from its slice.)"""
    times = [T0 + 120 + k * 30 for k in range(4)]
    root = _timeline(tmp_path, "prof", [5] * 4, [2, 2, 1, 1], 30, prof_pod=0, prof_until=times[2] - 90)
    res, _, retimes, rebuilt = _both(driver, root, 2)
    assert res[2]["mode"] == "full" and retimes == []
    assert rebuilt[-1] == "a DCGM_FI_PROF_GR_ENGINE_ACTIVE series has no sample left in the retimed window", rebuilt


def test_shorter_duration_mid_run_is_retimed(driver, tmp_path):
    root = _timeline(tmp_path, "dur", [5] * 5, [2, 2, 1, 1, 1], 30)
    res, _, retimes, _ = _both(driver, root, 2)
    assert [t["mode"] for t in res] == ["full"] + ["delta"] * 4
    assert retimes and retimes[0].startswith(RT.retime_line(24, 5, 120, 5, 60))


def test_restart_from_a_longer_window_is_retimed(driver, tmp_path):
    """a session saved at --duration 2 and restored at --duration 1 (as --snapshot-file restores it with the flag):
    the first delta retimes it"""
    root = _timeline(tmp_path, "restart", [5] * 5, [2, 2, 2, 1, 1], 30)
    res, _, retimes, _ = _both(driver, root, 2, EMUL_RESTORE_BEFORE="3")
    assert [t["mode"] for t in res] == ["full"] + ["delta"] * 4 and len(retimes) == 1


def test_restart_into_a_longer_window_takes_the_full_range(driver, tmp_path):
    root = _timeline(tmp_path, "longer", [5] * 5, [1, 1, 1, 2, 2], 30)
    res, _, retimes, rebuilt = _both(driver, root, 1, EMUL_RESTORE_BEFORE="3")
    assert res[3]["mode"] == "full" and retimes == [] and "the window got longer" in rebuilt[0]


def test_shorter_window_that_cuts_a_bucket_takes_the_full_range(driver, tmp_path):
    """step 8: a window of 120 s is 15 buckets, and 60 s ends inside one of them"""
    root = _timeline(tmp_path, "cut", [8] * 3, [2, 2, 1], 32)
    res, _, retimes, rebuilt = _both(driver, root, 2)
    assert res[2]["mode"] == "full" and retimes == [] and "cuts a bucket" in rebuilt[0]


def test_a_failed_retime_takes_the_full_range(driver, tmp_path):
    root = _timeline(tmp_path, "fail", [5, 5, 10, 10], [2] * 4, 30)
    res, _, retimes, rebuilt = _both(driver, root, 2, EMUL_FAIL_RETIME="1")
    assert [t["mode"] for t in res] == ["full", "delta", "full", "delta"] and retimes == []
    assert "could not be retimed" in rebuilt[0] and "out of device memory" in rebuilt[0]


def test_fuzz_timelines(driver, tmp_path):
    n_retimed = 0
    for seed in range(12):
        rng = random.Random(7000 + seed)
        s0 = rng.choice([1, 2, 5])
        interval = s0 * 6 * rng.randrange(1, 3)
        steps, durations = [s0], [2]
        for _ in range(rng.randrange(4, 8)):
            s = steps[-1]
            steps.append(rng.choice([s, s, s * 2, s * 3, max(1, s // 2)]) if interval % (s * 6) == 0 else s)
            durations.append(rng.choice([durations[-1]] * 3 + [1, 2]))
        root = _timeline(tmp_path, f"f{seed}", steps, durations, interval, seed=seed, power=rng.random() < 0.5,
                         n_pods=rng.randrange(2, 7), prof_pod=rng.choice([None, 1]))
        L = rng.choice([0, 0, s0 * 2])
        res, _, retimes, _ = _both(driver, root, 2, L=L, thr=150)
        n_retimed += len(retimes)
    assert n_retimed >= 4, n_retimed


# ---- CLI ---------------------------------------------------------------------------------------------------------------
def test_cli_retime_ring_needs_daemon_mode():
    r = H.parse_cli(["--prometheus-url", "file:///x", "--retime-ring"])
    assert not r["ok"] and r["exit_code"] == 2
    assert r["message"].endswith("the argument '--retime-ring' can only be used with '--daemon-mode'") or \
        "the argument '--retime-ring' can only be used with '--daemon-mode'" in r["message"]
    assert H.parse_cli(["--prometheus-url", "file:///x", "-d", "--retime-ring"])["ok"]
    r = H.parse_cli(["--prometheus-url", "file:///x", "-d", "--retime-ring=yes"])
    assert not r["ok"] and r["exit_code"] == 2
    assert "--retime-ring" in H.parse_cli(["--help"])["message"]


def test_cli_retime_ring_leaves_the_query_alone():
    base = ["--prometheus-url", "file:///x", "-d", "-t", "5", "--power-threshold", "150"]
    assert H.render_selectors(base + ["--retime-ring"]) == H.render_selectors(base)


def test_binary_retime_ring_without_daemon_mode_exits_2():
    if not os.path.exists(H.BIN):
        pytest.skip("gpu-pruner binary not built")
    p = subprocess.run([H.BIN, "--prometheus-url", "file:///x", "--retime-ring"], capture_output=True, text=True)
    assert p.returncode == 2 and "--retime-ring" in p.stderr
    p = subprocess.run([H.BIN, "--help"], capture_output=True, text=True)
    assert p.returncode == 0 and "--retime-ring" in p.stdout
