"""CPU: daemon mode with --reshape-ring (IngestOptions::reshape, DESIGN.md §8e) on the EMULATED device
(tests/cpp/reshape_emul.cpp: text_emul.cpp's device with the source of k_live_rows and k_remap_rows under the CPU shim,
ASan/UBSan).
A delta tick whose pods outgrow the ring's rows, or whose pod gains a series slot beyond G, reshapes the ring instead of
fetching the full range: the tick's buckets are opened, the live rows read, pods without a live row or a series in the
slice dropped, the rest remapped to [kept + kept / 4 + 64][max(G, slots needed)] and renumbered.

Every timeline runs twice, with and without the option.  With it, every tick after tick 0 is a delta tick except ticks
whose cause is not a shape cause (a gap, power on / off, a PROF change).  At every tick of both runs the ring holds
exactly the window of a fresh full-range ingest (the driver compares every series' row by identity and requires every
other row to be empty), and the per-series maxima the verdict is made of (its MAXIMA lines) are the same in both runs.
The GPU run of the same through the `gpu-pruner` binary is tests/test_gpu_daemon_reshape.py."""
import os
import random
import subprocess

import pytest

import hostlib as H
import ticks as TK
from test_resident_ticks import _series

SHAPE_CAUSES = ("more pods than the resident window", "GPU slot beyond")


def build_emul(out_dir, sanitize="address,undefined"):
    """tests/cpp/reshape_emul.cpp: text_emul.cpp's kernel flavour plus the source of k_live_rows and k_remap_rows, cut
    out as their own tests cut them"""
    import emul_build
    from test_hotpath_emul import _extract
    from test_ring_emul import _extract_ring
    d = str(out_dir)
    for name, body in (("text_kernel_extract.inc", emul_build.extract_parse_kernel()),
                       ("hotpath_extract.inc", _extract()), ("ring_extract.inc", _extract_ring())):
        with open(os.path.join(d, name), "w") as f:
            f.write(body)
    out = os.path.join(d, "reshape_emul")
    host = os.path.join(H.ROOT, "gpu-pruner_b200", "host")
    cmd = ["g++", "-O1", "-g", "-std=c++20", "-fsanitize=" + sanitize, "-fno-omit-frame-pointer",
           "-fno-sanitize-recover=all", "-DEMUL_PARSE_KERNEL", "-Wno-unknown-pragmas", "-I", host,
           "-I", os.path.join(H.ROOT, "tests", "cpp"), "-I", d, os.path.join(H.ROOT, "tests", "cpp", "reshape_emul.cpp")]
    cmd += [os.path.join(host, f) for f in ("ingest.cpp", "ingest_device.cpp", "json.cpp")]
    subprocess.check_call(cmd + ["-o", out, "-lpthread"])
    return out


@pytest.fixture(scope="module")
def driver(tmp_path_factory):
    return build_emul(tmp_path_factory.mktemp("emul_reshape"))


def _run(driver, root, duration_min, reshape, **env):
    e = dict(os.environ, ASAN_OPTIONS="detect_leaks=0:abort_on_error=1", **env)
    r = subprocess.run([driver] + (["--reshape"] if reshape else []) + [str(duration_min), str(root)],
                       capture_output=True, text=True, timeout=900, env=e)
    lines = r.stdout.splitlines()
    ticks = [l for l in lines if not l.startswith("MAXIMA ")]
    assert r.returncode == 0 and ticks and all(l.startswith("OK ") for l in ticks), (r.stdout[-3000:], r.stderr[-2000:])
    modes = [dict(kv.split("=", 1) for kv in l.split()[1:3]) | {"why": " ".join(l.split()[3:])} for l in ticks]
    return modes, [l for l in lines if l.startswith("MAXIMA ")]


def _both(driver, root, duration_min, **env):
    """runs the timeline with and without --reshape-ring; checks what holds for every timeline; returns the modes"""
    plain, m_plain = _run(driver, root, duration_min, False, **env)
    res, m_res = _run(driver, root, duration_min, True, **env)
    assert m_res == m_plain   # the same per-series maxima at every tick: the same verdicts
    assert len(res) == len(plain) and res[0]["mode"] == "full"
    for k, t in enumerate(res[1:], 1):
        if t["mode"] != "delta":
            assert not any(c in t["why"] for c in SHAPE_CAUSES), (k, t)
    return res, plain


def _reshaped(t):
    return t["mode"] == "delta" and t["why"].startswith("Resident window reshaped on the GPU:")


def _dropped(t):
    return int(t["why"].split(", ")[2].split()[0])


def test_late_third_slot_is_reshaped_not_rebuilt(driver, tmp_path):
    """the store of test_resident_ticks.test_series_come_and_go_and_age_out: the late duplicate needs a third slot"""
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
    TK.write_ticks(str(tmp_path), lambda k: store, times, N, step)
    res, plain = _both(driver, tmp_path, 2)
    assert [t["mode"] for t in plain] == ["full"] + ["delta"] * 4 + ["full"] + ["delta"] * 4
    assert [t["mode"] for t in res] == ["full"] + ["delta"] * 9
    assert _reshaped(res[5]) and ", 2 -> 3, " in res[5]["why"], res[5]
    assert not any(_reshaped(t) for k, t in enumerate(res) if k != 5)


def _join_store(rng, t0, horizon, step, n_base, joiners, join_at):
    store = [_series(rng, f"base-{p}", 0, t0, horizon, step, rng.choice(["idle", "busy"])) for p in range(n_base)]
    store += [_series(rng, f"new-{p}", p % 2, join_at + 1, horizon, step, "idle") for p in range(joiners)]
    return store


def test_pods_joining_past_the_head_room(driver, tmp_path):
    rng = random.Random(11)
    N, step, interval = 60, 5, 15
    t0 = 1_700_000_000
    times = [t0 + N + k * interval for k in range(5)]
    store = _join_store(rng, t0, times[-1] + 5, step, 3, 80, times[1])   # 3 pods: 67 rows; 80 join at tick 2
    TK.write_ticks(str(tmp_path), lambda k: store, times, N, step)
    res, plain = _both(driver, tmp_path, 1)
    assert plain[2]["mode"] == "full" and "more pods" in plain[2]["why"]
    assert [t["mode"] for t in res] == ["full"] + ["delta"] * 4
    assert _reshaped(res[2]) and res[2]["why"].startswith("Resident window reshaped on the GPU: 67 -> 167, 1 -> 1, 0 pods")


def _churn_store(rng, t0, horizon, step, interval, times, n_const, per_tick, extra_from=None):
    """n_const pods that stay, and per tick `per_tick` pods that report for one interval and leave (a cluster of
    constant size whose pod names never repeat); from tick extra_from on, as many more join and stay (growth)"""
    store = [_series(rng, f"stay-{p}", 0, t0, horizon, step, "busy") for p in range(n_const)]
    for k, t in enumerate(times):
        for j in range(per_tick):
            store.append(_series(rng, f"nb-{k}-{j}", 0, t - interval + 1, t + 2, step, rng.choice(["idle", "busy"])))
        if extra_from is not None and k >= extra_from:
            store += [_series(rng, f"grow-{k}-{j}", j % 3, t - interval + 1, horizon, step, "idle") for j in range(per_tick)]
    return store


def test_churn_uses_up_the_head_room_of_a_constant_cluster(driver, tmp_path):
    rng = random.Random(12)
    N, step, interval = 60, 5, 15
    t0 = 1_700_000_000
    times = [t0 + N + k * interval for k in range(12)]
    store = _churn_store(rng, t0, times[-1] + 5, step, interval, times, 10, 12)
    TK.write_ticks(str(tmp_path), lambda k: store, times, N, step)
    res, plain = _both(driver, tmp_path, 1)
    assert any(t["mode"] == "full" and "more pods" in t["why"] for t in plain[1:]), plain
    assert [t["mode"] for t in res] == ["full"] + ["delta"] * 11
    shaped = [t for t in res if _reshaped(t)]
    assert shaped and all(_dropped(t) > 0 for t in shaped), shaped


def test_churn_and_growth_in_the_same_tick(driver, tmp_path):
    rng = random.Random(13)
    N, step, interval = 60, 5, 15
    t0 = 1_700_000_000
    times = [t0 + N + k * interval for k in range(10)]
    store = _churn_store(rng, t0, times[-1] + 5, step, interval, times, 10, 14, extra_from=5)
    store.append(_series(rng, "stay-0", 3, times[6] + 1, times[-1] + 5, step, "idle", UUID="GPU-late"))   # a slot too
    TK.write_ticks(str(tmp_path), lambda k: store, times, N, step)
    res, _ = _both(driver, tmp_path, 1)
    assert [t["mode"] for t in res] == ["full"] + ["delta"] * 9
    shaped = [t for t in res if _reshaped(t)]
    assert any(_dropped(t) > 0 for t in shaped) and any(", 1 -> 2, " in t["why"] or ", 2 -> 3, " in t["why"]
                                                        for t in shaped), shaped


def test_a_dropped_pod_name_that_returns_is_a_new_pod(driver, tmp_path):
    rng = random.Random(14)
    N, step, interval = 60, 5, 15
    t0 = 1_700_000_000
    times = [t0 + N + k * interval for k in range(12)]
    horizon = times[-1] + 5
    store = [_series(rng, f"stay-{p}", 0, t0, horizon, step, "busy") for p in range(3)]
    store.append(_series(rng, "phoenix", 0, t0, times[1], step, "busy"))                 # ages out by tick 6
    store.append(("DCGM_FI_DEV_GPU_UTIL", TK.labels("phoenix", 0),
                  [(t, 0) for t in range(times[8] + 1, horizon, step)]))                   # the same series, back
    store.append(_series(rng, "phoenix", 1, times[9] + 1, horizon, step, "idle"))        # and a second one
    store += [_series(rng, f"wave-{p}", 0, times[6] + 1, times[7], step, "idle") for p in range(70)]   # forces a reshape
    TK.write_ticks(str(tmp_path), lambda k: store, times, N, step)
    res, _ = _both(driver, tmp_path, 1)
    assert [t["mode"] for t in res] == ["full"] + ["delta"] * 11
    assert _reshaped(res[7]) and _dropped(res[7]) == 1, res[7]


def test_power_on_and_off_still_takes_the_full_range(driver, tmp_path):
    rng = random.Random(15)
    N, step, interval = 60, 5, 15
    t0 = 1_700_000_000
    times = [t0 + N + k * interval for k in range(9)]
    horizon = times[-1] + 5
    store = [_series(rng, f"pod-{p}", 0, t0, horizon, step, "busy") for p in range(4)]
    store += [_series(rng, f"pod-{p}", 0, t0, horizon, step, "x", metric="DCGM_FI_DEV_POWER_USAGE") for p in range(4)]
    store += [_series(rng, f"j-{p}", 0, times[1] + 1, horizon, step, "idle") for p in range(70)]   # joins at tick 2
    store += [_series(rng, f"j-{p}", 0, times[1] + 1, horizon, step, "x", metric="DCGM_FI_DEV_POWER_USAGE")
              for p in range(70)]
    store += [_series(rng, f"k-{p}", 0, times[5] + 1, horizon, step, "idle") for p in range(120)]  # joins at tick 6
    TK.write_ticks(str(tmp_path), lambda k: store, times, N, step, with_power=True)
    for k in (3, 4):   # the power plane is off at ticks 3 and 4
        for kind in ("full", "delta"):
            os.remove(tmp_path / ("tick-%04d" % k) / kind / "power.json")
    res, _ = _both(driver, tmp_path, 1)
    assert [t["mode"] for t in res] == ["full", "delta", "delta", "full", "delta", "full", "delta", "delta", "delta"]
    assert all("power plane" in res[k]["why"] for k in (3, 5))
    assert _reshaped(res[2]) and _reshaped(res[6])


def test_fuzz_timelines(driver, tmp_path):
    """random clusters with churn, joins, late slots, PROF and power series and gaps: whatever path the session takes,
    the ring equals a fresh ingest, no tick rebuilds for a shape cause, and the maxima equal the run without reshaping"""
    n_shaped = 0
    for seed in range(12):
        rng = random.Random(2000 + seed)
        step = rng.choice([1, 2, 10])
        duration_min = rng.choice([1, 2])
        N = duration_min * 60
        interval = step * rng.randrange(2, 12)
        t0 = 1_700_000_000 + rng.randrange(1000)
        times = [t0 + N + k * interval for k in range(rng.randrange(5, 10))]
        horizon = times[-1] + 5
        store = []
        for p in range(rng.randrange(2, 7)):
            for g in range(rng.randrange(1, 4)):
                a = rng.choice([t0, t0, rng.randrange(t0, horizon)])
                b = rng.choice([horizon, horizon, rng.randrange(a, horizon + 1)])
                store.append(_series(rng, f"p{p}", g, a, b, step, rng.choice(["idle", "busy"]), jitter=rng.random() < 0.5))
                if rng.random() < 0.1:
                    store.append(_series(rng, f"p{p}", g, a, b, step, "busy", metric="DCGM_FI_PROF_GR_ENGINE_ACTIVE"))
                if rng.random() < 0.5:
                    store.append(_series(rng, f"p{p}", g, a, b, step, "x", metric="DCGM_FI_DEV_POWER_USAGE"))
        for w in range(rng.randrange(0, 3)):   # waves of short-lived pods: churn past the head-room
            at = rng.randrange(t0, horizon)
            n = rng.randrange(20, 90)
            store += [_series(rng, f"w{w}-{j}", rng.randrange(3), at, at + rng.randrange(1, 3) * interval, step, "idle")
                      for j in range(n)]
        if rng.random() < 0.5:   # a late slot
            store.append(_series(rng, "p0", 7, rng.randrange(t0, horizon), horizon, step, "idle", UUID="GPU-late"))
        d = tmp_path / f"s{seed}"
        TK.write_ticks(str(d), lambda k: store, times, N, step, with_power=True,
                       skip_delta={rng.randrange(1, len(times))} if rng.random() < 0.3 else ())
        res, _ = _both(driver, d, duration_min)
        n_shaped += sum(_reshaped(t) for t in res)
    assert n_shaped >= 6, n_shaped


def test_failed_remap_falls_back_to_the_full_range(driver, tmp_path):
    """the remap fails (GPR_E_NOMEM: the peak is the old ring plus the new one): the tick takes the full range and says
    why, it does not fail; the ring equals a fresh ingest at every tick"""
    rng = random.Random(16)
    N, step, interval = 60, 5, 15
    t0 = 1_700_000_000
    times = [t0 + N + k * interval for k in range(5)]
    store = _join_store(rng, t0, times[-1] + 5, step, 3, 80, times[1])
    TK.write_ticks(str(tmp_path), lambda k: store, times, N, step)
    res, _ = _run(driver, tmp_path, 1, True, EMUL_FAIL_REMAP="1")
    assert [t["mode"] for t in res] == ["full", "delta", "full", "delta", "delta"]
    assert "could not be reshaped" in res[2]["why"] and "out of device memory" in res[2]["why"]


# ---- CLI ---------------------------------------------------------------------------------------------------------------
def test_cli_reshape_ring_needs_daemon_mode():
    r = H.parse_cli(["--prometheus-url", "file:///x", "--reshape-ring"])
    assert not r["ok"] and r["exit_code"] == 2 and "--reshape-ring" in r["message"]
    assert H.parse_cli(["--prometheus-url", "file:///x", "-d", "--reshape-ring"])["ok"]
    r = H.parse_cli(["--prometheus-url", "file:///x", "-d", "--reshape-ring=yes"])
    assert not r["ok"] and r["exit_code"] == 2
    assert "--reshape-ring" in H.parse_cli(["--help"])["message"]


def test_cli_reshape_ring_leaves_the_query_alone():
    base = ["--prometheus-url", "file:///x", "-d", "-t", "5", "--power-threshold", "150"]
    assert H.render_selectors(base + ["--reshape-ring"]) == H.render_selectors(base)


def test_binary_reshape_ring_without_daemon_mode_exits_2():
    if not os.path.exists(H.BIN):
        pytest.skip("gpu-pruner binary not built")
    p = subprocess.run([H.BIN, "--prometheus-url", "file:///x", "--reshape-ring"], capture_output=True, text=True)
    assert p.returncode == 2 and "--reshape-ring" in p.stderr
    p = subprocess.run([H.BIN, "--help"], capture_output=True, text=True)
    assert p.returncode == 0 and "--reshape-ring" in p.stdout
