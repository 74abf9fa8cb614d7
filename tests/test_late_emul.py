"""CPU: `gpu-pruner -d --late-seconds L` (DESIGN.md §8e) on the EMULATED device (tests/cpp/late_emul.cpp: text_emul.cpp's
device with the sources of k_ring_cols, k_remap_rows and k_live_rows, ASan/UBSan), through the binary's FileSource, on a server whose
samples arrive late (tests/late_ticks.py).  At every tick the ring holds exactly what a fresh ingest of the samples
the ticks asked for yields — a fresh full-range ingest when no sample is more than L late, and without exactly the
samples that came later than that otherwise — and the late-cell counts of both planes equal the model's.
  * lags from 0 to beyond L; L a multiple of the step and not; with --query-slice, with --reshape-ring, with the power
    plane, across a restart from a saved session;
  * a hard sample (more than 19 significant digits, declined by the device parser) in the re-asked buckets of a row
    with an older sample in the partly re-asked bucket: the CPU re-parse is merged with what the ring held, not
    written over it;
  * L = 0: no band is read and nothing is counted;
  * 12 fuzzed timelines.
The GPU runs are tests/test_gpu_late_samples.py and tests/test_gpu_late_ticks.py."""
import os
import random
import subprocess

import pytest

import hostlib as H
import late_ticks as LT
import ticks as TK

T0 = 1_700_000_000
POWER_VALUES = (55, 60, 149.5, 310.25)


def build_emul(out_dir, sanitize="address,undefined"):
    import emul_build
    from test_hotpath_emul import _extract
    from test_ring_emul import _extract_ring
    d = str(out_dir)
    for name, body in (("text_kernel_extract.inc", emul_build.extract_parse_kernel()),
                       ("hotpath_extract.inc", _extract()), ("ring_extract.inc", _extract_ring())):
        with open(os.path.join(d, name), "w") as f:
            f.write(body)
    out = os.path.join(d, "late_emul")
    host = os.path.join(H.ROOT, "gpu-pruner_b200", "host")
    cmd = ["g++", "-O1", "-g", "-std=c++20", "-fsanitize=" + sanitize, "-fno-omit-frame-pointer",
           "-fno-sanitize-recover=all", "-DEMUL_PARSE_KERNEL", "-Wno-unknown-pragmas", "-I", host,
           "-I", os.path.join(H.ROOT, "tests", "cpp"), "-I", d, os.path.join(H.ROOT, "tests", "cpp", "late_emul.cpp")]
    cmd += [os.path.join(host, f) for f in ("ingest.cpp", "ingest_device.cpp", "json.cpp", "controller.cpp", "cli.cpp",
                                            "kube.cpp", "promql.cpp", "snapshot.cpp")]
    subprocess.check_call(cmd + ["-o", out, "-lpthread"])
    return out


@pytest.fixture(scope="module")
def driver(tmp_path_factory):
    return build_emul(tmp_path_factory.mktemp("emul_late"))


def _run(driver, root, L, S, duration_min, thr=0, reshape=False, **env):
    e = dict(os.environ, ASAN_OPTIONS="detect_leaks=0:abort_on_error=1", **env)
    r = subprocess.run([driver] + (["--reshape"] if reshape else []) + [str(L), str(S), str(duration_min), str(thr),
                                                                          str(root)],
                       capture_output=True, text=True, timeout=900, env=e)
    lines = r.stdout.splitlines()
    ticks = [l for l in lines if l.startswith(("OK ", "MISMATCH "))]
    assert r.returncode == 0 and ticks and all(l.startswith("OK ") for l in ticks), (r.stdout[-3000:], r.stderr[-2000:])
    modes = [dict(kv.split("=", 1) for kv in l.split()[1:4]) for l in ticks]
    total = dict(kv.split("=") for kv in [l for l in lines if l.startswith("TOTAL ")][0].split()[1:])
    return modes, {k: int(v) for k, v in total.items()}, r.stderr


def _hard(rng, v):
    """v written with more than 19 significant digits: the device parser declines the span, the CPU re-parses it"""
    return "%d.%s" % (v, "".join(rng.choice("0123456789") for _ in range(22)))


def _store(rng, step, horizon, lag, n_pods=5, power=False, hard_pod=None, slot_at=None):
    """lag(rng) -> seconds a sample takes to reach the server.  Samples every step / 2 (at least 1 s), values 0, 20, 55
    or 100; hard_pod writes some of its values with more than 19 digits; slot_at: pod-0 gains GPUs 7 and 8 then, one slot more than any pod had"""
    series = []
    every = max(1, step // 2)
    for p in range(n_pods):
        for g in range(1 + p % 2):
            smp, t = [], T0 + rng.randrange(every)
            while t <= horizon:
                v = rng.choice([0, 0, 20, 55, 100])
                if p == hard_pod and rng.random() < 0.4:
                    v = _hard(rng, v)
                smp.append((t, v, lag(rng)))
                t += every
            series.append(("DCGM_FI_DEV_GPU_UTIL", TK.labels(f"pod-{p}", g), smp))
        if power:
            smp, t = [], T0 + rng.randrange(every)
            while t <= horizon:
                smp.append((t, rng.choice(POWER_VALUES), lag(rng)))
                t += every
            series.append(("DCGM_FI_DEV_POWER_USAGE", TK.labels(f"pod-{p}", 0), smp))
    for g in ((7, 8) if slot_at is not None else ()):
        series.append(("DCGM_FI_DEV_GPU_UTIL", TK.labels("pod-0", g),
                       [(t, 20, lag(rng)) for t in range(slot_at, horizon + 1, every)]))
    return LT.LateStore(series)


def _lags(lo, hi, p_late=0.3):
    return lambda rng: rng.uniform(lo, hi) if rng.random() < p_late else rng.uniform(0, 2)


def _timeline(driver, tmp_path, *, seed, step, interval, duration_min, L, lag, S=0, power=False, reshape=False,
              hard_pod=None, slot_at=None, n_ticks=6, **env):
    rng = random.Random(seed)
    N = duration_min * 60
    times = [T0 + N + k * interval for k in range(n_ticks)]
    late = _store(rng, step, times[-1], lag, power=power, hard_pod=hard_pod,
                  slot_at=None if slot_at is None else times[slot_at] - interval // 2)
    root = tmp_path / f"s{seed}-L{L}-S{S}"
    LT.write_late_ticks(str(root), late, times, N, step, L, S=S, power=power)
    modes, total, err = _run(driver, root, L, S, duration_min, thr=150 if power else 0, reshape=reshape, **env)
    assert [m["mode"] for m in modes] == ["full"] + ["delta"] * (n_ticks - 1), (modes, err[-2000:])
    got = [tuple(int(x) for x in m["late"].split(",")) for m in modes[1:]]
    assert got == LT.late_cells_planes(late, times, N, step, L)
    assert all(m["late"] == "0,0" for m in modes[:1])
    return got, total, err


@pytest.mark.parametrize("step,interval,L", [(10, 30, 20), (10, 30, 25), (5, 20, 12), (1, 15, 7)])
def test_lags_up_to_L_equal_fresh_ingests(driver, tmp_path, step, interval, L):
    """no sample more than L late: expect/ is the full range, and late samples are counted"""
    got, total, _ = _timeline(driver, tmp_path, seed=step * 100 + L, step=step, interval=interval, duration_min=2, L=L,
                              lag=_lags(interval / 2, L))
    assert sum(u for u, _ in got) > 0 and total["band_reads"] == 2 * (len(got))


@pytest.mark.parametrize("L", [10, 25])
def test_lags_beyond_L_lose_exactly_the_late_samples(driver, tmp_path, L):
    _timeline(driver, tmp_path, seed=7 + L, step=10, interval=30, duration_min=2, L=L, lag=_lags(0, 3 * L, 0.5))


def test_no_reask_reads_no_band(driver, tmp_path):
    got, total, err = _timeline(driver, tmp_path, seed=3, step=10, interval=30, duration_min=2, L=0,
                                lag=_lags(5, 40, 0.5), power=True)
    assert got == [(0, 0)] * len(got) and total["band_reads"] == 0 and "Late samples" not in err


@pytest.mark.parametrize("S,L", [(20, 30), (30, 25), (40, 45)])
def test_query_slices(driver, tmp_path, S, L):
    """the delta range, re-ask included, asked as slices; L a multiple of the step and not"""
    got, _, _ = _timeline(driver, tmp_path, seed=S + L, step=10, interval=30, duration_min=2, L=L, S=S,
                          lag=_lags(5, L + 10, 0.4), power=True)
    assert sum(u + w for u, w in got) > 0


def test_power_plane(driver, tmp_path):
    got, _, _ = _timeline(driver, tmp_path, seed=91, step=5, interval=20, duration_min=2, L=15, power=True,
                          lag=_lags(5, 15, 0.5))
    assert sum(w for _, w in got) > 0 and sum(u for u, _ in got) > 0


def test_reshape_ring_with_a_new_slot(driver, tmp_path):
    """pod-0 gains two GPUs in the middle of the timeline: --reshape-ring reshapes the ring (the band is read after the
    remap, so its rows are the new ones)"""
    _, _, err = _timeline(driver, tmp_path, seed=33, step=10, interval=30, duration_min=2, L=25, reshape=True,
                          lag=_lags(5, 25), power=True, slot_at=3)
    assert "Resident window reshaped on the GPU" in err


def test_hard_sample_in_the_partly_reasked_bucket(driver, tmp_path):
    """L = 25 with step 10: the oldest re-asked bucket is half re-asked, so a hard row's re-parse lacks the samples in
    its older half; they stay because the re-parse is merged with the band, not written over it"""
    for seed in range(4):
        _timeline(driver, tmp_path, seed=200 + seed, step=10, interval=30, duration_min=2, L=25, hard_pod=0,
                  lag=_lags(5, 25))


def test_restart_from_a_saved_session(driver, tmp_path):
    _timeline(driver, tmp_path, seed=57, step=10, interval=30, duration_min=2, L=25, power=True, lag=_lags(5, 25),
              EMUL_RESTORE_BEFORE="3")


def test_fuzz_timelines(driver, tmp_path):
    for seed in range(12):
        rng = random.Random(5000 + seed)
        step = rng.choice([1, 2, 5, 10])
        interval = step * rng.randrange(2, 6)
        duration_min = rng.choice([1, 2])
        L = rng.choice([0, step, step * rng.randrange(1, 4), step * rng.randrange(1, 4) + rng.randrange(1, step + 1)])
        L = min(L, duration_min * 60 - interval - step)
        S = rng.choice([0, 0, step * rng.randrange(2, 8)])
        lag_hi = rng.choice([L, 2 * L + 5, interval])
        _timeline(driver, tmp_path, seed=6000 + seed, step=step, interval=interval, duration_min=duration_min, L=L,
                  S=S, power=rng.random() < 0.5, reshape=rng.random() < 0.5, hard_pod=rng.choice([None, 1]),
                  lag=_lags(0, max(1, lag_hi), rng.random()))
