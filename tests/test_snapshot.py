"""CPU: daemon mode across a restart (--snapshot-file, DESIGN.md §8i).  A session that ran ticks 0..k-1 writes a
snapshot; a fresh emulated device and session restored from it run ticks k.. (tests/cpp/snapshot_emul.cpp --save /
--resume, the export and chunk kernels' source under the CPU shim, ASan/UBSan).  After a restore every tick must take
the uninterrupted session's path, hold its ring bit for bit and its session (every series on the same (pod, slot,
result)), and hold the window of a fresh full-range ingest.  A snapshot that is refused leaves the session cold: the
next tick takes the full range, and every later ring again equals a fresh ingest.  The GPU run of the same through the
`gpu-pruner` binary is tests/test_gpu_daemon_snapshot.py."""
import ctypes as C
import json
import os
import random
import struct
import subprocess

import pytest

import hostlib as H
import snapshot_ref as SR
import ticks as TK
from test_resident_ticks import _series


# ---- CRC32C ----------------------------------------------------------------------------------------------------------
def _crc(data, crc=0, portable=False):
    lib = H.lib()
    lib.gph_crc32c.restype = C.c_uint
    lib.gph_crc32c.argtypes = [C.c_void_p, C.c_ulonglong, C.c_uint, C.c_int]
    buf = C.create_string_buffer(bytes(data), len(data) + 1)
    return lib.gph_crc32c(buf, len(data), crc, int(portable))


def _crc_at(data, offset, portable):
    """CRC of `data` starting `offset` bytes past an 8-byte boundary"""
    lib = H.lib()
    buf = C.create_string_buffer(len(data) + 16)
    base = (C.addressof(buf) + 7) // 8 * 8 + offset
    C.memmove(base, bytes(data), len(data))
    return lib.gph_crc32c(C.c_void_p(base), len(data), 0, int(portable))


@pytest.mark.parametrize("portable", [False, True], ids=["dispatch", "slice8"])
def test_crc32c_known_answers(portable):
    assert _crc(b"123456789", portable=portable) == 0xE3069283
    # RFC 3720 §B.4
    assert _crc(bytes(32), portable=portable) == 0x8A9136AA
    assert _crc(b"\xff" * 32, portable=portable) == 0x62A8AB43
    assert _crc(bytes(range(32)), portable=portable) == 0x46DD794E
    assert _crc(bytes(range(31, -1, -1)), portable=portable) == 0x113FDB5C
    iscsi = bytes.fromhex("01c00000000000000000000000000000" "14000000000004000000001400000018"
                          "28000000000000000200000000000000")   # the read command PDU
    assert len(iscsi) == 48
    assert _crc(iscsi, portable=portable) == 0xD9963A56


@pytest.mark.parametrize("portable", [False, True], ids=["dispatch", "slice8"])
def test_crc32c_every_length_and_alignment(portable):
    rng = random.Random(3)
    data = bytes(rng.randrange(256) for _ in range(80))
    for n in range(65):
        for off in range(8):
            assert _crc_at(data[:n], off, portable) == SR.crc32c(data[:n]), (n, off)
    # piecewise: the CRC of a file checked part by part
    assert _crc(data[40:], _crc(data[:40], portable=portable), portable=portable) == SR.crc32c(data)


# ---- CLI ---------------------------------------------------------------------------------------------------------------
def test_cli_snapshot_file_needs_daemon_mode():
    r = H.parse_cli(["--prometheus-url", "file:///x", "--snapshot-file", "/tmp/s"])
    assert not r["ok"] and r["exit_code"] == 2 and "--snapshot-file" in r["message"]
    assert H.parse_cli(["--prometheus-url", "file:///x", "-d", "--snapshot-file", "/tmp/s"])["ok"]
    assert "--snapshot-file <PATH>" in H.parse_cli(["--help"])["message"]


def test_binary_snapshot_file_without_daemon_mode_exits_2():
    if not os.path.exists(H.BIN):
        pytest.skip("gpu-pruner binary not built")
    p = subprocess.run([H.BIN, "--prometheus-url", "file:///x", "--snapshot-file", "/tmp/s"], capture_output=True, text=True)
    assert p.returncode == 2 and "--snapshot-file" in p.stderr
    p = subprocess.run([H.BIN, "--help"], capture_output=True, text=True)
    assert p.returncode == 0 and "--snapshot-file" in p.stdout


# ---- resume equals uninterrupted ------------------------------------------------------------------------------------
def build_emul(out_dir, sanitize="address,undefined"):
    """tests/cpp/snapshot_emul.cpp: text_emul.cpp's kernel flavour plus the export, chunk check and chunk scatter kernels'
    source, cut out as their own tests cut them"""
    import emul_build
    from test_chunks_emul import _extract_chunks
    from test_chunks_export_emul import _extract as extract_export
    from test_samples_emul import _extract_samples
    d = str(out_dir)
    for name, body in (("text_kernel_extract.inc", emul_build.extract_parse_kernel()),
                       ("samples_extract.inc", _extract_samples()), ("chunks_extract.inc", _extract_chunks()),
                       ("chunks_export_extract.inc", extract_export())):
        with open(os.path.join(d, name), "w") as f:
            f.write(body)
    out = os.path.join(d, "snapshot_emul")
    host = os.path.join(H.ROOT, "gpu-pruner_b200", "host")
    cmd = ["g++", "-O1", "-g", "-std=c++20", "-fsanitize=" + sanitize, "-fno-omit-frame-pointer", "-fno-sanitize-recover=all",
           "-DEMUL_PARSE_KERNEL", "-Wno-unknown-pragmas", "-I", host, "-I", os.path.join(H.ROOT, "tests", "cpp"), "-I", d,
           os.path.join(H.ROOT, "tests", "cpp", "snapshot_emul.cpp")]
    cmd += [os.path.join(host, f) for f in ("ingest.cpp", "ingest_device.cpp", "snapshot.cpp", "json.cpp")]
    subprocess.check_call(cmd + ["-o", out, "-lpthread"])
    return out


@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    return build_emul(tmp_path_factory.mktemp("emul_snapshot"))


def _key(path, dur, *cli, thr=0.0, span=None):
    sel = H.render_selectors(["--prometheus-url", "file:///x", "-t", str(dur), *cli])
    with open(path, "w") as f:
        json.dump({"span": span if span is not None else dur * 60, "power_threshold": thr,
                   "selectors": [sel["util"], sel["prof"], sel["power"]]}, f)
    return str(path)


def _drive(emul, mode, dur, root, k, snap, key):
    env = dict(os.environ, ASAN_OPTIONS="detect_leaks=0:abort_on_error=1")
    r = subprocess.run([emul, mode, str(dur), str(root), str(k), str(snap), str(key)], capture_output=True, text=True,
                       timeout=900, env=env)
    assert r.returncode == 0 and "MISMATCH" not in r.stdout, (r.stdout[-3000:], r.stderr[-3000:])
    return r.stdout.splitlines()


def _ticks(lines):
    return [dict(kv.split("=", 1) for kv in l.split()[1:4]) for l in lines if l.startswith("OK tick=")]


def _resume_everywhere(emul, tmp_path, root, n, dur, cuts=None):
    key = _key(tmp_path / "key.json", dur, "--power-threshold", "150")
    for k in cuts or range(1, n):
        snap = tmp_path / ("snap-%d" % k)
        save = _drive(emul, "--save", dur, root, k, snap, key)
        assert save[-1].startswith("SAVED"), save
        snap_doc = SR.read(open(snap, "rb").read())
        lines = _drive(emul, "--resume", dur, root, k, snap, key)
        assert lines[0] == "RESTORE ok", lines
        ticks = _ticks(lines)
        assert [int(t["tick"]) for t in ticks] == list(range(k, n)), lines
        # the first tick after a restore appends its slice, unless the scenario forces the full range there
        assert all(t["mode"] == t["umode"] for t in ticks), lines
        assert snap_doc["t_end"] > 0


def _come_and_go(root):
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
    TK.write_ticks(str(root), lambda k: store, times, N, step)
    return len(times), 2


def _gap_prof_power(root):
    rng = random.Random(9)
    N, step, interval = 60, 1, 15
    t0 = 1_700_000_000
    times = [t0 + N + k * interval for k in range(8)]
    horizon = times[-1] + 5
    util = [_series(rng, f"pod-{p}", 0, t0, horizon, step, "idle") for p in range(3)]
    prof_same = ("DCGM_FI_PROF_GR_ENGINE_ACTIVE", util[0][1], [(t, 0.25 if t % 7 == 0 else 0.0) for t in range(t0, horizon)])
    prof_late = ("DCGM_FI_PROF_GR_ENGINE_ACTIVE", util[1][1], [(t, 0.5) for t in range(times[4] + 2, horizon)])
    power = [_series(rng, f"pod-{p}", 0, t0, horizon, step, "x", metric="DCGM_FI_DEV_POWER_USAGE") for p in range(3)]
    store = util + [prof_same, prof_late] + power
    TK.write_ticks(str(root), lambda k: store, times, N, step, with_power=True, skip_delta={2})
    return len(times), 1


def test_resume_come_and_go_series(emul, tmp_path):
    n, dur = _come_and_go(tmp_path / "ticks")
    _resume_everywhere(emul, tmp_path, tmp_path / "ticks", n, dur)


def test_resume_gap_ticks_prof_changes_and_power(emul, tmp_path):
    n, dur = _gap_prof_power(tmp_path / "ticks")
    _resume_everywhere(emul, tmp_path, tmp_path / "ticks", n, dur)


def test_resume_fuzz_timelines(emul, tmp_path):
    """the random clusters of test_resident_ticks.test_fuzz_timelines, cut at every tick"""
    for seed in range(0, 12, 2):
        rng = random.Random(1000 + seed)
        step = rng.choice([1, 2, 10])
        duration_min = rng.choice([1, 2])
        N = duration_min * 60
        interval = step * rng.randrange(2, 12)
        t0 = 1_700_000_000 + rng.randrange(1000)
        times = [t0 + N + k * interval for k in range(rng.randrange(4, 9))]
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
        d = tmp_path / f"s{seed}"
        TK.write_ticks(str(d / "ticks"), lambda k: store, times, N, step, with_power=True,
                       skip_delta={rng.randrange(1, len(times))} if rng.random() < 0.3 else ())
        d.mkdir(exist_ok=True)
        _resume_everywhere(emul, d, d / "ticks", len(times), duration_min)


# ---- refusals ---------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def saved(emul, tmp_path_factory):
    """the PROF / power / gap timeline, cut after tick 3: (root, n, dur, key, snapshot bytes, parsed)"""
    d = tmp_path_factory.mktemp("refusals")
    n, dur = _gap_prof_power(d / "ticks")
    key = _key(d / "key.json", dur, "--power-threshold", "150")
    snap = d / "snap"
    assert _drive(emul, "--save", dur, d / "ticks", 3, snap, key)[-1].startswith("SAVED")
    blob = open(snap, "rb").read()
    return d, n, dur, key, blob, SR.read(blob)


def _refused(emul, saved, tmp_path, blob, key=None, reason=None):
    d, n, dur, k0, _, _ = saved
    snap = tmp_path / "snap"
    snap.write_bytes(blob)
    lines = _drive(emul, "--resume", dur, d / "ticks", 3, snap, key or k0)
    assert lines[0].startswith("RESTORE refused"), lines[0]
    if reason:
        assert reason in lines[0], lines[0]
    ticks = _ticks(lines)
    assert [int(t["tick"]) for t in ticks] == list(range(3, n)) and ticks[0]["mode"] == "full", lines
    return lines[0]


def test_snapshot_layout_matches_the_design(saved):
    _, _, dur, _, blob, doc = saved
    assert [s[0] for s in doc["sections"]] == ["header", "fingerprint", "t_end", "session", "plane0", "plane1", "trailer"]
    assert doc["power"] and doc["span"] == dur * 60 and doc["step"] == 1 and doc["T"] == 60 and doc["G"] >= 1
    assert doc["pods_cap"] >= len(doc["pods"]) == 3
    assert doc["prof_rows"] and doc["prof_sigs"] and all(len(k) == 1 for k in doc["power_keys"])
    assert {k[2] for k in doc["known"]} >= {2, 1}   # placed and shadowed series are both remembered
    for p in doc["planes"]:
        assert p["series_chunks"][0] == 0 and p["chunk_bytes"][-1] == len(p["data"]) and len(p["rows"]) > 0


def test_truncated_snapshots_are_refused(emul, saved, tmp_path):
    blob, doc = saved[4], saved[5]
    cuts = sorted({b for _, b, _ in doc["sections"]} | {e for _, _, e in doc["sections"]} - {len(blob)})
    rng = random.Random(11)
    cuts += sorted(rng.randrange(len(blob)) for _ in range(20))
    for c in cuts:
        _refused(emul, saved, tmp_path, blob[:c])


def test_flipped_bytes_are_refused(emul, saved, tmp_path):
    blob, doc = saved[4], saved[5]
    for name, b, e in doc["sections"]:
        at = (b + e) // 2
        bad = bytearray(blob)
        bad[at] ^= 0x40
        why = _refused(emul, saved, tmp_path, bytes(bad))
        assert name in ("header", "trailer") or "checksum" in why, (name, why)


def test_wrong_magic_and_unknown_version(emul, saved, tmp_path):
    blob = saved[4]
    _refused(emul, saved, tmp_path, b"GPRSNAQ\0" + blob[8:], reason="magic")
    _refused(emul, saved, tmp_path, blob[:8] + struct.pack("<I", 2) + blob[12:], reason="version")


@pytest.mark.parametrize("cli,thr,span,why", [
    ((), 0.0, 180, "window"),                                   # --duration 3 instead of 1
    (("--power-threshold", "150"), 150.0, None, "power threshold"),
    ((), 0.0, None, "power selector"),                          # no power plane
    (("--power-threshold", "150", "-n", "team-a"), 0.0, None, "selector"),
    (("--power-threshold", "150", "-m", "NVIDIA H100"), 0.0, None, "selector"),
    (("--power-threshold", "150", "--honor-labels"), 0.0, None, "selector"),
], ids=["duration", "power-threshold", "power-plane-off", "namespace", "model-name", "honor-labels"])
def test_fingerprint_changes_are_refused(emul, saved, tmp_path, cli, thr, span, why):
    key = _key(tmp_path / "key.json", saved[2], *cli, thr=thr, span=span)
    _refused(emul, saved, tmp_path, saved[4], key=key, reason=why)


def test_step_change_rebuilds_on_the_first_tick(emul, tmp_path):
    """the step is the query's, not the CLI's: a snapshot taken at another step is restored, and the first slice, whose
    step differs, is refused by the existing delta check — the full range is fetched"""
    rng = random.Random(4)
    t0 = 1_700_000_000
    times = [t0 + 120 + k * 30 for k in range(5)]
    store = [_series(rng, f"pod-{p}", 0, t0, times[-1] + 5, 2, "busy") for p in range(3)]
    TK.write_ticks(str(tmp_path / "a"), lambda k: store, times, 120, 2)
    TK.write_ticks(str(tmp_path / "b"), lambda k: store, times, 120, 1)
    key = _key(tmp_path / "key.json", 2)
    assert _drive(emul, "--save", 2, tmp_path / "a", 2, tmp_path / "snap", key)[-1].startswith("SAVED")
    env = dict(os.environ, ASAN_OPTIONS="detect_leaks=0:abort_on_error=1")
    r = subprocess.run([emul, "--resume", "2", str(tmp_path / "b"), "2", str(tmp_path / "snap"), key],
                       capture_output=True, text=True, timeout=600, env=env)
    lines = r.stdout.splitlines()
    assert lines[0] == "RESTORE ok"
    # U, uninterrupted on the new step, appends; B's snapshot is at the old step, so B takes the full range.  (The
    # driver reports the differing path only once B's ring has been found equal to a fresh ingest of the tick.)
    assert lines[1] == "MISMATCH tick=2 B took the full path, U the delta path", lines
    assert all(l.startswith("OK tick=") for l in lines[2:]) and len(lines) == 4, lines


def test_chunk_refused_by_the_scatter(emul, saved, tmp_path):
    """a chunk that passes the CRC (rewritten after the corruption) but that gpr_chunks_scatter refuses"""
    blob, doc = saved[4], saved[5]
    p = doc["planes"][0]
    bad = bytearray(blob)
    at = p["data_at"] + int(p["chunk_bytes"][0])
    bad[at:at + 2] = b"\xff\xff"   # 65,535 samples in a short chunk: the decode would read past it
    _refused(emul, saved, tmp_path, SR.reseal(bad), reason="ring not restored")


def test_stale_tmp_file_is_ignored(emul, saved, tmp_path):
    d, n, dur, key, blob, _ = saved
    snap = tmp_path / "snap"
    snap.write_bytes(blob)
    (tmp_path / "snap.tmp").write_bytes(blob[:100])
    lines = _drive(emul, "--resume", dur, d / "ticks", 3, snap, key)
    assert lines[0] == "RESTORE ok", lines
    # a save overwrites a stale PATH.tmp and replaces PATH whole
    assert _drive(emul, "--save", dur, d / "ticks", 4, snap, key)[-1].startswith("SAVED")
    assert not os.path.exists(str(snap) + ".tmp") and SR.read(open(snap, "rb").read())["t_end"] > doc_t_end(blob)


def doc_t_end(blob):
    return SR.read(blob)["t_end"]
