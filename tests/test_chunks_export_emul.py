"""gpr_resident_export on the CPU: k_export_size, k_export_scan and k_export_write of
gpu-pruner_b200/csrc/gpr_chunks_encode.cuh, compiled from their source under tests/cpp/cuda_shim.hpp
(tests/cpp/chunks_export_emul.cpp), under AddressSanitizer + UndefinedBehaviorSanitizer and ThreadSanitizer:
  * every array byte for byte equal to tests/chunks_ref.py's encoder on the same (ts_ms, value) lists, for rings of
    T in {1, 2, 63, 64, 65, 120, 121, 1800} at several heads (T - 1 among them) and max_per_chunk in
    {1, 2, 119, 120, 65535};
  * rows empty, full, sparse, and of special values: +-0.0, denormals, +-Inf, large and negative values, 17-digit
    ratios, power cells snapped by the power rule, NaNs other than the fill (skipped like it);
  * the reference decoder gives the unrolled ring back from the export;
  * the size protocol: a capacity one short of the need writes nothing and reports the true counts;
  * the ring unchanged."""
import os
import subprocess

import numpy as np
import pytest

import chunks_ref as R
import export_ref as X

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
T_END, STEP = 1_700_000_123, 10


def _extract():
    src = open(os.path.join(ROOT, "gpu-pruner_b200", "csrc", "gpr_chunks_encode.cuh")).read()
    body = src[src.index("namespace chunks {") + len("namespace chunks {"):src.index("}  // namespace chunks")]
    old = "extern __shared__ __align__(16) unsigned char smem[];"
    assert body.count(old) == 1
    body = body.replace(old, "unsigned char* smem = tl_cta->smem;")
    assert "asm" not in body and "__shared__" not in body
    for name in ("k_export_size", "k_export_scan", "k_export_write", "encode_chunk", "for_each_chunk"):
        assert name in body, name
    return body


def _build(d, sanitize):
    (d / "chunks_export_extract.inc").write_text(_extract())
    exe = d / ("chunks_export_emul_" + sanitize.replace(",", "_"))
    cmd = ["g++", "-std=c++20", "-O1", "-g", "-pthread", "-Wno-unknown-pragmas", "-fsanitize=" + sanitize,
           "-fno-omit-frame-pointer"]
    if sanitize != "thread":
        cmd.append("-fno-sanitize-recover=all")
    subprocess.run(cmd + ["-I", str(d), "-I", os.path.join(ROOT, "tests", "cpp"),
                          os.path.join(ROOT, "tests", "cpp", "chunks_export_emul.cpp"), "-o", str(exe)],
                   check=True, capture_output=True, text=True)
    return str(exe)


@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    return _build(tmp_path_factory.mktemp("export"), "address,undefined")


BIG = 1 << 62


def run(exe, d, plane, head, M, caps=(BIG, BIG, BIG), sm=1, env=None):
    d.mkdir(parents=True, exist_ok=True)
    rows, T = plane.shape
    (d / "params.txt").write_text(" ".join(str(x) for x in (rows, T, head, M, T_END * 1000, STEP * 1000, *caps)) + "\n")
    np.ascontiguousarray(plane, np.uint32).tofile(d / "plane.u32")
    r = subprocess.run([exe, str(sm), str(d)], capture_output=True, text=True, timeout=1800, env=env)
    assert r.returncode == 0, r.stderr[-3000:]
    raw = np.fromfile(d / "out.bin", np.uint8)
    status, ns, nc, nb, n_samples = (int(x) for x in raw[:40].view(np.uint64))
    if status:
        assert raw.size == 40
        return status, (ns, nc, nb, n_samples), None
    o = 40
    sc = raw[o:o + 8 * (ns + 1)].view(np.uint64); o += 8 * (ns + 1)
    cb = raw[o:o + 8 * (nc + 1)].view(np.uint64); o += 8 * (nc + 1)
    rows_out = raw[o:o + 4 * ns].view(np.uint32); o += 4 * ns
    data = raw[o:o + nb]; o += nb
    assert o == raw.size
    return status, (ns, nc, nb, n_samples), (sc, rows_out, cb, data)


def check(exe, d, plane, head, M, **kw):
    status, counts, got = run(exe, d, plane, head, M, **kw)
    sc, rows, cb, data, n_samples = X.export(plane, head, T_END, STEP, M)
    assert status == 0
    assert counts == (len(rows), len(cb) - 1, len(data), n_samples)
    for name, g, w in (("series_chunks", got[0], sc), ("rows", got[1], rows), ("chunk_bytes", got[2], cb)):
        assert np.array_equal(g, w), name
    if not np.array_equal(got[3], data):
        k = int(np.argmax(got[3] != data))
        c = int(np.searchsorted(cb, k, side="right")) - 1
        raise AssertionError(f"data byte {k} (chunk {c}): {got[3][k]:#04x} != {data[k]:#04x}")
    back = X.restore(*got, plane.shape[0], plane.shape[1], T_END, STEP)
    assert np.array_equal(back, X.canonical(X.unroll(plane, head)))
    return counts


def f32bits(x):
    return np.asarray(x, np.float32).view(np.uint32)


SPECIAL = f32bits([0.0, -0.0, 1e-45, -1e-45, 1.17e-38, 3.4e38, -3.4e38, np.inf, -np.inf, 100.0, -7.5, 1e30, -1e-30,
                   0.333333343267, 0.1, 149.99998, 150.0, 150.00002, 1.0])
POWER_SNAPPED = f32bits([np.nextafter(np.float32(150), np.float32(0)), np.float32(150),
                         np.nextafter(np.float32(150), np.float32(1e9))])
OTHER_NANS = np.array([0x7FC00000, 0xFFC00000, 0x7F800001, 0x7FF00002], np.uint32)


def ring(rng, rows, T):
    """rows of every kind: empty, full, sparse util, special values, 17-digit ratios, snapped power, odd NaNs"""
    plane = np.full((rows, T), X.FILL, np.uint32)
    for r in range(rows):
        kind = r % 7
        if kind == 0:
            continue
        if kind == 1:
            plane[r] = f32bits(rng.integers(0, 101, T))
        elif kind == 2:
            keep = rng.random(T) < 0.3
            plane[r, keep] = f32bits(rng.integers(0, 101, int(keep.sum())))
        elif kind == 3:
            plane[r] = rng.choice(SPECIAL, T)
        elif kind == 4:
            plane[r] = f32bits(rng.random(T))   # DCGM_FI_PROF_GR_ENGINE_ACTIVE ratios: 17-digit decimals
        elif kind == 5:
            plane[r] = rng.choice(POWER_SNAPPED, T)
            plane[r, rng.random(T) < 0.2] = X.FILL
        else:
            plane[r] = f32bits(rng.uniform(-1e6, 1e6, T))
            plane[r, rng.random(T) < 0.25] = rng.choice(OTHER_NANS)
    return plane


@pytest.mark.parametrize("T", [1, 2, 63, 64, 65, 120, 121, 1800])
def test_byte_equal_to_the_reference_encoder(emul, tmp_path, T):
    rng = np.random.default_rng(T)
    plane = ring(rng, 9, T)
    heads = sorted({0, 1 % T, T // 2, T - 1})
    Ms = (1, 2, 119, 120, 65535) if T <= 121 else (1, 119, 120, 65535)
    k = 0
    for head in heads:
        for M in Ms:
            if T == 1800 and M == 1 and head not in (0, T - 1):
                continue
            k += 1
            check(emul, tmp_path / f"r{k}", plane, head, M)


def test_every_row_shape_at_every_chunk_boundary(emul, tmp_path):
    """rows of 1 .. 2 * 32 * 3 + 1 present cells with per_chunk 3: every count of chunks in a round of 32 lanes and
    the round boundaries, the present cells spread so chunk starts fall at every lane of a window"""
    rng = np.random.default_rng(5)
    T = 200
    rows = 40
    plane = np.full((rows, T), X.FILL, np.uint32)
    for r in range(rows):
        n = min(T, 1 + 5 * r)
        cols = np.sort(rng.choice(T, n, replace=False))
        plane[r, cols] = f32bits(rng.integers(0, 50, n))
    for head in (0, 77, T - 1):
        check(emul, tmp_path / f"h{head}", plane, head, 3)
        check(emul, tmp_path / f"h{head}m1", plane, head, 1)


def test_empty_ring(emul, tmp_path):
    plane = np.full((5, 64), X.FILL, np.uint32)
    assert check(emul, tmp_path / "e", plane, 10, 120) == (0, 0, 0, 0)


def test_capacity_protocol(emul, tmp_path):
    """a capacity one short of the need: status 1, the true counts, nothing written; exactly the need: written"""
    rng = np.random.default_rng(7)
    plane = ring(rng, 11, 130)
    status, counts, _ = run(emul, tmp_path / "full", plane, 5, 20)
    assert status == 0
    ns, nc, nb, _ = counts
    for k, caps in enumerate(((ns - 1, nc, nb), (ns, nc - 1, nb), (ns, nc, nb - 1), (0, 0, 0))):
        st, got_counts, out = run(emul, tmp_path / f"c{k}", plane, 5, 20, caps=caps)
        assert st == 1 and got_counts == counts and out is None
    check(emul, tmp_path / "exact", plane, 5, 20, caps=(ns, nc, nb))


def test_export_under_thread_sanitizer(tmp_path):
    """two SMs' worth of CTAs, the 1024-thread scan's shared memory and barriers, outputs written by many lanes: no
    data race, and the same bytes"""
    exe = _build(tmp_path, "thread")
    rng = np.random.default_rng(9)
    plane = ring(rng, 40, 150)
    env = dict(os.environ, TSAN_OPTIONS="halt_on_error=1")
    check(exe, tmp_path / "t", plane, 149, 7, sm=2, env=env)
