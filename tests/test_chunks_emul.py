"""gpr_chunks_scatter on the CPU: k_chunks_check and k_chunks_scatter of gpu-pruner_b200/csrc/gpr_chunks.cuh, compiled
from their source under tests/cpp/cuda_shim.hpp (tests/cpp/chunks_emul.cpp), under AddressSanitizer +
UndefinedBehaviorSanitizer and ThreadSanitizer, against a numpy model: the chunks decoded by tests/chunks_ref.py, then
the samples path's model of the text rules (tests/test_samples_emul.py) — cell for cell, bit for bit, with the
sample, out-of-window and tiny counts:
  * ragged series of 120-sample chunks (and empty series, several series per row, overlapping chunks), the data at
    odd offsets from a 16-byte boundary;
  * special values: the staleness marker, +-Inf, -0.0, tiny values, the power plane at its threshold's neighbours;
  * host batches cut into tiny pieces of whole chunks: every chunk merged exactly once;
  * every malformed batch rejected by the check, host walk and kernel alike, naming the first bad chunk, with the
    plane untouched."""
import os
import subprocess

import numpy as np
import pytest

import chunks_ref as R
import emul_build
from chunks_ref import BitWriter
from test_samples_emul import FILL, SPECIAL, T, T_END, STEP, _extract_samples, model as samples_model

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NONE = 0xFFFFFFFFFFFFFFFF


def _extract_chunks():
    src = open(os.path.join(ROOT, "gpu-pruner_b200", "csrc", "gpr_chunks.cuh")).read()
    body = src[src.index("namespace chunks {") + len("namespace chunks {"):src.index("}  // namespace chunks")]
    assert "asm" not in body and "__shared__" not in body
    for name in ("k_chunks_scatter", "k_chunks_check", "decode_chunk", "chunk_faults", "bound_faults"):
        assert name in body, name
    return body


def _build(d, sanitize):
    (d / "chunks_extract.inc").write_text(_extract_chunks())
    (d / "samples_extract.inc").write_text(_extract_samples())
    (d / "text_kernel_extract.inc").write_text(emul_build.extract_parse_kernel())
    exe = d / ("chunks_emul_" + sanitize.replace(",", "_"))
    cmd = ["g++", "-std=c++20", "-O1", "-g", "-pthread", "-Wno-unknown-pragmas", "-fsanitize=" + sanitize,
           "-fno-omit-frame-pointer"]
    if sanitize != "thread":
        cmd.append("-fno-sanitize-recover=all")
    subprocess.run(cmd + ["-I", str(d), "-I", os.path.join(ROOT, "tests", "cpp"),
                          os.path.join(ROOT, "tests", "cpp", "chunks_emul.cpp"), "-o", str(exe)],
                   check=True, capture_output=True, text=True)
    return str(exe)


@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    return _build(tmp_path_factory.mktemp("chunks"), "address,undefined")


# ---- batches ----------------------------------------------------------------------------------------------------
def make(series_chunks_list, rows, n_rows, Tn=T, thr=None, col_end=None, plane=None):
    """series_chunks_list: per series, a list of chunk bytes"""
    sc, cb, data = R.batch(series_chunks_list)
    return dict(series=sc, rows=np.asarray(rows, np.uint32), cbytes=cb, data=data, T=Tn, t_end=T_END,
                t_lo=T_END - Tn * STEP, step=STEP, col_end=Tn - 1 if col_end is None else col_end, thr=thr,
                plane=np.full((n_rows, Tn), FILL, np.uint32) if plane is None else plane)


def decoded(b):
    """the batch's samples in CSR form, as the samples path's model takes them"""
    ts, vals, lengths = [], [], []
    for s in range(len(b["rows"])):
        n = 0
        for c in range(int(b["series"][s]), int(b["series"][s + 1])):
            t, v, fault = R.decode(b["data"][int(b["cbytes"][c]):int(b["cbytes"][c + 1])].tobytes())
            assert fault is None
            ts += t
            vals += v
            n += len(t)
        lengths.append(n)
    offsets = np.concatenate([[0], np.cumsum(lengths)]).astype(np.uint64)
    return dict(b, offsets=offsets, ts=np.array(ts, np.int64),
                values=np.array(vals, np.uint64).view(np.float64) if vals else np.zeros(0))


def model(b):
    s = decoded(b)
    plane, n_oow, n_tiny = samples_model(s)
    return plane, len(s["ts"]), n_oow, n_tiny


def _write(d, b, piece, shift):
    d.mkdir(parents=True, exist_ok=True)
    thr = b["thr"] if b["thr"] is not None else 0.0
    (d / "params.txt").write_text(" ".join(str(x) for x in (
        len(b["rows"]), b["plane"].shape[0], b["T"], b["t_end"], b["t_lo"], b["step"], b["col_end"], repr(float(thr)),
        piece, shift)) + "\n")
    b["series"].astype(np.uint64).tofile(d / "series.u64")
    b["rows"].astype(np.uint32).tofile(d / "rows.u32")
    b["cbytes"].astype(np.uint64).tofile(d / "cbytes.u64")
    b["data"].astype(np.uint8).tofile(d / "data.u8")
    b["plane"].astype(np.uint32).tofile(d / "plane.u32")


def run(exe, d, b, piece=0, shift=0, sm=1, env=None):
    _write(d, b, piece, shift)
    r = subprocess.run([exe, str(sm), str(d)], capture_output=True, text=True, timeout=1800, env=env)
    assert r.returncode == 0, r.stderr[-3000:]
    raw = np.fromfile(d / "out.bin", np.uint8)
    bad = int(raw[:4].view(np.uint32)[0])
    first, n_in, n_oow, n_tiny = (int(x) for x in raw[8:40].view(np.uint64))
    plane = raw[40:].view(np.uint32).reshape(b["plane"].shape)
    return bad, first, (n_in, n_oow, n_tiny), plane


def check(exe, d, b, **kw):
    bad, first, counts, plane = run(exe, d, b, **kw)
    assert bad == 0 and first == NONE
    want, w_in, w_oow, w_tiny = model(b)
    if not np.array_equal(plane, want):
        r, c = np.argwhere(plane != want)[0]
        raise AssertionError(f"cell ({r}, {c}): {plane[r, c]:#010x} != {want[r, c]:#010x}")
    assert counts == (w_in, w_oow, w_tiny)
    return b


def series_samples(rng, n, kind, t0=None):
    """one series' (ts, value bits): a scrape every STEP ms with jitter, from some seconds before the window on"""
    t0 = T_END - (T + 3) * STEP + int(rng.integers(-2000, 2000)) if t0 is None else t0
    ts = t0 + np.arange(n) * STEP + rng.integers(-3, 4, n) * (rng.random(n) < 0.3)
    if kind == "util":
        v = rng.integers(0, 101, n).astype(np.float64)
        v[rng.random(n) < 0.3] = 0.0
        ratio = rng.random(n) < 0.2
        v[ratio] = rng.random(int(ratio.sum()))
        v[rng.random(n) < 0.05] = np.nan
    elif kind == "special":
        v = rng.integers(0, 400, n).astype(np.float64)
        pick = rng.random(n) < 0.5
        v[pick] = rng.choice(SPECIAL, int(pick.sum()))
    else:   # "random": any bits
        v = rng.integers(0, 1 << 64, n, dtype=np.uint64).view(np.float64)
    bits = v.view(np.uint64).copy()
    bits[rng.random(n) < 0.05] = R.STALE_NAN_BITS
    return ts.tolist(), bits.tolist()


def ragged(rng, n_series, n_rows, kind="util", max_len=150, per_chunk=120, **kw):
    chunks = []
    for s in range(n_series):
        n = int(rng.integers(0, max_len))
        if n == 0 or rng.random() < 0.05:
            chunks.append([])
            continue
        ts, bits = series_samples(rng, n, kind)
        cs = R.split(ts, bits, per_chunk)
        if rng.random() < 0.1:   # an overlapping chunk from another block: order-independent merge
            cs.append(R.encode(ts[: n // 2], bits[: n // 2]))
        chunks.append(cs)
    return make(chunks, rng.integers(0, n_rows, n_series), n_rows, **kw)


def test_ragged_series_every_alignment(emul, tmp_path):
    """some 100 chunks over several warps' groups, the data at 0, 1, 7, 8 and 15 bytes past a 16-byte boundary"""
    rng = np.random.default_rng(1)
    b = ragged(rng, 90, 30)
    assert int(b["series"][-1]) > 64
    for shift in (0, 1, 7, 8, 15):
        check(emul, tmp_path / f"s{shift}", b, shift=shift)


def test_special_values_and_the_power_plane(emul, tmp_path):
    rng = np.random.default_rng(3)
    for thr in (150.0, 149.99, -2.0, None):
        b = ragged(rng, 40, 12, kind="special", thr=thr)
        check(emul, tmp_path / str(thr), b)
    # 149.999999 W stays below a 150 W threshold and 150.0000001 W reaches it; the staleness marker is dropped
    ts = [T_END - 2 * STEP, T_END - STEP, T_END]
    b = make([[R.encode(ts, [149.999999, 150.0000001, R.STALE_NAN_BITS])]], [0], 1, thr=150.0)
    got = run(emul, tmp_path / "edge", b)[3][0].view(np.float32)
    assert got[T - 3] < np.float32(150) and got[T - 2] == np.float32(150) and np.isnan(got[T - 1])
    check(emul, tmp_path / "edge2", b)


def test_resident_ring_wraps(emul, tmp_path):
    rng = np.random.default_rng(4)
    Tr = 10
    plane = np.full((6, Tr), FILL, np.uint32)
    plane[:, :5] = rng.integers(0, 60, (6, 5)).astype(np.float32).view(np.uint32)
    for col_end in (0, 3, 9):
        chunks = []
        for s in range(12):
            ts, bits = series_samples(rng, int(rng.integers(1, 30)), "util", t0=T_END - 15 * STEP)
            chunks.append(R.split(ts, bits, 7))
        b = make(chunks, rng.integers(0, 6, 12), 6, Tn=Tr, col_end=col_end, plane=plane)
        check(emul, tmp_path / f"r{col_end}", b)


@pytest.mark.parametrize("piece", [2, 40, 300, 1000, 5000])
def test_host_pieces_merge_every_chunk_once(emul, tmp_path, piece):
    """the host piece walk (samples::for_each_cut with gpr_api.cu's cut of whole chunks up to `piece` bytes) at tiny
    sizes, down to one chunk per piece and chunks larger than a piece: the counts, which a chunk merged twice or never
    would change, and every cell equal the model's"""
    rng = np.random.default_rng(10 + piece)
    b = ragged(rng, 50, 20, max_len=60, per_chunk=int(rng.choice([5, 17, 120])))
    check(emul, tmp_path / "p", b, piece=piece)
    check(emul, tmp_path / "pu", b, piece=piece, shift=5)


def test_empty_batches(emul, tmp_path):
    for k, lists in enumerate(([], [[], [], []], [[R.encode([], [])], []])):
        b = make(lists, np.zeros(len(lists), np.uint32), 2)
        check(emul, tmp_path / f"d{k}", b)
        check(emul, tmp_path / f"h{k}", b, piece=100)


def malformed_cases(rng):
    """name -> (batch, fault bit, first bad chunk); each batch otherwise good (chunk 2 is the bad one)"""
    good = [R.encode(*series_samples(rng, n, "util")) for n in (5, 9, 7, 4)]
    plane = rng.integers(0, 100, (8, T)).astype(np.float32).view(np.uint32)

    def with_chunk(c, **kw):
        lists = [[good[0], good[1]], [c, good[2]], [good[3]]]
        return make(lists, [1, 2, 7], 8, plane=plane, **kw)

    cases = {}
    b = with_chunk(good[2])
    cases["row >= n_rows"] = (dict(b, rows=np.array([1, 8, 7], np.uint32)), 1, None)
    sc = b["series"].copy()
    sc[1], sc[2] = sc[2], sc[1]
    cases["series_chunks decrease"] = (dict(b, series=sc), 2, None)
    cases["series_chunks[0] != 0"] = (dict(b, series=b["series"] + np.uint64(1)), 4, None)
    cb = b["cbytes"].copy()
    cb[0] = 1
    cases["chunk_bytes[0] != 0"] = (dict(b, cbytes=cb), 8, 0)
    cb = b["cbytes"].copy()
    cb[3] = cb[2] - 1
    cases["chunk_bytes decrease"] = (dict(b, cbytes=cb), 16, 2)
    cases["chunk of 1 byte"] = (with_chunk(b"\x00"), 32, 2)
    cases["chunk of 0 bytes"] = (with_chunk(b""), 32, 2)
    full = R.encode(*series_samples(rng, 6, "util"))
    cases["ends mid-sample"] = (with_chunk(full[:-2]), 64, 2)
    cases["count past the stream"] = (with_chunk(b"\x00\x30" + full[2:]), 64, 2)
    reuse = BitWriter().varint(0).put(0, 64).uvarint(1).string("10").put(0, 8).chunk(2)
    cases["reuse before a window"] = (with_chunk(reuse), 128, 2)
    long = BitWriter().put((1 << 80) - 1, 80).byte(1).put(0, 64).chunk(1)
    cases["varint past 64 bits"] = (with_chunk(long), 256, 2)
    return good, plane, cases


def test_malformed_batches_leave_the_plane_untouched(emul, tmp_path):
    rng = np.random.default_rng(6)
    good, plane, cases = malformed_cases(rng)
    ok = make([[good[0], good[1]], [good[2]], [good[3]]], [1, 2, 7], 8, plane=plane)
    check(emul, tmp_path / "ok", ok)
    k = 0
    for name, (b, bit, first) in cases.items():
        for piece in (0, 64):
            k += 1
            bad, got_first, counts, got = run(emul, tmp_path / f"bad{k}", b, piece=piece)
            assert bad & bit, (name, piece, bad)
            if first is not None:
                assert got_first == first, (name, piece, got_first)
            assert np.array_equal(got, plane) and counts[1:] == (0, 0), (name, piece)


def test_scatter_under_thread_sanitizer(tmp_path):
    """16 CTAs (two SMs' worth) of ragged series that share rows, whole and in host pieces: the merges of concurrent threads into one cell go through atomics only.  Values are non-negative: the
    merge of a negative value reads its cell before its compare-and-swap, which the GPU's memory model allows and
    C++'s calls a race."""
    exe = _build(tmp_path, "thread")
    rng = np.random.default_rng(8)
    chunks = []
    for s in range(60):
        ts, bits = series_samples(rng, int(rng.integers(0, 250)), "util")
        bits = [b & 0x7FFFFFFFFFFFFFFF for b in bits]
        chunks.append(R.split(ts, bits) if ts else [])
    b = make(chunks, rng.integers(0, 4, 60), 4)
    env = dict(os.environ, TSAN_OPTIONS="halt_on_error=1")
    want, w_in, w_oow, w_tiny = model(b)
    for piece in (0, 3000):
        bad, _, counts, plane = run(exe, tmp_path / f"t{piece}", b, piece=piece, sm=2, env=env)
        assert bad == 0 and np.array_equal(plane, want) and counts == (w_in, w_oow, w_tiny)


def test_known_answer_chunks_on_the_device_decoder(emul, tmp_path):
    """the hand-written chunks of tests/test_chunks_ref.py, every one inside the window, through the kernels' decoder:
    both ends of every delta-of-delta bucket (a sample a bucket's width off lands in another column), the leading-zero
    clamp, 64 significant bits written as 0, window reuse, the staleness marker, +-Inf and -0.0"""
    import test_chunks_ref as K
    t0, d1 = T_END - 30 * STEP, STEP
    chunks = []
    for dod, prefix, sz in K.DOD_CASES:
        if abs(dod) < 20 * STEP:
            chunks.append(R.encode([t0, t0 + d1, t0 + 2 * d1 + dod, t0 + 3 * d1 + dod], [5.0, 6.0, 7.0, 8.0]))
    for payload_sz in (14, 17, 20):
        half = 1 << (payload_sz - 1)
        prefix = {14: "10", 17: "110", 20: "1110"}[payload_sz]
        for payload in (half, half + 1, (1 << payload_sz) - 1):
            dod = payload if payload <= half else payload - (1 << payload_sz)
            if abs(dod) < 20 * STEP:
                chunks.append(K._two(t0, 1.0).uvarint(d1).bit(0).string(prefix).put(payload, payload_sz).bit(0)
                              .chunk(3))
    v0 = 0x4059000000000000
    for vals in ([0, 0x0000000000F00000], [0, 0x8000000000000001],
                 [v0, v0 ^ 0x000ABC0000000000, v0 ^ 0x000ABC0000000000 ^ 0x0008040000000000,
                  v0 ^ 0x000ABC0000000000 ^ 0x0008040000000000 ^ 0x0000000000000F00],
                 [R.STALE_NAN_BITS, R.f2b(float("inf")), R.f2b(-0.0), R.f2b(float("-inf")), R.f2b(0.0), R.f2b(7.0)]):
        chunks.append(R.encode([t0 + k * d1 for k in range(len(vals))], vals))
    b = make([[c] for c in chunks], np.arange(len(chunks)) % 7, 7)
    check(emul, tmp_path / "kat", b)
    check(emul, tmp_path / "kat_h", b, piece=64, shift=9)
