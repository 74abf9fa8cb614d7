"""GPU: the device text scan (gpr_text_scan, gpr_text_scan_begin / _next: k_text_scan_chunk, k_publish_marks and the
producer threads in gpu-pruner_b200/csrc/gpr_api.cu) at every series density, from every source memory, and on a text
of more than 4 GiB.

The scan's contract (include/gpr.h, DESIGN.md §8c): the text is delivered in pieces of at most 2 MB (1 MB when pageable
text is staged in 1 MB chunks), and every piece has room for 16,384 markers of each kind.  So a text whose
`},"values":[` and `"]]` markers are at least 128 bytes apart always scans, from pageable, pinned or device memory
and at every GPR_TEXT_CHUNK_MB; a denser piece makes the scan return GPR_E_CAPACITY naming that piece, never wrong
or missing markers, and the context scans the next text as usual.  References:
  * markers: the offsets re.finditer finds (or, for the 4.5 GB text, arithmetic over fixed-length records);
  * whether a source declines, and which piece: the marker counts of its pieces;
  * the parse after the scan: the millisecond bucketing model of tests/test_gpu_text_numbers.py, cell by cell;
  * the binary's fallback: the same binary with GPR_INGEST=cpu and promql_mini's float64 evaluation.
"""
import ctypes as C
import json
import os
import random
import re
import subprocess

import numpy as np
import pytest

import hostlib as H
import promql_mini as Q
from test_gpu_text_numbers import FILL, _assert_cells, _assert_spans, _engine, _reference

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")
MB, GB = 1 << 20, 1 << 30
ROOM = 16384                                   # markers of each kind per piece
T_END, STEP, T = 1_700_000_000, 15, 12         # the 15 s daemon slice: 12 samples per series
OPEN, CLOSE = b'},"values":[', b'"]]'
# values of one length, so that every series of a pitch has its markers at the same offsets
VALUES = ["0.000", "1.000", "37.00", "100.0", "0.500", "12.25", "99.99", "1e-03", "2.5e2", "-0.00", "3.5e1"]
N_TEXT = 36 * MB + 333                         # every text: three 16 MB chunks, 18 or more 2 MB pieces


# ---- texts ---------------------------------------------------------------------------------------------------
def _samples(i, k):
    """the k samples of series i: 15 s apart, ending at T_END"""
    return [(str(T_END - STEP * (k - 1 - j)), VALUES[(i * 7 + j * 3) % len(VALUES)]) for j in range(k)]


_K = {}   # samples per series that fit a pitch, by (pitch, digits of the index, index mod len(VALUES))


def _record(i, pitch):
    """one series of the matrix response, `pitch` bytes long with its separating comma (as close to it as the
    densest form allows: an empty label map and one sample); up to T samples, a filler label takes the rest.
    -> (bytes, samples)"""
    if pitch < 42:
        return b'{"metric":{},"values":[[1,"0"]]},', [("1", "0")]
    key = (pitch, len(str(i)), i % len(VALUES))
    for k in ([_K[key]] if key in _K else range(T, 0, -1)):
        s = _samples(i, k)
        body = b'"values":[' + b",".join(b'[%s,"%s"]' % (t.encode(), v.encode()) for t, v in s) + b"]},"
        head = b'{"metric":{"i":"%d"' % i
        fill = pitch - len(head) - len(b'},') - len(body)
        if fill >= 0 or k == 1:
            _K[key] = k
            pad = b',"f":"' + b"x" * (fill - 7) + b'"' if fill >= 7 else b" " * max(fill, 0)
            return head + pad + b"}," + body, s
    raise AssertionError


class Text:
    """a Prometheus matrix response of about `n` bytes whose series have the pitches `pitch_at(offset)` asks for"""

    def __init__(self, n, pitch_at):
        parts = [b'{"status":"success","data":{"resultType":"matrix","result":[']
        self.samples = []
        size, i = len(parts[0]), 0
        while size < n - 64 * 1024:
            rec, s = _record(i, pitch_at(size))
            parts.append(rec)
            self.samples.append((i, s))
            size += len(rec)
            i += 1
        parts[-1] = parts[-1][:-1]                         # no comma after the last series
        parts.append(b"]}}")
        body = b"".join(parts)
        self.buf = body + b" " * (n - len(body))       # white space after the document
        self.n = len(self.buf)
        t = self.buf
        self.opens = np.array([m.start() for m in re.finditer(re.escape(OPEN), t)], np.uint64)
        self.closes = np.array([m.start() for m in re.finditer(re.escape(CLOSE), t)], np.uint64)
        assert len(self.opens) == len(self.closes) == len(self.samples)

    def pieces_over(self, unit):
        """(first piece of `unit` bytes holding more markers of a kind than its room, its counts) or None"""
        n_pieces = -(-self.n // unit)
        co = np.bincount((self.opens // unit).astype(np.int64), minlength=n_pieces)
        cc = np.bincount((self.closes // unit).astype(np.int64), minlength=n_pieces)
        bad = np.flatnonzero((co > ROOM) | (cc > ROOM))
        return None if len(bad) == 0 else (int(bad[0]), int(co[bad[0]]), int(cc[bad[0]]))

    def min_gap(self):
        return int(min(np.diff(self.opens).min(), np.diff(self.closes).min()))


def _mix(off):
    """dense and sparse stretches of about 1.5 MB in one text, none denser than the room"""
    return [128, 530, 4096, 200, 65536, 1024, 128, 320][(off // (3 * MB // 2)) % 8]


PITCHES = {"34B": 34, "100B": 100, "127B": 127, "128B": 128, "320B": 320, "530B": 530, "1KB": 1024, "3KB": 3000,
           "64KB": 65536, "mix": None}
_TEXTS = {}


def _text(name):
    if name not in _TEXTS:
        p = PITCHES[name]
        _TEXTS[name] = Text(N_TEXT, _mix if p is None else (lambda off, p=p: p))
    return _TEXTS[name]


# ---- sources -------------------------------------------------------------------------------------------------
# name -> (environment of the engine, memory the text is scanned from, piece size)
SOURCES = {
    "pageable-2MB-x8": ({}, "pageable", 2 * MB),
    "pageable-2MB-x1": ({"GPR_TEXT_UPLOAD_THREADS": "1"}, "pageable", 2 * MB),
    "pageable-1MB-x8": ({"GPR_TEXT_CHUNK_MB": "1"}, "pageable", 1 * MB),
    "pageable-1MB-x1": ({"GPR_TEXT_CHUNK_MB": "1", "GPR_TEXT_UPLOAD_THREADS": "1"}, "pageable", 1 * MB),
    "pageable-16MB-x8": ({"GPR_TEXT_CHUNK_MB": "16"}, "pageable", 2 * MB),
    "pageable-16MB-x1": ({"GPR_TEXT_CHUNK_MB": "16", "GPR_TEXT_UPLOAD_THREADS": "1"}, "pageable", 2 * MB),
    "pinned": ({}, "pinned", 2 * MB),
    "device": ({}, "device", 2 * MB),
}


class Source:
    def __init__(self, name):
        env, self.memory, self.unit = SOURCES[name]
        self.eng = _engine(**env)
        self.pinned = self.eng.host_array((N_TEXT + MB,), np.uint8) if self.memory != "pageable" else None
        self.dev = self.eng.device_alloc(N_TEXT + MB) if self.memory == "device" else None

    def put(self, buf):
        """-> (text argument, n_bytes, mem_kind) for the scan calls"""
        import gpu_pruner_b200 as g
        n = len(buf)
        if self.memory == "pageable":
            return np.frombuffer(buf, np.uint8), n, g.ffi.GPR_MEM_HOST
        self.pinned[:n] = np.frombuffer(buf, np.uint8)
        if self.memory == "pinned":
            return self.pinned, n, g.ffi.GPR_MEM_HOST
        self.eng.memcpy(self.dev, self.pinned, n, 1, 0)
        return self.dev, n, g.ffi.GPR_MEM_DEVICE

    def close(self):
        if self.dev is not None:
            self.eng.device_free(self.dev)
        self.eng.close()


@pytest.fixture(scope="module")
def sources():
    made = {}

    def get(name):
        if name not in made:
            made[name] = Source(name)
        return made[name]
    yield get
    for s in made.values():
        s.close()


def _scan_next(eng, cap):
    """one gpr_text_scan_next -> (rc, opens, closes, n_opens, n_closes, bytes_done, more)"""
    from gpu_pruner_b200.engine import _ptr
    o, c = np.full(max(cap, 1), 2**64 - 1, np.uint64), np.full(max(cap, 1), 2**64 - 1, np.uint64)
    no, nc, done, more = C.c_uint64(0), C.c_uint64(0), C.c_uint64(0), C.c_int32(0)
    rc = eng._lib.gpr_text_scan_next(eng.handle, _ptr(o), _ptr(c), cap, C.byref(no), C.byref(nc), C.byref(done),
                                     C.byref(more))
    return rc, o[:min(cap, no.value)], c[:min(cap, nc.value)], no.value, nc.value, done.value, more.value


def _error(eng):
    return (eng._lib.gpr_last_error(eng.handle) or b"").decode()


def _check_pieces(parts, text, unit, what):
    """the pieces of a pipelined scan: in text order, at most `unit` bytes each, markers inside their piece"""
    lo = 0
    for o, c, done in parts:
        assert lo < done <= text.n and done - lo <= unit, (what, lo, done)
        for m in (o, c):
            assert np.all(np.diff(m.astype(np.int64)) > 0) and (len(m) == 0 or (lo <= int(m[0]) and int(m[-1]) < done)), \
                (what, lo, done)
        lo = done
    assert lo == text.n, what
    assert np.array_equal(np.concatenate([p[0] for p in parts]), text.opens), what
    assert np.array_equal(np.concatenate([p[1] for p in parts]), text.closes), what


# ---- A. every density from every source -----------------------------------------------------------------------
def test_the_texts_have_the_pitches_they_are_named_for():
    for name, p in PITCHES.items():
        t = _text(name)
        gaps = np.diff(t.opens.astype(np.int64))
        if p is None:
            assert t.min_gap() >= 128 and {128, 530, 4096, 65536} <= set(np.unique(gaps).tolist()), name
        elif p < 42:
            assert gaps.max() == 33, name
        else:
            assert np.all(gaps == p), (name, np.unique(gaps)[:5])


@pytest.mark.parametrize("source", list(SOURCES))
@pytest.mark.parametrize("name", list(PITCHES))
def test_every_density_scans_alike_from_every_source(sources, source, name):
    """markers at least 128 B apart: the regex's markers from every source, blocking and piece by piece.  Denser:
    whatever the pieces of this source hold decides — a piece over its room declines with GPR_E_CAPACITY naming that
    piece, and the same context then scans the next text"""
    import gpu_pruner_b200 as g
    src, text = sources(source), _text(name)
    over = text.pieces_over(src.unit)
    if text.min_gap() >= 128:
        assert over is None, name                       # what the header promises
    if name == "34B":
        assert over is not None                         # denser than the room of every source
    arg, n, kind = src.put(text.buf)
    if over is None:
        o, c = src.eng.text_scan(arg, slot=1, n_bytes=n, mem_kind=kind)
        assert np.array_equal(o, text.opens), (source, name, np.setxor1d(o, text.opens)[:8])
        assert np.array_equal(c, text.closes), (source, name, np.setxor1d(c, text.closes)[:8])
        parts = list(src.eng.text_scan_chunks(arg, slot=1, n_bytes=n, mem_kind=kind))
        _check_pieces(parts, text, src.unit, (source, name))
        return
    k, no, nc = over
    piece = min(src.unit, text.n - k * src.unit)
    want = f"{no} / {nc} markers in the {piece} bytes of text at offset {k * src.unit}, room for {ROOM}"
    with pytest.raises(g.GprError) as e:
        src.eng.text_scan(arg, slot=1, n_bytes=n, mem_kind=kind)
    assert e.value.code == g.ffi.GPR_E_CAPACITY and want in e.value.message, (source, name, e.value.message)
    # piece by piece: every piece before the full one is delivered, then the same refusal
    src.eng._check(src.eng._lib.gpr_text_scan_begin(src.eng.handle, 1, g.engine._ptr(arg), n, kind))
    for j in range(k):
        rc, o, c, *_ = _scan_next(src.eng, ROOM)
        assert rc == 0, (source, name, j, _error(src.eng))
        lo, hi = j * src.unit, (j + 1) * src.unit
        assert np.array_equal(o, text.opens[(text.opens >= lo) & (text.opens < hi)]), (source, name, j)
    rc, _, _, a, b, _, _ = _scan_next(src.eng, ROOM)
    assert rc == g.ffi.GPR_E_CAPACITY and (a, b) == (no, nc) and want in _error(src.eng), (source, name)
    # the scan is over; the next one on the same context works
    ok = _text("530B")
    arg, n, kind = src.put(ok.buf)
    o, c = src.eng.text_scan(arg, slot=1, n_bytes=n, mem_kind=kind)
    assert np.array_equal(o, ok.opens) and np.array_equal(c, ok.closes), source


def _block_text(n_series, pitch, at):
    """sparse series (4 KB apart) around a block of `n_series` series of `pitch` bytes starting at offset `at`"""
    parts, size, i = [], 0, 0
    while size + 4096 <= at:
        rec, _ = _record(i, 4096)
        parts.append(rec)
        size, i = size + len(rec), i + 1
    parts.append(b" " * (at - size))
    for _ in range(n_series):
        rec, _ = _record(i, pitch)
        parts.append(rec)
        i += 1
    size = at + n_series * pitch
    nxt = -(-(at + 2 * MB) // (2 * MB)) * 2 * MB          # sparse again from the next 2 MB boundary
    parts.append(b" " * (nxt - size))
    while nxt + 4096 <= N_TEXT:
        rec, _ = _record(i, 4096)
        parts.append(rec)
        nxt, i = nxt + 4096, i + 1
    buf = b"".join(parts)
    return buf + b" " * (N_TEXT - len(buf))


@pytest.mark.parametrize("source", list(SOURCES))
def test_a_piece_holds_exactly_its_room(sources, source):
    """16,384 series of 64 bytes in the MB at 18 MB (one piece of every source: unit 9 of the second 16 MB chunk of
    pinned and device text) scan; 16,385 series of 63 bytes in the same MB decline, from every source"""
    import gpu_pruner_b200 as g
    src = sources(source)
    at = 18 * MB
    full = _block_text(ROOM, 64, at)
    over = _block_text(ROOM + 1, 63, at)
    for buf, fits in ((full, True), (over, False), (full, True)):
        opens = np.array([m.start() for m in re.finditer(re.escape(OPEN), buf)], np.uint64)
        closes = np.array([m.start() for m in re.finditer(re.escape(CLOSE), buf)], np.uint64)
        inside = (opens >= at) & (opens < at + MB)
        assert inside.sum() == (ROOM if fits else ROOM + 1)
        arg, n, kind = src.put(buf)
        if fits:
            o, c = src.eng.text_scan(arg, slot=0, n_bytes=n, mem_kind=kind)
            assert np.array_equal(o, opens) and np.array_equal(c, closes), source
        else:
            with pytest.raises(g.GprError) as e:
                src.eng.text_scan(arg, slot=0, n_bytes=n, mem_kind=kind)
            assert e.value.code == g.ffi.GPR_E_CAPACITY, e.value.message
            assert f"{ROOM + 1} / {ROOM + 1} markers in the {src.unit} bytes of text at offset {at}" in e.value.message


@pytest.mark.parametrize("source", ["pageable-2MB-x8", "pageable-16MB-x1", "pinned", "device"])
def test_a_cap_below_a_piece_can_be_retried(sources, source):
    """gpr_text_scan_next with a cap one short of the piece's count: GPR_E_CAPACITY with the true counts, the scan
    still open; the same call with the count as cap delivers that piece and the scan goes on to the end.
    gpr_text_scan with a whole-text cap one short reports the true totals."""
    import gpu_pruner_b200 as g
    src, text = sources(source), _text("mix")
    arg, n, kind = src.put(text.buf)
    eng = src.eng
    eng._check(eng._lib.gpr_text_scan_begin(eng.handle, 2, g.engine._ptr(arg), n, kind))
    parts, short, more = [], 0, 1
    while more:
        rc, o, c, no, nc, done, more = _scan_next(eng, 1)
        if rc == 0:
            assert no <= 1 and nc <= 1
            parts.append((o.copy(), c.copy(), done))
            continue
        assert rc == g.ffi.GPR_E_CAPACITY and "room for 1" in _error(eng), _error(eng)
        cap = max(no, nc) - 1
        if cap >= 1:
            rc, _, _, a, b, _, _ = _scan_next(eng, cap)
            assert rc == g.ffi.GPR_E_CAPACITY and (a, b) == (no, nc), _error(eng)
        rc, o, c, a, b, done, more = _scan_next(eng, max(no, nc))
        assert rc == 0 and (a, b) == (no, nc), _error(eng)
        parts.append((o.copy(), c.copy(), done))
        short += 1
    assert short > 10
    _check_pieces(parts, text, src.unit, source)
    from gpu_pruner_b200.engine import _ptr
    cap = len(text.opens) - 1
    o, c = np.zeros(cap, np.uint64), np.zeros(cap, np.uint64)
    no, nc = C.c_uint64(0), C.c_uint64(0)
    rc = eng._lib.gpr_text_scan(eng.handle, 0, _ptr(arg), n, kind, _ptr(o), _ptr(c), cap, C.byref(no), C.byref(nc))
    assert rc == g.ffi.GPR_E_CAPACITY and (no.value, nc.value) == (len(text.opens), len(text.closes)), _error(eng)
    o2, c2 = eng.text_scan(arg, slot=0, n_bytes=n, mem_kind=kind)
    assert np.array_equal(o2, text.opens) and np.array_equal(c2, text.closes)


def _spans(eng, text, opens, closes):
    spans = np.zeros(len(opens), eng.SPAN_DTYPE)
    spans["begin"] = opens + 12
    spans["end"] = closes[np.searchsorted(closes, opens + 12)] + 2
    spans["row"] = np.arange(len(opens))
    return spans


_REFS = {}


@pytest.mark.parametrize("resident", [False, True], ids=["plane", "ring"])
@pytest.mark.parametrize("source", ["pageable-16MB-x8", "pinned", "device"])
@pytest.mark.parametrize("name", ["530B", "mix"])
def test_dense_texts_parse_cell_by_cell(sources, name, source, resident):
    """the dense texts scanned from pageable (16 MB chunks), pinned and device memory, then parsed into a context
    plane or the resident ring: every cell and every span count equals the bucketing model"""
    src, text = sources(source), _text(name)
    eng = src.eng
    arg, n, kind = src.put(text.buf)
    o, c = eng.text_scan(arg, slot=0, n_bytes=n, mem_kind=kind)
    n_rows = len(o)
    grid = (T_END, T * STEP, STEP, T - 1)
    if name not in _REFS:
        _REFS[name] = _reference(text.samples, grid, n_rows, T)
    want, hard, counts = _REFS[name]
    spans = _spans(eng, text, o, c)
    if not resident:
        out = eng.text_parse(spans, T_END, STEP, T, n_rows, slot=0)
        got = np.empty((n_rows, T), np.uint32)
        eng.memcpy(got, eng.text_planes()[0], got.nbytes, 0, 1)
        _assert_spans(out, hard, counts, f"{name} {source} plane")
        _assert_cells(got, want, f"{name} {source} plane")
        return
    G = 4
    P = -(-n_rows // G)
    eng.resident_init(P, G, T)
    eng.resident_advance(T + 5)                     # every bucket opened, head away from 0
    head = eng.resident_head()
    col_end = (head + T - 1) % T
    # the model's ring: its newest bucket is column col_end instead of T - 1; rows beyond the series stay empty
    ring_want = np.full((P * G, T), FILL, np.uint32)
    ring_want[:n_rows] = np.roll(want, col_end - (T - 1), axis=1)
    out = eng.text_parse(spans, T_END, STEP, T, n_rows, slot=0, resident=True)
    got = np.empty((P * G, T), np.uint32)
    eng.memcpy(got, eng.resident_planes()[0], got.nbytes, 0, 1)
    _assert_spans(out, hard, counts, f"{name} {source} ring")
    _assert_cells(got, ring_want, f"{name} {source} ring (head {head})")
    assert np.all(got[n_rows:] == FILL)


# ---- A. the binary: a response too dense for the device scan ----------------------------------------------------
NOW = 1_700_000_000


def _dense_store(n_pods, per_pod, seed):
    """pods with `per_pod` series each, one sample per series, labels as short as the honour-labels query allows:
    about 100 bytes per series"""
    rng = random.Random(seed)
    store = []
    for p in range(n_pods):
        busy = rng.random() < 0.5                    # a pod is idle if any of its GPUs is: busy pods are busy on all
        for s in range(per_pod):
            v = rng.choice([3, 40, 100]) if busy else 0
            lab = {"pod": f"p{p}", "namespace": "n", "container": f"c{s}", "modelName": "m"}
            store.append(("DCGM_FI_DEV_GPU_UTIL", lab, [(NOW - 1, v)]))
    return store


def _response(store):
    parts = []
    for name, lab, samples in store:
        vals = ",".join('[%d,"%s"]' % (t, v) for t, v in samples)
        parts.append('{"metric":%s,"values":[%s]}' % (json.dumps(lab, separators=(",", ":")), vals))
    return ('{"status":"success","data":{"resultType":"matrix","result":[' + ",".join(parts) + "]}}").encode()


def _run_bin(prom, kube, ingest):
    cmd = [H.BIN, "--prometheus-url", f"file://{prom}", "--kube-fixture", str(kube), "-t", "1", "-g", "300",
           "--now", str(NOW), "-l", "json", "--honor-labels"]
    p = subprocess.run(cmd, capture_output=True, text=True, timeout=600, env=dict(os.environ, GPR_INGEST=ingest))
    assert p.returncode == 0, p.stderr[-3000:]
    msgs = [json.loads(l)["fields"]["message"] for l in p.stderr.splitlines() if l.startswith("{")]
    verdict = [m for m in msgs if m.startswith("Query returned")]
    sent = {(m.group(2), m.group(1)) for m in (re.match(r"Dry-run: Would have sent \[Deployment\] ([^:]+):dep-(\S+) for scaledown", x)
                                               for x in msgs) if m}
    return msgs, verdict, sent


def test_the_binary_falls_back_to_the_cpu_parser_when_the_scan_declines(tmp_path):
    """1,200 pods of 24 series, about 100 bytes a series: the first 2 MB piece holds more than 16,384 series, so the
    device scan declines and the binary takes the CPU text parser for the whole response; the verdict and the pods it
    would scale equal GPR_INGEST=cpu and promql_mini"""
    from test_gpu_promql import _kube
    store = _dense_store(1200, 24, 11)
    body = _response(store)
    opens = [m.start() for m in re.finditer(re.escape(OPEN), body)]
    assert len(opens) == len(store) and np.bincount(np.array(opens) // (2 * MB)).max() > ROOM
    prom, kube = tmp_path / "prom", tmp_path / "kube"
    prom.mkdir()
    (prom / "util.json").write_bytes(body)
    (prom / "query.json").write_text(json.dumps({"end": NOW, "step": 1}))
    _kube(kube, sorted({(lab["pod"], lab["namespace"]) for _, lab, _ in store}))
    msgs, verdict, sent = _run_bin(prom, kube, "gpu")
    note = [m for m in msgs if m.startswith("Device ingest")]
    assert len(note) == 1 and note[0].startswith("Device ingest not used (device scan: ") and \
        "markers in the 2097152 bytes of text at offset 0, room for 16384" in note[0], note
    _, verdict_cpu, sent_cpu = _run_bin(prom, kube, "cpu")
    db = [Q.series(name, lab, samples) for name, lab, samples in store]
    n_series, pods = Q.unique_pods(Q.evaluate_template(db, NOW, 1, honor_labels=True), honor_labels=True)
    assert verdict == verdict_cpu == [f"Query returned {n_series} series across {len(pods)} unique pods"], verdict
    assert sent == sent_cpu == set(pods) and 300 < len(pods) < 900, (len(sent), len(sent_cpu), len(pods))


# ---- B. a text of more than 4 GiB --------------------------------------------------------------------------------
REC = 512                       # bytes per series record
BIG_N = 8_800_000               # records: 4.5 GB
PRE = b'{"status":"success","data":{"resultType":"matrix","result":['


def _big_template():
    """a record with fixed-width fields: index i in the label (7 digits), samples 5, 10 + i % 90 and 1,000,000 + i
    at T_END - 30, T_END - 15 and T_END; -> (template, offset of the label digits, of the middle value, of the last
    value, of the open marker, of the close marker)"""
    head = b'{"metric":{"__name__":"DCGM_FI_DEV_GPU_UTIL","i":"0000000","f":"'
    tail = b'"},"values":[[%d,"5"],[%d,"00"],[%d,"0000000"]]},' % (T_END - 30, T_END - 15, T_END)
    rec = head + b"x" * (REC - len(head) - len(tail)) + tail
    assert len(rec) == REC
    lab = rec.index(b'"i":"') + 5
    mid = rec.index(b'"00"') + 1
    last = rec.index(b'"0000000"]]') + 1
    return rec, lab, mid, last, rec.index(OPEN), rec.index(CLOSE)


def _digits(arr, col, values, width):
    for k in range(width):
        arr[:, col + width - 1 - k] = (values // 10 ** k % 10 + ord("0")).astype(np.uint8)


def _mem_available():
    with open("/proc/meminfo") as f:
        for line in f:
            if line.startswith("MemAvailable:"):
                return int(line.split()[1]) * 1024
    return 0


@pytest.mark.slow
def test_a_text_over_4_gib_scans_and_parses_at_64_bit_offsets():
    import gpu_pruner_b200 as g
    n = len(PRE) + BIG_N * REC + 3
    plane_bytes = BIG_N * 3 * 4
    host_need = 2 * n + BIG_N * (g.IdleEngine.SPAN_DTYPE.itemsize + 2 * 8 + 3 * 4)
    if _mem_available() < host_need + 4 * GB:
        pytest.skip(f"needs {host_need / GB:.1f} GB of host memory, {_mem_available() / GB:.1f} GB available")
    free, _ = torch.cuda.mem_get_info()
    dev_need = 2 * n + plane_bytes + BIG_N * g.IdleEngine.SPAN_DTYPE.itemsize
    if free < dev_need + 2 * GB:
        pytest.skip(f"needs {dev_need / GB:.1f} GB of device memory, {free / GB:.1f} GB free")
    rec, lab, mid, last, o_off, c_off = _big_template()
    text = np.empty(n, np.uint8)
    text[:len(PRE)] = np.frombuffer(PRE, np.uint8)
    body = text[len(PRE):len(PRE) + BIG_N * REC].reshape(BIG_N, REC)
    body[:] = np.frombuffer(rec, np.uint8)
    idx = np.arange(BIG_N, dtype=np.int64)
    _digits(body, lab, idx, 7)
    _digits(body, mid, 10 + idx % 90, 2)
    _digits(body, last, 1_000_000 + idx, 7)
    body[-1, -1] = ord(" ")                                  # no comma after the last series
    text[-3:] = np.frombuffer(b"]}}", np.uint8)
    want_o = (len(PRE) + idx * REC + o_off).astype(np.uint64)
    want_c = (len(PRE) + idx * REC + c_off).astype(np.uint64)
    assert want_o[-1] > 2**32 and np.any((want_o < 2**32) & (want_o + 16 * MB > 2**32))
    eng = _engine()
    dev = None
    try:
        for source in ("pageable", "device"):
            if source == "device":
                dev = eng.device_alloc(n)
                eng.memcpy(dev, text, n, 1, 0)
                o, c = eng.text_scan(dev, n_bytes=n, mem_kind=g.ffi.GPR_MEM_DEVICE)
                eng.device_free(dev)
                dev = None
            else:
                o, c = eng.text_scan(text)
            for got, want, what in ((o, want_o, "opens"), (c, want_c, "closes")):
                bad = np.flatnonzero(got != want) if len(got) == len(want) else [len(got) - len(want)]
                assert len(bad) == 0, (source, what, bad[:8], [int(got[i]) for i in bad[:4]], [int(want[i]) for i in bad[:4]])
        spans = np.zeros(BIG_N, eng.SPAN_DTYPE)
        spans["begin"], spans["end"], spans["row"] = want_o + 12, want_c + 2, idx
        out = eng.text_parse(spans, T_END, STEP, 3, BIG_N, window_seconds=45)
        assert np.all(out["n_in"] == 3) and np.all(out["n_oow"] == 0) and not np.any(out["flags"] & 2), \
            np.flatnonzero((out["n_in"] != 3) | (out["flags"] & 2 != 0))[:8]
        first = int(np.searchsorted(want_o + 12, 2**32 - MB))
        rows = BIG_N - first
        got = np.empty((rows, 3), np.float32)
        eng.memcpy(got, eng.text_planes()[0] + first * 3 * 4, got.nbytes, 0, 1)
        i = idx[first:]
        want = np.stack([np.full(rows, 5.0), 10 + i % 90, 1_000_000 + i], 1).astype(np.float32)
        bad = np.flatnonzero((got != want).any(1))
        assert len(bad) == 0, [(int(first + b), got[b].tolist(), want[b].tolist()) for b in bad[:8]]
        print(f"\n[4.5 GB] {n} bytes, {BIG_N} series, {2 * BIG_N} markers from 2 sources, {rows} rows above 4 GiB - 1 MB")
    finally:
        if dev is not None:
            eng.device_free(dev)
        eng.close()
