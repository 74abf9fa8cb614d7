"""The XOR chunk codec on an H100 against the plain references, at every format edge and on corrupted chunks.

Decoder (gpr_chunks_scatter), on the cases of tests/chunk_cases.py: the hand-written known answers and random-bit
series, from pageable, pinned and device memory (the data 0, 1, 7 and 15 bytes past a 16-byte boundary), into the
util plane and the power plane at 150 and 149.99 W, into the context plane (GPR_TEXT_FILL) and into the resident ring
at several newest columns: every cell bit-equal to the numpy model of the samples tests/chunks_ref.py decodes
(test_chunks_emul.model), with equal counts.  Not against gpr_samples_scatter: it shares scatter_sample with the code
under test.

Corrupted batches: thousands of corrupted chunks per seed among good ones, as host and device batches.  A batch whose
chunks all decode leaves the model's plane; a batch with a bad chunk fails with GPR_E_INVALID naming the reference's
first bad chunk and the kind the message rule picks from the reference's faults, leaves the destination byte for byte
as it was, and an _async decision enqueued before it completes with the right result.

Encoder (gpr_resident_export), on rings built by gpr_append from the row kinds of test_chunks_export_emul.ring, f32
neighbours of 150 W and rows of NaNs only: T in {1, 2, 31, 32, 33, 63, 64, 65, 120, 121, 1800}, the heads the CPU test
uses and a random one, per_chunk in {1, 2, 3, 31, 32, 33, 119, 120, 65535}; rows of k * M - 1, k * M and k * M + 1
present cells around the 32-chunk rounds of for_each_chunk; a ring of 40,000 rows.  The arrays byte for byte equal to
the reference encoder's (tests/chunks_encode.cpp), and tests/chunks_ref.py's decode of the chunks gives back the
unrolled ring with every NaN dropped."""
import functools

import numpy as np
import pytest

import chunk_cases as K
import chunks_ref as R
import export_ref as X
import test_chunks_emul as CE
import test_chunks_export_emul as EE
from test_chunk_cases import corrupt_batches, expected_fault
from test_gpu_resident_export import _read_ring
from test_gpu_samples import _engine, _plane, _torch_dev
from test_samples_emul import FILL, STEP, T, T_END, model as samples_model

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

T_S, STEP_S = T_END // 1000, STEP // 1000        # the window of the cases (ms) in the grid's seconds


@pytest.fixture(scope="module")
def eng():
    e = _engine()
    yield e
    e.close()


# ---- the decoder ----------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def _plan(seed):
    """the decoder plan as one batch, a row per series, and its samples decoded by the reference"""
    lists = [cs for _, cs in K.decoder_plan(seed, T_END, STEP, T)]
    b = CE.make(lists, np.arange(len(lists)), len(lists))
    return b, CE.decoded(b)


def _want(s, thr, col_end=T - 1, plane=None):
    d = dict(s, thr=thr or None, col_end=col_end, plane=s["plane"] if plane is None else plane)
    p, n_oow, n_tiny = samples_model(d)
    return p, {"n_in": len(s["ts"]), "n_oow": n_oow, "n_tiny": n_tiny}


def _scatter(eng, b, source, **kw):
    """gpr_chunks_scatter of batch b from `source` memory: pageable, pinned or device+<shift>"""
    import gpu_pruner_b200 as g
    n_rows, Tn = b["plane"].shape
    sc, rows, cb, data = b["series"], b["rows"], b["cbytes"], b["data"]
    if source == "pageable":
        return eng.chunks_scatter(sc, rows, cb, data, T_S, STEP_S, Tn, n_rows, **kw)
    if source == "pinned":
        pinned = eng.host_array(max(len(data), 1), np.uint8)
        pinned[:len(data)] = data
        return eng.chunks_scatter(sc, rows, cb, pinned[:len(data)], T_S, STEP_S, Tn, n_rows, **kw)
    shift = int(source.split("+")[1])
    raw = torch.zeros(len(data) + 16, dtype=torch.uint8, device="cuda")
    raw[shift:shift + len(data)] = torch.from_numpy(data).cuda()
    torch.cuda.synchronize()
    assert raw[shift:].data_ptr() % 16 == shift
    d = [_torch_dev(sc.view(np.int64)), _torch_dev(rows.view(np.int32)), _torch_dev(cb.view(np.int64))]
    return eng.chunks_scatter(*d, raw[shift:].data_ptr(), T_S, STEP_S, Tn, n_rows, mem_kind=g.ffi.GPR_MEM_DEVICE,
                              n_series=len(rows), **kw)


def _same(got, want, what):
    if not np.array_equal(got, want):
        r, c = np.argwhere(got != want)[0]
        raise AssertionError(f"{what}: cell ({r}, {c}) {got[r, c]:#010x} != {want[r, c]:#010x}")


@pytest.mark.parametrize("source", ["pageable", "pinned", "device+0", "device+1", "device+7", "device+15"])
def test_decoder_into_the_context_planes(eng, source):
    for seed in (1, 2):
        b, s = _plan(seed)
        n_rows = b["plane"].shape[0]
        for plane, thr in ((0, 0.0), (1, 150.0), (1, 149.99)):
            st = _scatter(eng, b, source, plane=plane, power_threshold=thr)
            want, counts = _want(s, thr if plane else None)
            _same(_plane(eng, n_rows, T, plane), want, (seed, source, plane, thr))
            assert st == counts, (seed, source, plane, thr)
            assert counts["n_oow"] > 0 and counts["n_tiny"] > 0 and (want != FILL).sum() > 2000


@pytest.mark.parametrize("source", ["pageable", "device+7"])
def test_decoder_into_the_resident_ring(eng, source):
    """the ring holds older values; its newest column at T - 1, 0, 17 and T - 2 (the head 0, 1, 18, T - 1)"""
    b, s = _plan(3)
    n_rows = b["plane"].shape[0]
    rng = np.random.default_rng(4)
    eng.resident_init(n_rows, 1, T, power_plane=True)
    old = rng.integers(0, 200, (n_rows, T)).astype(np.float32).view(np.uint32)
    old[rng.random(old.shape) < 0.3] = FILL     # no sample: the fill, as the ring's own gaps hold it
    eng.append(old.view(np.float32), old.view(np.float32))
    head = 0
    for want_head in (0, 1, 18, T - 1):
        eng.resident_advance((want_head - head) % T)
        head = want_head
        assert eng.resident_head() == head
        for plane, thr in ((0, 0.0), (1, 150.0)):
            before = _read_ring(eng, n_rows, T, 2)[plane]
            st = _scatter(eng, b, source, plane=plane, power_threshold=thr, resident=True)
            want, counts = _want(s, thr if plane else None, col_end=(head + T - 1) % T, plane=before)
            _same(_read_ring(eng, n_rows, T, 2)[plane], want, (source, head, plane))
            assert st == counts, (source, head, plane)


# ---- corrupted batches ----------------------------------------------------------------------------------------------
def _fails(eng, b, source, first, bits):
    import gpu_pruner_b200 as g
    with pytest.raises(g.GprError) as ei:
        _scatter(eng, b, source)
    assert ei.value.code == g.ffi.GPR_E_INVALID, (source, ei.value)
    want = f"chunk {first} is the first malformed one ({K.fault_text(bits)})"
    assert want in ei.value.message, (source, want, ei.value.message)


@pytest.mark.parametrize("seed", [11, 12])
def test_corrupted_batches(eng, seed):
    n_rows, n_ok, n_bad = 8, 0, 0
    batches = corrupt_batches(seed, n_rows, n_chunks=2500)
    current = None
    for k, (lists, rows, where) in enumerate(batches):
        b = CE.make(lists, rows, n_rows)
        bits, first = expected_fault(where)
        for source in ("pageable", "device+%d" % (k % 16)):
            if not bits:
                st = _scatter(eng, b, source)
                want, w_in, w_oow, w_tiny = CE.model(b)
                current = _plane(eng, n_rows, T)
                _same(current, want, (seed, k, source))
                assert st == {"n_in": w_in, "n_oow": w_oow, "n_tiny": w_tiny}, (seed, k, source)
                n_ok += 1
            else:
                _fails(eng, b, source, first, bits)
                if current is not None:
                    _same(_plane(eng, n_rows, T), current, ("untouched", seed, k, source))
                n_bad += 1
    assert n_ok > 30 and n_bad > 600, (n_ok, n_bad)


def test_failing_batches_keep_a_pending_decision(eng):
    """an _async decision on the plane, then failing host and device batches, then gpr_sync: the decision's result is
    the blocking decision's on the same plane, which the failures left as it was"""
    batches = corrupt_batches(13, 8, n_chunks=300)
    good = next(CE.make(l, r, 8) for l, r, w in batches if not w)
    _scatter(eng, good, "pageable")
    before = _plane(eng, 8, T)
    dbits = torch.zeros(1, dtype=torch.int32, device="cuda")
    r_async = eng.decide_ptr(eng.text_planes()[0], 4, 2, T, dbits, blocking=False)
    n = 0
    for k, (lists, rows, where) in enumerate(batches):
        if where and n < 40:
            bits, first = expected_fault(where)
            _fails(eng, CE.make(lists, rows, 8), ("pageable", "pinned", "device+1")[k % 3], first, bits)
            n += 1
    eng.sync()
    _same(_plane(eng, 8, T), before, "untouched")
    w_bits = torch.zeros(1, dtype=torch.int32, device="cuda")
    want = eng.decide_ptr(eng.text_planes()[0], 4, 2, T, w_bits)
    assert (r_async.n_series, r_async.n_candidates) == (want.n_series, want.n_candidates)
    assert torch.equal(dbits, w_bits) and n == 40


def test_a_short_chunk_after_a_bad_one(eng):
    """regression: a host batch whose chunk 1 runs past its bytes and whose chunk 3 is shorter than its header names
    chunk 1 and the short chunk's kind, as the device batch does (the host walk used to name chunk 3)"""
    from test_chunk_cases import short_after_bad
    b = short_after_bad()
    for source in ("pageable", "pinned", "device+0"):
        _fails(eng, b, source, 1, 32 | 64)


# ---- the encoder ----------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def native(tmp_path_factory):
    return R.build_native(str(tmp_path_factory.mktemp("encode")))


NEAR150 = (np.float32(150).view(np.uint32) + np.arange(-8, 9)).astype(np.uint32)   # 150 W and its 16 f32 neighbours


def _ring(rng, rows, Tn):
    """EE.ring's row kinds, then rows of f32 neighbours of 150 W (XOR windows of 29 to 33 leading zeros) and rows of
    NaNs only, of several payloads"""
    plane = EE.ring(rng, rows, Tn)
    for r in range(7, rows, 9):
        plane[r] = rng.choice(NEAR150, Tn)
    for r in range(8, rows, 9):
        plane[r] = rng.choice(EE.OTHER_NANS, Tn)
    return plane


def _load(eng, cols, head):
    """a ring whose cells oldest first are `cols`, at `head`, by gpr_append -> its plane as read back"""
    rows, Tn = cols.shape
    eng.resident_init(rows, 1, Tn)
    if head:
        eng.append(np.zeros((rows, head), np.float32))
    eng.append(cols.view(np.float32))
    assert eng.resident_head() == head
    plane = _read_ring(eng, rows, Tn, 1)[0]
    assert np.array_equal(X.canonical(X.unroll(plane, head)), X.canonical(cols))
    return plane


def _export_equal(eng, native, plane, head, M, decode_every=1):
    rows, Tn = plane.shape
    got = eng.resident_export(EE.T_END, EE.STEP, max_per_chunk=M)
    sc, rr, cb, data, n = X.export_native(plane, head, EE.T_END, EE.STEP, M, native)
    where = (Tn, head, M)
    assert got["n_samples"] == n, where
    for name, w in (("series_chunks", sc), ("rows", rr), ("chunk_bytes", cb), ("data", data)):
        assert np.array_equal(got[name], w), (name, where)
    keep = np.arange(0, len(rr), decode_every)
    sub = dict(got, rows=rr[keep])
    if decode_every > 1:
        from test_gpu_resident_export import _keep
        new_rows = np.full(len(rr), 0xFFFFFFFF, np.uint32)
        new_rows[keep] = rr[keep]
        sub["series_chunks"], sub["rows"], sub["chunk_bytes"], sub["data"] = _keep(got, new_rows)
    back = X.restore(sub["series_chunks"], sub["rows"], sub["chunk_bytes"], sub["data"], rows, Tn, EE.T_END, EE.STEP)
    want = X.canonical(X.unroll(plane, head))
    assert np.array_equal(back[sub["rows"]], want[sub["rows"]]), where
    return n


@pytest.mark.parametrize("Tn", [1, 2, 31, 32, 33, 63, 64, 65, 120, 121, 1800])
def test_encoder_byte_equal_at_every_head_and_chunk_size(eng, native, Tn):
    rng = np.random.default_rng(Tn)
    cols = _ring(rng, 9 if Tn == 1800 else 18, Tn)
    heads = sorted({0, 1 % Tn, Tn // 2, Tn - 1, int(rng.integers(0, Tn))})
    for head in heads:
        plane = _load(eng, cols, head)
        for M in (1, 2, 3, 31, 32, 33, 119, 120, 65535):
            _export_equal(eng, native, plane, head, M)


def test_encoder_rows_at_every_32_chunk_round(eng, native):
    """rows of k * M - 1, k * M and k * M + 1 present cells for k around the 32 chunks a warp takes per round, the
    cells spread so chunk starts fall at every lane of a window"""
    rng = np.random.default_rng(21)
    Tn = 256
    for M in (1, 2, 3):
        counts = sorted({k * M + d for k in (1, 2, 31, 32, 33, 63, 64, 65) for d in (-1, 0, 1)} - {0})
        counts = [c for c in counts if c <= Tn]
        cols = np.full((len(counts), Tn), X.FILL, np.uint32)
        for r, c in enumerate(counts):
            cols[r, np.sort(rng.choice(Tn, c, replace=False))] = EE.f32bits(rng.integers(0, 50, c))
        for head in (0, 77, Tn - 1):
            plane = _load(eng, cols, head)
            _export_equal(eng, native, plane, head, M)


def test_encoder_ring_of_40000_rows(eng, native):
    """more rows than the size and write passes' grids and more than one row per thread of the 1024-thread scan; the
    reference decode on every 16th series"""
    rng = np.random.default_rng(31)
    cols = _ring(rng, 40_000, 20)
    plane = _load(eng, cols, 13)
    for M in (7, 120):
        assert _export_equal(eng, native, plane, 13, M, decode_every=16) > 300_000
