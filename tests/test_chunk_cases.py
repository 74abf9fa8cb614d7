"""CPU: the seeded chunk cases of tests/chunk_cases.py, and the corrupted ones through the kernels' source.

  * the plans are reproducible (pinned digests), bounded, and reach every format path coverage() knows; the coverage
    decoder equals tests/chunks_ref.py's on every case;
  * corrupted chunks mixed into good batches go through k_chunks_check and k_chunks_scatter compiled from their
    source under AddressSanitizer + UndefinedBehaviorSanitizer (tests/cpp/chunks_emul.cpp), as device batches and as
    host batches cut into small pieces: a batch whose chunks all decode leaves the numpy model's plane
    (test_chunks_emul.model); a batch with a bad chunk reports exactly the reference's faults and its first bad chunk,
    and leaves the plane as it was;
  * the encoder at the top end of every delta-of-delta bucket, which gpr_resident_export cannot reach (its timestamps
    are whole seconds, and no bucket's top end is a multiple of 1000 ms): k_export_* from their source on a ring whose
    step is 4096 ms, byte for byte against the reference encoder.
tests/test_gpu_chunk_codec.py runs the same cases on an H100."""
import subprocess

import numpy as np
import pytest

import chunk_cases as K
import chunks_ref as R
import test_chunks_emul as CE
import test_chunks_export_emul as EE
from test_samples_emul import FILL, STEP, T, T_END

SEEDS = (1, 2, 3)
# sha256 of each seed's plan (test_plans_are_reproducible): a change of a generator changes the cases every test runs
PINNED = {
    ("decoder", 1): "3ed66ace49c96645fe70d05363f2fe01cabdb5c43a0aa9a9c1ee44081632d5c7",
    ("corrupt", 1): "0702bb527b5fe88fd632e9ef112debccc5efee2e030f2be3b8ca7944d0a9ad90",
    ("corrupt", 2): "a84bed7f42b3c745ea9ea1c9c53724ea4b2984ff608234682f782ff58f73aec3",
}


def _chunks_of_decoder_plan(seed):
    return [c for _, cs in K.decoder_plan(seed, T_END, STEP, T) for c in cs]


def test_plans_are_reproducible_and_bounded():
    for (kind, seed), want in PINNED.items():
        if kind == "decoder":
            a, b = _chunks_of_decoder_plan(seed), _chunks_of_decoder_plan(seed)
        else:
            a, b = ([c for _, c, _ in K.corrupt_plan(seed, T_END, STEP, T)] for _ in range(2))
        assert K.digest(a) == K.digest(b) == want, (kind, seed, K.digest(a))
        assert sum(len(c) for c in a) < 4 << 20 and len(a) < 20_000
    assert K.digest(_chunks_of_decoder_plan(1)) != K.digest(_chunks_of_decoder_plan(2))


def test_known_answers_decode_and_land_in_the_window():
    """every hand-written chunk is well formed, and its samples one column apart land inside the window"""
    for name, c in K.known_answers(T_END, STEP, T):
        ts, vals, fault = R.decode(c)
        assert fault is None, name
        if name.startswith(("dod", "window", "lead", "64 sig")):
            assert T_END - T * STEP < ts[2 if name.startswith("dod") else 1] <= T_END, name


def test_plans_reach_every_format_path():
    seen = set()
    for seed in SEEDS:
        for c in _chunks_of_decoder_plan(seed) + [c for _, c, _ in K.corrupt_plan(seed, T_END, STEP, T)]:
            paths, got = K.coverage(c)
            assert got == R.decode(c)
            seen |= paths
    assert seen == K.PATHS, sorted(K.PATHS - seen)
    # and the known answers alone reach every path of a well-formed chunk
    kat = set().union(*(K.coverage(c)[0] for _, c in K.known_answers(T_END, STEP, T)))
    assert kat == K.PATHS - {"short", "overrun", "no_window", "varint"}, sorted(K.PATHS - kat)


# ---- corrupted chunks through the kernels' source ------------------------------------------------------------------
def corrupt_batches(seed, n_rows=8, per_batch=24, n_chunks=2000, max_bad=3):
    """-> [(series chunk lists, rows, bad: [(chunk index, fault bit)])]: the n_chunks corrupted chunks of
    corrupt_plan(seed) in batches among good chunks; batches of chunks that all decode, and batches with 1 to max_bad
    bad chunks"""
    rng = np.random.default_rng(seed)
    plan = K.corrupt_plan(seed, T_END, STEP, T, n_chunks)
    decodes = [c for _, c, v in plan if v[2] == 0]
    bad = [(c, v[2]) for _, c, v in plan if v[2]]
    out = []
    while decodes or bad:
        chunks = [R.encode(*K.random_series(rng, int(rng.integers(1, 30)), T_END, STEP, T))
                  for _ in range(int(rng.integers(2, 8)))]
        take = min(len(decodes), per_batch - len(chunks))
        chunks += decodes[:take]
        del decodes[:take]
        faults = []
        if rng.random() < 0.5 or not decodes:
            k = min(len(bad), int(rng.integers(1, max_bad + 1)))
            chunks += [c for c, _ in bad[:k]]
            faults = [f for _, f in bad[:k]]
            del bad[:k]
        order = rng.permutation(len(chunks))
        chunks = [chunks[i] for i in order]
        n_good = len(chunks) - len(faults)
        where = [(int(np.flatnonzero(order == n_good + j)[0]), f) for j, f in enumerate(faults)]
        cuts = np.sort(rng.integers(0, len(chunks) + 1, int(rng.integers(1, 6))))
        lists = [chunks[a:b] for a, b in zip(np.concatenate([[0], cuts]), np.concatenate([cuts, [len(chunks)]]))]
        out.append((lists, rng.integers(0, n_rows, len(lists)), sorted(where)))
    return out


def expected_fault(where):
    """(fault bits of the batch, its first bad chunk) as the reference classifies its chunks"""
    bits = 0
    for _, f in where:
        bits |= f
    return bits, (where[0][0] if where else None)


@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    return CE._build(tmp_path_factory.mktemp("chunk_cases"), "address,undefined")


@pytest.mark.parametrize("seed", SEEDS[:2])
def test_corrupted_chunks_in_good_batches(emul, tmp_path, seed):
    rng = np.random.default_rng(100 + seed)
    n_rows = 8
    base = rng.integers(0, 100, (n_rows, T)).astype(np.float32).view(np.uint32)
    n_ok = n_bad = 0
    batches = corrupt_batches(seed, n_rows, per_batch=40, n_chunks=600, max_bad=6)
    for k, (lists, rows, where) in enumerate(batches):
        b = CE.make(lists, rows, n_rows, plane=base.copy(), thr=150.0 if k % 3 == 0 else None)
        bits, first = expected_fault(where)
        for piece, shift in ((0, k % 16), (64, 3))[:1 + (k % 3 == 0)]:   # a host batch in small pieces every third
            if not bits:
                CE.check(emul, tmp_path / f"b{k}_{piece}", b, piece=piece, shift=shift)
                n_ok += 1
                continue
            bad, got_first, counts, got = CE.run(emul, tmp_path / f"b{k}_{piece}", b, piece=piece, shift=shift)
            assert (bad, got_first) == (bits, first), (k, piece, where, bad, got_first)
            assert np.array_equal(got, base) and counts == (0, 0, 0), (k, piece)
            n_bad += 1
    assert n_ok >= 3 and n_bad > 50, (n_ok, n_bad)


def short_after_bad():
    """regression: a host batch whose chunk 1 runs past its bytes and whose chunk 3 is shorter than its header names
    chunk 1, and reports both faults, as a device batch does (the host walk used to stop at the short chunk)"""
    good = R.encode([T_END - 5000, T_END - 4000], [1.0, 2.0])
    lists = [[good, good[:-1]], [good, b"\x00"], [good]]
    b = CE.make(lists, [0, 1, 2], 3)
    return b


def test_short_chunk_after_a_bad_one_in_the_shim(emul, tmp_path):
    b = short_after_bad()
    for piece in (0, 64):
        bad, first, _, got = CE.run(emul, tmp_path / f"p{piece}", b, piece=piece)
        assert (bad, first) == (32 | 64, 1), (piece, bad, first)
        assert np.array_equal(got, b["plane"])


# ---- the encoder at the top end of every bucket --------------------------------------------------------------------
def _export(exe, d, plane, head, M, t_end_ms, step_ms):
    """the export emulator on a ring whose step is any number of ms -> (series_chunks, rows, chunk_bytes, data)"""
    d.mkdir(parents=True, exist_ok=True)
    rows, Tn = plane.shape
    big = 1 << 62
    (d / "params.txt").write_text(f"{rows} {Tn} {head} {M} {t_end_ms} {step_ms} {big} {big} {big}\n")
    np.ascontiguousarray(plane, np.uint32).tofile(d / "plane.u32")
    r = subprocess.run([exe, "1", str(d)], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    raw = np.fromfile(d / "out.bin", np.uint8)
    status, ns, nc, nb, _ = (int(x) for x in raw[:40].view(np.uint64))
    assert status == 0
    o = 40
    sc = raw[o:o + 8 * (ns + 1)].view(np.uint64)
    o += 8 * (ns + 1)
    cb = raw[o:o + 8 * (nc + 1)].view(np.uint64)
    o += 8 * (nc + 1)
    rr = raw[o:o + 4 * ns].view(np.uint32)
    return sc, rr, cb, raw[o + 4 * ns:o + 4 * ns + nb]


def test_encoder_at_every_bucket_top_in_the_shim(tmp_path):
    """step 4096 ms: a row whose gaps go 1, 3, 1 cells has dods of 8192 = 2^13, the top of the 14-bit bucket, and
    -8192, one past its bottom; gaps of 1, 17 give +-2^16 and 1, 129 give +-2^19"""
    exe = EE._build(tmp_path, "address,undefined")
    step_ms, t_end_ms, Tn = 4096, 1_700_000_000_000, 400
    plane = np.full((8, Tn), FILL, np.uint32)
    for r, gaps in enumerate(([1, 3, 1], [1, 17, 1], [1, 129, 1], [3, 1, 3], [17, 1, 17], [129, 1, 129],
                              [2, 3, 2, 1], [2, 18, 1, 130])):
        cols = np.cumsum([5] + gaps)
        plane[r, cols] = np.float32(r + 1.5).view(np.uint32)
    want_dods = {8192, -8192, 65536, -65536, 524288, -524288}
    for head in (0, 123):
        ring = np.roll(plane, head, axis=1)       # unrolled from `head`, the ring is `plane`
        sc, rr, cb, data = _export(exe, tmp_path / f"h{head}", ring, head, 120, t_end_ms, step_ms)
        series = []
        dods = set()
        for r in range(plane.shape[0]):
            js = np.flatnonzero(plane[r] != FILL)
            ts = [t_end_ms - (Tn - 1 - int(j)) * step_ms for j in js]
            dods |= set(np.diff(ts, 2).tolist())
            series.append(R.split(ts, [R.f2b(float(plane[r, j].view(np.float32))) for j in js], 120))
        assert want_dods <= dods
        w_sc, w_cb, w_data = R.batch(series)
        assert np.array_equal(rr, np.arange(plane.shape[0])) and np.array_equal(sc, w_sc)
        assert np.array_equal(cb, w_cb) and np.array_equal(data, w_data), head
