"""The ring sequences of tests/test_gpu_session_ring.py, generated without a device (tests/ring_session_ops.py): the plans
are reproducible and stay within their bounds, every operation, failure and transition occurs across the seeds, and
the references the GPU test holds the library to agree with each other on everything the plans do: the export
reference with the C++ encoder, the reference decoder's restore of every export with the model's canonical window, and
every merge slice written as samples, as XOR chunks and as text with the same model cells and counts.  The call
sequences of tests/session_ops.py stay what they were."""
import hashlib
import json

import numpy as np
import pytest

import chunks_ref as CR
import export_ref as X
import ring_session_ops as RO
import session_ops as S
from test_samples_emul import model as samples_model


@pytest.fixture(scope="module")
def plans():
    return {seed: RO.plan_ring(seed) for seed in RO.SEEDS}


@pytest.fixture(scope="module")
def replays(plans):
    out = {}
    for seed, ops in plans.items():
        steps = []
        for op, res, md in RO.replay(ops):
            m = md.ring
            steps.append((op, res, None if m is None else ([p.copy() for p in m.planes], m.head, m.T),
                          md.t_end, md.pending))
        out[seed] = steps
    return out


# sha256 of every sequence of tests/session_ops.py as JSON (sorted keys), first 16 hex digits: the sequences the
# mixed-call session test has always run
SESSION_PLANS = ["576cf593d2aa055f", "f748889f2aa3c10b", "442735685cc2b90f", "e580d15bf5b89022", "7cfe44ca1d28a3fd",
                 "b4abdb4642153c79", "2bf45b5b24162788", "911be2ebaaf89327", "0e78bb4abb99cb3c", "bcc473c73a2dfe58",
                 "07c2a2f336d2e71a", "b4352ddf42eb6bae"]


def test_session_plans_are_unchanged():
    got = [hashlib.sha256(json.dumps(S.plan(s), sort_keys=True).encode()).hexdigest()[:16] for s in S.SEEDS]
    assert got == SESSION_PLANS


def test_plans_are_reproducible_and_bounded(plans, replays):
    assert RO.plan_ring(2) == plans[2]
    for seed, ops in plans.items():
        assert RO.N_OPS <= len(ops) <= RO.N_OPS + 40, (seed, len(ops))
        for i, (op, _, ring, _, pending) in enumerate(replays[seed]):
            assert pending <= RO.MAX_PENDING - 1, (seed, i)
            if op["kind"] == "init":
                r = op["ring"]
                assert r["P"] in RO.PS and r["G"] in RO.GS and r["T"] in RO.TS, (seed, i)
                assert r["P"] * r["G"] * r["T"] <= RO.MAX_RING_CELLS
            if ring is not None:
                assert sum(p.size for p in ring[0][:1]) <= RO.MAX_RING_CELLS, (seed, i)
            if op["kind"] in ("append", "advance", "merge") and ring is not None:
                T = ring[2]
                assert op["n_new"] in (1, max(1, T - 1), T, T + 5, max(1, T // 3)), (seed, i, op["n_new"], T)
            if op["kind"] == "merge":
                assert op["n_rows"] <= ring[0][0].shape[0]
                assert op["src"] in RO.MERGE_SOURCES and op["M"] in RO.CHUNK_M
            if op["kind"] == "export":
                assert op["M"] in RO.EXPORT_M


def test_every_operation_failure_and_transition_occurs(plans, replays):
    kinds = {op["kind"] for ops in plans.values() for op in ops}
    assert kinds == set(RO.KINDS), set(RO.KINDS) - kinds
    seen = set()
    for seed, ops in plans.items():
        fails = {op["fail"] for op in ops if op["kind"] == "fail"}
        assert fails == set(RO.FAILURES), (seed, set(RO.FAILURES) - fails)
        t = RO.transitions(ops)
        # every failure of every sequence finds results pending, which it must leave pending
        assert {f for f in RO.FAILURES if "fail " + f + " with results pending" in t} == set(RO.FAILURES), seed
        first_init = min(i for i, op in enumerate(ops) if op["kind"] == "init")
        assert all(i < first_init for i, op in enumerate(ops) if op.get("fail") in RO.NO_RING), seed
        seen |= t
    assert set(RO.TRANSITIONS) <= seen, set(RO.TRANSITIONS) - seen
    ops = [op for o in plans.values() for op in o]
    assert {op["src"] for op in ops if op["kind"] == "merge"} == set(RO.MERGE_SOURCES)
    assert {op["M"] for op in ops if op["kind"] == "export"} == set(RO.EXPORT_M)
    assert {(op["how"], op["mem"]) for op in ops if op["kind"] == "remap"} == {
        (h, m) for h in ("recipe", "random") for m in ("host", "dev")}
    assert {op["out"] for op in ops if op["kind"] == "live_rows"} == {"host", "dev"}
    assert {op["plane"] for op in ops if op["kind"] == "merge"} == {0, 1}
    assert {op["ring"]["T"] for op in ops if op["kind"] == "init"} == set(RO.TS)
    assert any(op["n_rows"] < r[0][0].shape[0] for steps in replays.values() for op, _, r, _, _ in steps
               if op["kind"] == "merge"), "no merge with grid.n_rows < P * G"


@pytest.fixture(scope="module")
def native_encoder(tmp_path_factory):
    return CR.build_native(str(tmp_path_factory.mktemp("chunks_encode")))


def _exports(replays):
    """(seed, step, plane cells, head, t_end, M, the reference's export) of every export the plans check"""
    for seed, steps in replays.items():
        for i, (op, res, ring, t_end, _) in enumerate(steps):
            k = op["kind"]
            if k == "export" or (k == "fail" and op["fail"] == "export_capacity"):
                yield seed, i, ring[0][op["plane"]], ring[1], t_end, op["M"], res["export"]
            elif k == "restore":
                for pl, ex in enumerate(res["exports"]):
                    yield seed, i, ring[0][pl], ring[1], t_end, 120, ex


def test_exports_equal_the_native_encoder_and_restore_to_the_canonical_window(replays, native_encoder):
    n = 0
    for seed, i, plane, head, t_end, M, ex in _exports(replays):
        nat = X.export_native(plane, head, t_end, RO.STEP, M, exe=native_encoder)
        for k, (a, b) in enumerate(zip(ex, nat)):
            assert np.array_equal(a, b) if k < 4 else a == b, (seed, i, k)
        sc, rows, cb, data, _ = ex
        T = plane.shape[1]
        back = X.restore(sc, rows, cb, data, plane.shape[0], T, t_end, RO.STEP)
        assert np.array_equal(back, X.canonical(X.unroll(plane, head))), (seed, i)
        n += 1
    assert n >= 3 * len(replays)


def _parsed_text(text, order):
    """the samples of a rendered slice read back: (ts ms, value f64) per span, in order"""
    out = []
    body = text.decode()
    at = 0
    for _ in order:
        at = body.index('"values":[', at) + len('"values":[')
        end = body.index("]]", at) + 1
        pairs = json.loads("[" + body[at:end] + "]")
        at = end
        ts = [int(round(float(t) * 1000)) for t, _ in pairs]
        vals = [float(v.replace("Inf", "inf")) for _, v in pairs]
        out.append((ts, vals))
    return out


def test_merge_slices_agree_as_samples_chunks_and_text(replays):
    """every merge slice: the model's cells and counts are the same whether the slice is taken as decoded samples, as
    the XOR chunks the GPU test sends (decoded by tests/chunks_ref.py) or as the text it sends (parsed back)"""
    n = 0
    for seed, steps in replays.items():
        for i in range(1, len(steps)):
            op, res, ring, t_end, _ = steps[i]
            if op["kind"] != "merge":
                continue
            planes_before = steps[i - 1][2][0]
            T, head = ring[2], ring[1]
            col_end = (head + T - 1) % T
            base = planes_before[op["plane"]].copy()
            base[:, (col_end - np.arange(min(op["n_new"], T))) % T] = RO.RS.NO_SAMPLE   # the opened buckets
            offsets, rows, ts, bits = RO.merge_slice(op, T, t_end)

            def model_of(o, t, b):
                return samples_model(RO.samples_batch(op, o, rows, t, b, base, T, t_end, col_end))
            want, w_oow, w_tiny = model_of(offsets, ts, bits)
            assert np.array_equal(want, ring[0][op["plane"]]), (seed, i)
            assert res["stats"] == (len(ts), w_oow, w_tiny), (seed, i)
            # as chunks
            sc, cb, data = RO.slice_chunks(op, offsets, ts, bits)
            cts, cbits, counts = [], [], []
            for s in range(len(rows)):
                k = 0
                for c in range(int(sc[s]), int(sc[s + 1])):
                    t, v, fault = CR.decode(bytes(data[int(cb[c]):int(cb[c + 1])]))
                    assert fault is None and len(t) <= op["M"]
                    cts += t
                    cbits += v
                    k += len(t)
                counts.append(k)
            co = np.concatenate([[0], np.cumsum(counts)]).astype(np.uint64)
            got, g_oow, g_tiny = model_of(co, np.array(cts, np.int64), np.array(cbits, np.uint64))
            assert np.array_equal(got, want) and (g_oow, g_tiny) == (w_oow, w_tiny), (seed, i, "chunks")
            # as text
            text, order = RO.text_of(offsets, rows, ts, bits)
            assert order == [int(r) for r in rows]
            tts, tvals = [], []
            for t, v in _parsed_text(text, order):
                tts += t
                tvals += v
            tb = np.array(tvals, np.float64).view(np.uint64)
            got, g_oow, g_tiny = model_of(offsets, np.array(tts, np.int64), tb)
            assert np.array_equal(got, want) and (g_oow, g_tiny) == (w_oow, w_tiny), (seed, i, "text")
            n += 1
    assert n >= 4 * len(replays)
