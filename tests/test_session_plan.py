"""The call sequences of tests/test_gpu_session.py, generated without a device (tests/session_ops.py): across the seeds
every operation and every failure occurs, the transitions where a context's state carries bugs occur, and the
references the GPU test uses agree with each other on every window the sequences decide."""
import numpy as np
import pytest

import groups_ref as R
import session_ops as S


@pytest.fixture(scope="module")
def plans():
    return {seed: S.plan(seed) for seed in S.SEEDS}


def _windows(plans):
    for seed, ops in plans.items():
        for i, op in enumerate(ops):
            for w in ([op["win"]] if "win" in op else []) + op.get("wins", []) + op.get("before", []) + \
                    op.get("after", []):
                yield seed, i, op, w


def test_plans_are_reproducible(plans):
    assert S.plan(3) == plans[3]
    assert all(S.N_OPS <= len(ops) <= S.N_OPS + 20 for ops in plans.values())


def test_every_operation_and_failure_occurs(plans):
    kinds = {op["kind"] for ops in plans.values() for op in ops}
    assert kinds == set(S.KINDS), set(S.KINDS) - kinds
    for seed, ops in plans.items():           # every sequence has every failure
        fails = {op["fail"] for op in ops if op["kind"] == "fail"}
        assert fails == set(S.FAILURES), (seed, set(S.FAILURES) - fails)
        no_ring = [i for i, op in enumerate(ops) if op.get("fail") == "resident_no_ring"]
        first_init = min(i for i, op in enumerate(ops) if op["kind"] == "resident_init")
        assert no_ring[0] < first_init, seed


def test_blocking_failures_have_results_pending(plans):
    """a failing blocking call must find earlier results pending, or the test of keeping them proves nothing"""
    for seed, ops in plans.items():
        pending = 0
        for i, op in enumerate(ops):
            k = op["kind"]
            if k == "fail" and op["fail"] in S.BLOCKING_FAILURES:
                assert pending > 0, (seed, i, op["fail"])
            if k in ("async",):
                pending += 1
            elif k == "batch":
                pending += len(op["wins"])
            elif k == "text_planes":
                pending += len(op["decisions"])
            elif k == "fail" and op["fail"] == "batch_fail":
                pending += op["k"]
            elif k in ("decide", "decide_resident", "sync") or (k == "fail" and op["fail"] in (
                    "async_bad_device_table", "slots_full")):
                pending = 0
            assert pending <= S.MAX_PENDING - 1, (seed, i)


def test_transitions_occur(plans):
    seen = set()
    for ops in plans.values():
        seen |= S.transitions(ops)
    assert seen == set(S.TRANSITIONS), set(S.TRANSITIONS) - seen


def test_windows_cover_the_space(plans):
    ws = [w for _, _, _, w in _windows(plans)]
    assert {w["src"] for w in ws} == set(S.SOURCES)
    assert {w["P"] for w in ws} == set(S.PS) and {w["G"] for w in ws} == set(S.GS) and {w["T"] for w in ws} == set(S.TS)
    assert {w["thr"] for w in ws if w["thr"]} == set(S.edges.THRESHOLDS)
    assert {(w["table"] is True, w["gates"], w["out_kind"]) for w in ws} == {
        (t, g, o) for t in (False, True) for g in (False, True) for o in ("host", "dev")}
    for k in S.OUTPUTS:
        assert {w["outs"][k] for w in ws} == {False, True}
    assert max(S.cells(w) for w in ws) <= S.MAX_CELLS
    assert all(w["P"] * w["G"] <= S.MAX_TABLE_SLOTS for w in ws if w["table"] is True)


def test_references_agree_on_every_window(plans, oracle_c, oracle_np):
    """oracle_c, oracle_np and groups_ref on every window the sequences decide (with a valid table, groups_ref alone
    defines the verdict; its table-free answer must still match the oracles)"""
    n = 0
    for seed, i, op, w in _windows(plans):
        d = S.window_data(w)
        util, power, thr = d["util"], d["power"], w["thr"]
        tag = (seed, i, op["kind"], w["src"], w["P"], w["G"], w["T"])
        if S.is_u8(w["src"]):
            import gpu_pruner_b200 as g
            assert np.array_equal(g.from_biased_u8(g.to_biased_u8(util)), util, equal_nan=True), tag
        kw = dict(eligible=d["eligible"], created_ts=d["created_ts"], cutoff_ts=d["cutoff_ts"],
                  power_threshold=thr or 0.0)
        c = oracle_c.decide(util, power, **kw)
        p = oracle_np.decide(util, power, **kw)
        for k in ("decision_bits", "candidate_bits", "n_series", "n_candidates", "n_decisions"):
            assert np.array_equal(c[k], p[k]), (tag, k)
        e = S.expected(util, power, thr, d["eligible"], d["created_ts"], d["cutoff_ts"], None)
        gr = R.decide(util, power, thr or 0.0, None)
        assert np.array_equal(e["veto_bits"], gr["veto_bits"]) and np.array_equal(e["veto_bits"], p["veto_bits"]), tag
        assert np.array_equal(e["candidate_bits"], gr["candidate_bits"]), tag
        assert e["n_series"] == gr["n_series"] and e["n_candidates"] == gr["n_candidates"], tag
        assert S.kat.smax_equal(e["series_max"], R.row_max(util)), tag
        if d["table"] is not None and w["table"] is True:
            t = S.expected(util, power, thr, d["eligible"], d["created_ts"], d["cutoff_ts"], d["table"])
            gt = R.decide(util, power, thr or 0.0, d["table"])
            assert np.array_equal(t["candidate_bits"], gt["candidate_bits"]), tag
            assert np.array_equal(t["idle_slots"], gt["idle_slots"]), tag
            dec = gt["candidate"] & S.gate_mask(w["P"], d["eligible"], d["created_ts"], d["cutoff_ts"])
            assert np.array_equal(t["decision_bits"], oracle_np.pack_bits(dec)), tag
        if w["table"] == "bad":
            assert not R.valid(d["table"]), tag
        n += 1
    assert n > 500


def test_text_slices_and_planes_model(plans):
    """the text the GPU test parses reads back as the model's cells: every sample inside its window, values exact"""
    for seed, ops in plans.items():
        for op in ops:
            if op["kind"] == "text_planes":
                us, ws, u, wc = S.plane_text(op["seed"], op["P"], op["G"], op["T"], op["thr"])
                text, spans = S.text_bytes(us)
                for (b, e, row), (r2, samples) in zip(spans, us):
                    assert row == r2 and text[b - 1:b] == b"[" and text[e:e + 1] == b"]"
                    assert text[b:e].count(b"[") == len(samples)
                if ws is not None:
                    x = np.array([[float(v) for _, v in s] for _, s in ws]).reshape(wc.shape)
                    up = S.edges.f32_up(op["thr"])
                    assert np.array_equal(x >= op["thr"], wc.astype(np.float64) >= up)
