"""The launch path of the C ABI (gpu-pruner_b200/csrc/gpr_api.cu).  Every kernel on a context's stream goes through one
helper, launch(), which counts it (gpr_launch_count) and is the only place programmatic dependent launch is asked for.
Every entry point that enqueues work or waits for the stream starts with enter(), which clears last_was_reduce: a
decision's reduce may start early only behind one of our folds.  Read from the source like
tests/test_context_ownership.py, so a new entry point or launch site that skips either fails here on any machine; and on
the H100, the exact launch count of every call of one scripted sequence."""
import re

import numpy as np
import pytest

from test_context_ownership import _body, _code, _definition

# entry points that only read the context: they must not break a PDL chain, so they do not call enter()
QUERIES = {"gpr_sync", "gpr_launch_count", "gpr_step_stamps", "gpr_phase_stamps", "gpr_get_device_info",
           "gpr_resident_planes", "gpr_resident_head", "gpr_text_planes", "gpr_p2p_debug", "gpr_last_error",
           "gpr_version"}
# the decisions (decide_impl keeps last_was_reduce itself), the context's creation and destruction, and two calls that
# touch no stream
OWN = {"gpr_decide", "gpr_decide_async", "gpr_decide_batch_async", "gpr_decide_resident", "gpr_create", "gpr_destroy",
       "gpr_comm_unique_id", "gpr_host_free"}


def _where(pattern):
    """the definitions that hold a match of `pattern`, one entry per match"""
    lines = _code().split("\n")
    return [_definition(lines, at) for at, line in enumerate(lines) for _ in re.finditer(pattern, line)]


def _entry_points():
    """name -> body of every gpr_* function defined with C linkage"""
    code = _code()
    heads = re.finditer(r"^(?:extern \"\" GPR_API )?(?:int|void|const char\*) (gpr_\w+)\(", code, re.M)
    return {m.group(1): _body(code, m.group(0)) for m in heads}


def test_only_the_scan_producer_launches_with_chevrons():
    assert _where(r"<<<") == ["scan_producer", "scan_producer"]


def test_one_helper_launches_and_counts():
    assert _where(r"\bcudaLaunchKernelEx\s*\(") == ["launch"]
    counted = _where(r"\bctx->launches\s*(?:\+\+|[-+]=|=(?!=))|(?:\+\+|--)\s*ctx->launches\b")
    assert sorted(set(counted)) == ["gpr_text_scan_begin", "launch"], counted


def test_only_enter_and_the_decision_clear_the_pdl_chain():
    assert set(_where(r"(?:->|\.)last_was_reduce\s*=(?!=)")) == {"enter", "decide_impl"}


def test_every_entry_point_that_touches_the_stream_enters_first():
    entries = _entry_points()
    assert QUERIES | OWN <= set(entries) and {"gpr_samples_scatter", "gpr_text_parse", "gpr_append"} <= set(entries)
    for name, body in entries.items():
        called = re.search(r"\benter\(", body)
        if name in QUERIES or name in OWN:
            assert not called, name
            continue
        assert called, name
        for first_use in (r"ctx->stream\b", r"\blaunch\(", r"\bgpr_text_scan_begin\("):
            m = re.search(first_use, body)
            assert not m or called.start() < m.start(), (name, first_use)


# ---- on the H100 --------------------------------------------------------------------------------------------------
T_END = 1_700_000_000

# launches of each call below.  k_synth_fill and k_synth_eligible count like every other kernel; the rest are the
# kernels each call has always launched (with a power plane and a block index on the ring).
EXPECTED = {
    "synth_fill": 1, "synth_eligible": 1, "resident_init": 0,
    "append (util and power)": 2,        # k_append per plane
    "append (util only)": 2,             # k_append, and k_open for the power plane
    "resident_advance": 2,               # k_open per plane (the index's blocks are recomputed)
    "resident_reindex": 2,
    "resident_remap (host map)": 4,      # k_remap_rows for util, power and both index planes
    "resident_remap (device map)": 6,    # and k_remap_check's two passes
    "text_scan": 2,                      # one chunk: k_text_scan_chunk and k_publish_marks
    "text_parse": 1,
    "samples_scatter (host)": 1,         # one piece
    "samples_scatter (device)": 2,       # k_samples_check, k_samples_scatter
    "resident_export": 5,                # the sizes (k_export_size, k_export_scan), then all three
    "chunks_scatter (host)": 2,          # k_chunks_check, k_chunks_scatter on the same staged piece
    "chunks_scatter (device)": 3,        # k_samples_check, k_chunks_check, k_chunks_scatter
    "decide (device window)": 2,         # the reduce, the fold
    "decide (host window)": 2,           # one staged chunk of pods: the reduce, the fold
}


@pytest.mark.gpu
def test_launch_count_of_every_entry_point():
    torch = pytest.importorskip("torch")
    import gpu_pruner_b200 as g
    if not torch.cuda.is_available():
        pytest.fail("-m gpu tests need a CUDA device; the engine has no CPU fallback")
    P, G, T = 8, 2, 128
    rows = P * G
    rng = np.random.default_rng(7)
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()  # noqa: E731
    with g.IdleEngine(device=0, max_pods=P, max_gpus=G, max_samples=T, power_plane=True) as eng:
        got = {}

        def count(what, call):
            n0 = eng.launch_count()
            out = call()
            got[what] = eng.launch_count() - n0
            return out

        u = torch.empty((P, G, T), dtype=torch.float32, device="cuda")
        elig = torch.empty(P, dtype=torch.uint8, device="cuda")
        count("synth_fill", lambda: eng.synth_fill(1, 0, u, 0, P, G, T))
        count("synth_eligible", lambda: eng.synth_eligible(1, elig, 0, P))
        count("resident_init", lambda: eng.resident_init(P, G, T, power_plane=True, block_index=True))
        cols = rng.integers(0, 100, (rows, 5)).astype(np.float32)
        count("append (util and power)", lambda: eng.append(cols, cols * 2))
        count("append (util only)", lambda: eng.append(cols))
        count("resident_advance", lambda: eng.resident_advance(3))
        count("resident_reindex", lambda: eng.resident_reindex())
        grow = np.concatenate([np.arange(rows), np.full(G, g.ffi.GPR_ROW_NONE)]).astype(np.uint32)
        count("resident_remap (host map)", lambda: eng.resident_remap(P + 1, G, grow))
        shrink = torch.arange(rows, dtype=torch.int32, device="cuda")
        count("resident_remap (device map)", lambda: eng.resident_remap(P, G, shrink))

        series = ['{"metric":{"gpu":"%d"},"values":[[%d,"%d"],[%d,"%d"]]}' % (r, T_END - 1, r, T_END, r + 1)
                  for r in range(rows)]
        text = ('{"status":"success","data":{"resultType":"matrix","result":[' + ",".join(series) + "]}}").encode()
        opens, closes = count("text_scan", lambda: eng.text_scan(text))
        spans = np.zeros(len(opens), eng.SPAN_DTYPE)
        spans["begin"] = opens + 12
        spans["end"] = closes[np.searchsorted(closes, opens + 12)] + 2
        spans["row"] = np.arange(len(opens))
        out = count("text_parse", lambda: eng.text_parse(spans, T_END, 1, T, rows))
        assert int(out["n_in"].sum()) == 2 * rows

        offsets = np.arange(rows + 1, dtype=np.uint64) * 2
        r_ids = np.arange(rows, dtype=np.uint32)
        ts = np.tile(np.array([T_END - 1, T_END], np.int64) * 1000, rows)
        vals = rng.integers(0, 100, 2 * rows).astype(np.float64)
        st = count("samples_scatter (host)", lambda: eng.samples_scatter(offsets, r_ids, ts, vals, T_END, 1, T, rows))
        assert st["n_in"] == 2 * rows
        d = [dev(offsets.view(np.int64)), dev(r_ids.view(np.int32)), dev(ts), dev(vals)]
        st = count("samples_scatter (device)", lambda: eng.samples_scatter(*d, T_END, 1, T, rows, n_series=rows,
                                                                           mem_kind=g.ffi.GPR_MEM_DEVICE))
        assert st["n_in"] == 2 * rows

        x = count("resident_export", lambda: eng.resident_export(T_END, 1))
        assert x["n_samples"] > 0
        k = x["grid"]
        args = (k["t_end"], k["step"], k["T"], rows)
        kw = dict(window_seconds=k["window_seconds"], resident=True)
        arrays = (x["series_chunks"], x["rows"], x["chunk_bytes"], x["data"])
        st = count("chunks_scatter (host)", lambda: eng.chunks_scatter(*arrays, *args, **kw))
        assert st["n_in"] == x["n_samples"]
        d = [dev(a.view(np.int64) if a.dtype == np.uint64 else a.view(np.int32) if a.dtype == np.uint32 else a)
             for a in arrays]
        st = count("chunks_scatter (device)", lambda: eng.chunks_scatter(*d, *args, **kw, n_series=len(x["rows"]),
                                                                         mem_kind=g.ffi.GPR_MEM_DEVICE))
        assert st["n_in"] == x["n_samples"]

        dbits = torch.zeros((P + 31) // 32, dtype=torch.int32, device="cuda")
        count("decide (device window)", lambda: eng.decide_ptr(u, P, G, T, dbits, eligible=elig))
        count("decide (host window)", lambda: eng.decide(u.cpu().numpy()))
        assert got == EXPECTED
