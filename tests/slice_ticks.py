"""Recorded daemon-mode ticks asked as query slices (`--query-slice S`, TEST INFRASTRUCTURE).

write_sliced_ticks() lays out tests/ticks.py's fixtures (whole-range answers under tick-%04d/{full,delta}/) and, for
every range longer than S, the answers to the consecutive queries the binary asks instead: <kind>/slice-%04d/ with
util.json [prof.json] [power.json] and query.json = {"start", "end", "step"}, oldest first, each covering (start, end].
The newest slice ends at the range's end and only the oldest may be shorter (controller.cpp FileSource)."""
import json
import os

import ticks as TK

_write_ticks = TK.write_ticks   # (kept: a scenario may route TK.write_ticks through write_sliced_ticks)


def slice_ranges(start, end, S):
    """(start, end] as the binary asks it with --query-slice S: oldest first"""
    n = -(-(end - start) // S)
    return [(max(start, end - (n - j) * S), end - (n - 1 - j) * S) for j in range(n)]


def write_sliced_ticks(root, store_at, tick_times, window_s, step, S, **kw):
    _write_ticks(root, store_at, tick_times, window_s, step, **kw)
    for k, t in enumerate(tick_times):
        store = store_at(k)
        for kind in ("full", "delta"):
            d = os.path.join(root, "tick-%04d" % k, kind)
            if not os.path.isdir(d):
                continue
            q = json.load(open(os.path.join(d, "query.json")))
            start = q.get("start", t - window_s)
            if t - start <= S:
                continue
            for j, (a, b) in enumerate(slice_ranges(start, t, S)):
                sd = os.path.join(d, "slice-%04d" % j)
                os.makedirs(sd, exist_ok=True)
                for name, metric in (("util.json", "DCGM_FI_DEV_GPU_UTIL"), ("prof.json", "DCGM_FI_PROF_GR_ENGINE_ACTIVE"),
                                     ("power.json", "DCGM_FI_DEV_POWER_USAGE")):
                    if os.path.exists(os.path.join(d, name)):
                        with open(os.path.join(sd, name), "w") as f:
                            f.write(TK.response(store, metric, a, b))
                with open(os.path.join(sd, "query.json"), "w") as f:
                    json.dump({"start": a, "end": b, "step": step}, f)
    return root
