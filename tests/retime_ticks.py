"""Recorded daemon-mode ticks whose query step or window changes between ticks (TEST INFRASTRUCTURE, `--retime-ring`).

write_retime_ticks() lays out, per tick k at time t_k with step steps[k] and window durations[k] minutes:
  full/    the answer over (t_k - window, t_k]
  delta/   the answer over (t_{k-1} - L, t_k]  (L = the --late-seconds the run re-asks)
each with util.json [prof.json] [power.json] and query.json = {"end", "step"[, "start"]}; with S > 0, every range longer
than S also as the consecutive queries the binary asks instead (tests/slice_ticks.py's layout); and tick-%04d/duration
(minutes) at every tick whose window differs from the previous tick's.  The responses hold raw samples, so the step only
changes how the binary buckets them."""
import json
import os

import slice_ticks as ST
import ticks as TK

FILES = (("util.json", "DCGM_FI_DEV_GPU_UTIL"), ("prof.json", "DCGM_FI_PROF_GR_ENGINE_ACTIVE"),
         ("power.json", "DCGM_FI_DEV_POWER_USAGE"))


def _answer(d, store, lo, hi, step, start, power, S):
    os.makedirs(d, exist_ok=True)
    metrics = {s[0] for s in store}
    names = [(n, m) for n, m in FILES if m in metrics and (power or m != "DCGM_FI_DEV_POWER_USAGE")]
    for name, metric in names:
        with open(os.path.join(d, name), "w") as f:
            f.write(TK.response(store, metric, lo, hi))
    q = {"end": hi, "step": step}
    if start is not None:
        q["start"] = start
    with open(os.path.join(d, "query.json"), "w") as f:
        json.dump(q, f)
    if S and hi - lo > S:
        for j, (a, b) in enumerate(ST.slice_ranges(lo, hi, S)):
            sd = os.path.join(d, "slice-%04d" % j)
            os.makedirs(sd, exist_ok=True)
            for name, metric in names:
                with open(os.path.join(sd, name), "w") as f:
                    f.write(TK.response(store, metric, a, b))
            with open(os.path.join(sd, "query.json"), "w") as f:
                json.dump({"start": a, "end": b, "step": step}, f)


def write_retime_ticks(root, store, times, steps, durations, L=0, S=0, power=False, skip_delta=()):
    """steps[k], durations[k] (minutes): the query step and --duration at tick k"""
    for k, t in enumerate(times):
        base = os.path.join(root, "tick-%04d" % k)
        window = durations[k] * 60
        _answer(os.path.join(base, "full"), store, t - window, t, steps[k], None, power, S)
        if k and k not in skip_delta:
            lo = times[k - 1] - L
            _answer(os.path.join(base, "delta"), store, lo, t, steps[k], lo, power, S)
        if k and durations[k] != durations[k - 1]:
            with open(os.path.join(base, "duration"), "w") as f:
                f.write(str(durations[k]))
    return root


def retime_line(T, step, N, step2, N2):
    """the start of the binary's log line for a retime from (T buckets, step, N s) to (step2, N2 s)"""
    n_keep = T if N2 == N else N2 // step
    k = step2 // step
    return "Resident window retimed on the GPU: %d -> %d (step %d -> %d s, window %d -> %d s, retime " % (
        T, -(-n_keep // k), step, step2, N, N2)
