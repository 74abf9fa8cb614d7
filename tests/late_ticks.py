"""Recorded daemon-mode ticks from a server whose samples arrive late (TEST INFRASTRUCTURE, `--late-seconds L`).

A store of samples, each with an arrival time ts + lag.  The server's answer at t_k over (lo, t_k] holds the samples with
ts in range and arrival <= t_k.  write_late_ticks() lays out, per tick:
  full/    that answer over the window (what a cold start or a rebuild asks)
  delta/   that answer over (t_{k-1} - L, t_k]
  expect/  what the resident ring holds after tick k if every tick from 0 on was taken as asked: the samples of the
           window that some tick j <= k asked for (tick 0 the window, tick j > 0 (t_{j-1} - L, t_j]) and that had
           arrived by t_j.  With no lag above L that is full/; with more, it lacks exactly the samples that came too late.
and with S the query slices of full/ and delta/ (tests/slice_ticks.py's layout).  late_cells() is the model of what the
binary's late-cell count reports per delta tick: the (series, bucket) cells of the re-asked buckets whose maximum
changed between the rings of tick k-1 and tick k.  One series feeds one row (no PROF series here)."""
import json
import math
import os

import numpy as np

import slice_ticks as ST
import ticks as TK

FILES = (("util.json", "DCGM_FI_DEV_GPU_UTIL"), ("power.json", "DCGM_FI_DEV_POWER_USAGE"))


class LateStore:
    """[(metric, labels, [(ts, value, lag)])]"""

    def __init__(self, series):
        self.series = series

    def visible(self, now):
        """the store as tests/ticks.py reads it: what the server holds at `now`"""
        return [(m, lab, [(t, v) for t, v, lag in s if t + lag <= now]) for m, lab, s in self.series]

    def held(self, k, tick_times, window_s, L, first_full=0):
        """the store as the resident ring holds it after tick k (ticks first_full..k taken as asked, first_full a full
        fetch)"""
        def asked(ts, lag):
            for j in range(first_full, k + 1):
                t = tick_times[j]
                lo = t - window_s if j == first_full else tick_times[j - 1] - L
                if lo < ts <= t and ts + lag <= t:
                    return True
            return False
        t = tick_times[k]
        return [(m, lab, [(ts, v) for ts, v, lag in s if t - window_s < ts <= t and asked(ts, lag)])
                for m, lab, s in self.series]


def _write(d, store, lo, hi, step, start=None, power=False):
    os.makedirs(d, exist_ok=True)
    for name, metric in FILES[:2 if power else 1]:
        with open(os.path.join(d, name), "w") as f:
            f.write(TK.response(store, metric, lo, hi))
    q = {"end": hi, "step": step}
    if start is not None:
        q["start"] = start
    with open(os.path.join(d, "query.json"), "w") as f:
        json.dump(q, f)


def write_late_ticks(root, late, tick_times, window_s, step, L, S=0, prev=None, power=False):
    """prev: the tick before the first one (a run that resumes from a snapshot taken then; expect/ assumes tick 0 of
    tick_times was a full fetch, so it is meant for runs that start cold)"""
    for k, t in enumerate(tick_times):
        store = late.visible(t)
        base = os.path.join(root, "tick-%04d" % k)
        ranges = [("full", t - window_s)] + ([("delta", prev - L)] if prev is not None else [])
        for kind, lo in ranges:
            d = os.path.join(base, kind)
            _write(d, store, lo, t, step, lo if kind == "delta" else None, power)
            if S and t - lo > S:
                for j, (a, b) in enumerate(ST.slice_ranges(lo, t, S)):
                    sd = os.path.join(d, "slice-%04d" % j)
                    _write(sd, store, a, b, step, power=power)
                    with open(os.path.join(sd, "query.json"), "w") as f:
                        json.dump({"start": a, "end": b, "step": step}, f)
        _write(os.path.join(base, "expect"), late.held(k, tick_times, window_s, L), t - window_s, t, step, power=power)
        prev = t
    return root


def _f32(v):
    return np.float32(float(v))


def _bucket_maxima(series, t, step, backs):
    """per back in `backs`: the max of the samples in bucket `back` (0 = newest) of the grid ending at t; None = none"""
    out = []
    for back in backs:
        hi, lo = t - back * step, t - (back + 1) * step
        vals = [_f32(v) for ts, v in series if lo < ts <= hi]
        out.append(max(vals) if vals else None)
    return out


def late_cells_planes(late, tick_times, window_s, step, L):
    """per delta tick k >= 1: (util cells, power cells) of the re-asked buckets whose maximum tick k changed"""
    T = window_s // step
    out = []
    for k in range(1, len(tick_times)):
        t, prev = tick_times[k], tick_times[k - 1]
        n_new, n_re = (t - prev) // step, math.ceil(L / step)
        backs = range(n_new, min(T, n_new + n_re))
        now, before = late.held(k, tick_times, window_s, L), late.held(k - 1, tick_times, window_s, L)
        n = {"DCGM_FI_DEV_GPU_UTIL": 0, "DCGM_FI_DEV_POWER_USAGE": 0}
        for (m, _, s_now), (_, _, s_before) in zip(now, before):
            a = _bucket_maxima(s_now, t, step, backs)
            b = _bucket_maxima(s_before, t, step, backs)
            n[m] += sum(x != y for x, y in zip(a, b))
        out.append((n["DCGM_FI_DEV_GPU_UTIL"], n["DCGM_FI_DEV_POWER_USAGE"]))
    return out


def late_cells(late, tick_times, window_s, step, L):
    """per delta tick: the util cells of the re-asked buckets that the late samples changed"""
    return [u for u, _ in late_cells_planes(late, tick_times, window_s, step, L)]
