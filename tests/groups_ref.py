"""A plain restatement of the `sum by` group rule of include/gpr.h (gpr_window.groups) for the tests: window max per
row, Prometheus' Neumaier sum of a group's members in slot order (UTIL members / 100 first), and the verdict,
idle_slots and counts the engine must return.  tests/test_groups_emul.py holds it to gph::resolve_sum_by_groups."""
import math

import numpy as np

UTIL = 0x100


def neumaier(xs):
    """Prometheus' kahanSumInc; NaN for no addend"""
    s = c = 0.0
    n = 0
    for x in xs:
        n += 1
        t = s + x
        if math.isinf(t):
            c = 0.0
        elif abs(s) >= abs(x):
            c += (s - t) + x
        else:
            c += (x - t) + s
        s = t
    if not n:
        return math.nan
    return s if math.isinf(s) else s + c


def row_max(x):
    """max_over_time per row: NaN = no sample, NaN only if no sample"""
    with np.errstate(invalid="ignore"):
        return np.fmax.reduce(np.asarray(x, np.float32), axis=-1)


def members(table_p, g):
    return [h for h in range(g, len(table_p)) if table_p[h] & 0xFF == g]


def group_value(m_p, table_p, g):
    xs = []
    for h in members(table_p, g):
        v = float(m_p[h])
        if math.isnan(v):
            continue
        xs.append(v / 100.0 if table_p[h] & UTIL else v)
    return neumaier(xs)


def valid(table):
    P, G = table.shape
    for p in range(P):
        for g in range(G):
            x, l = int(table[p, g]), int(table[p, g]) & 0xFF
            if x & ~(0xFF | UTIL) or l > g or (int(table[p, l]) & 0xFF) != l:
                return False
    return True


def thr_f32(thr):
    t = np.float32(thr)
    return np.nextafter(t, np.float32(np.inf)) if float(t) < float(thr) else t


def decide(util, power=None, thr=0.0, table=None, m=None):
    """util / power float32[P, G, T] (or `m`, the row maxima, instead of util); table uint32[P, G] or None.
    Returns dict: idle bool[P, G] (slots that start an idle element), veto/candidate bool[P], n_series,
    idle_slots uint32[P, ceil(G/32)], candidate_bits / decision_bits / veto_bits, values (leader -> value)."""
    m = row_max(util) if m is None else m
    P, G = m.shape
    with np.errstate(invalid="ignore"):
        idle = m == 0
    values = {}
    if table is not None:
        for p in range(P):
            t = [int(x) for x in table[p]]
            for g in range(G):
                if t[g] & 0xFF != g:
                    idle[p, g] = False
                    continue
                if len(members(t, g)) < 2:
                    continue
                v = group_value(m[p], t, g)
                values[(p, g)] = v
                idle[p, g] = v == 0.0
    veto = np.zeros(P, bool)
    if power is not None and thr and not math.isnan(thr):
        with np.errstate(invalid="ignore"):
            veto = (row_max(power) >= thr_f32(thr)).any(axis=1)
    cand = idle.any(axis=1) & ~veto
    n_series = int(idle[cand].sum())
    MW = (G + 31) // 32
    slots = np.zeros((P, MW * 32), bool)
    slots[:, :G] = idle
    islots = np.packbits(slots.reshape(P, MW, 32), axis=-1, bitorder="little").view("<u4").reshape(P, MW)

    def bits(b):
        pad = np.zeros(((P + 31) // 32) * 32, bool)
        pad[:P] = b
        return np.packbits(pad, bitorder="little").view("<u4").astype(np.uint32)
    return dict(idle=idle, veto=veto, candidate=cand, n_series=n_series, n_candidates=int(cand.sum()),
                idle_slots=islots.astype(np.uint32), candidate_bits=bits(cand), decision_bits=bits(cand),
                veto_bits=bits(veto), values=values)


PALETTE = [0.0, -0.0, 5.0, -5.0, 7.0, np.nan, np.inf, -np.inf, 1e-45, -1e-45, 1e16, -1e16, 1.0, -1.0, 0.5, 100.0]
PALETTE_U8 = [0.0, 5.0, 7.0, np.nan, 1.0, 100.0, 254.0]


def random_table(rng, P, G, share=0.5, max_size=None):
    """pods with groups (about `share` of them) next to pods without; sizes 2..max_size, members anywhere after their
    leader; random UTIL / PROF members"""
    t = np.zeros((P, G), np.uint32)
    for p in range(P):
        lead = np.arange(G)
        if rng.random() < share and G > 1:
            for _ in range(rng.integers(1, 4)):
                leader = int(rng.integers(0, G - 1))
                if lead[leader] != leader:
                    continue
                size = int(rng.integers(2, (max_size or G) + 1))
                free = [h for h in range(leader + 1, G) if lead[h] == h and not (lead == h).sum() > 1]
                rng.shuffle(free)
                for h in free[:size - 1]:
                    lead[h] = leader
        util = rng.random(G) < 0.5
        t[p] = lead.astype(np.uint32) | np.where(util, UTIL, 0).astype(np.uint32)
    assert valid(t)
    return t


def window_for(rng, m, T, u8=False):
    """rows whose max is m[p, g]: the value at a random sample, the rest NaN, zeros or (below m) negatives"""
    P, G = m.shape
    x = np.full((P, G, T), np.nan, np.float32)
    for p in range(P):
        for g in range(G):
            v = m[p, g]
            if np.isnan(v):
                continue
            pos = int(rng.integers(0, T))
            if v > 0 and rng.random() < 0.5:
                x[p, g, :] = 0.0 if not u8 else 0.0
            x[p, g, pos] = v
    return x
