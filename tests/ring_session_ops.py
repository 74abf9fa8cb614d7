"""Seeded call sequences that reshape, merge into, export and restore the resident ring of one context, and the plain
model they are checked against.  TEST INFRASTRUCTURE, shared by tests/test_gpu_session_ring.py (the sequences on an
H100) and tests/test_session_ring_plan.py (the generator and the references on the CPU).

`plan_ring(seed)` draws the operations; `Model` replays them without a device and says, after every operation, what
the ring holds (both planes, bit for bit), where its head is, whether its block index is current, how many results are
pending, and what every call must return.  The references are the suite's own: tests/ring_scripts.py (the ring and its
pools of quiet and loud cells), tests/test_samples_emul.py's `model` (where a merged sample lands and what it leaves),
tests/chunks_ref.py (the XOR encoder), tests/export_ref.py (the export, byte for byte, and the restore), and, for the
verdicts, the C oracle and tests/groups_ref.py through tests/session_ops.py's `expected`.

Operations (dicts with a "kind"):
  init            gpr_resident_init of a ring spec (P, G, T, power plane, block index)
  append/advance  n_new in {1, T - 1, T, T + 5}; an append from host or device columns, power columns or NULL
  merge           advance n_new, then one slice into the util or the power plane as text, decoded samples (pageable,
                  pinned or device memory) or XOR chunks (host or device), sometimes with grid.n_rows < P * G
  plant           the planes rewritten through gpr_resident_planes (then reindexed) so that the only loud cell of a
                  block, or every sample of a row, sits where the next advance, merge or remap changes the ring
  live_rows       gpr_resident_live_rows into host or device memory
  remap           gpr_resident_remap by the gpr.h recipe or by a random map with GPR_ROW_NONE rows, host or device map
  export          Engine.resident_export of one plane at max_per_chunk in {1, 7, 120, 65535}
  restore         both planes exported and scattered into a second context, maybe of another [P][G], then reindexed
  ring_async      1 to 4 gpr_decide_async on the pointers of gpr_resident_planes, left pending
  async           one gpr_decide_async of a small device window (results pending before any ring exists)
  sync / reindex / decide_resident (whole or early, with or without a `sum by` table)
  fail            a failing call (FAILURES), each with the ABI's code, always with results pending
"""
from __future__ import annotations

import numpy as np

import chunks_ref as CR
import edges
import export_ref as X
import ring_scripts as RS
import session_ops as S
from test_live_rows_emul import live_model
from test_remap_emul import NONE, first_bad, remap_model
from test_samples_emul import SPECIAL, model as samples_model

SEEDS = list(range(6))
N_OPS = 60
PS, GS, TS = [1, 3, 33, 200], [1, 4, 5], [4, 63, 64, 65, 181, 1800]
MAX_RING_CELLS = 60_000      # P * G * T of a ring (the export reference is a plain Python encoder)
STEP = S.STEP
T_END = S.T_END
MAX_PENDING = S.MAX_PENDING
E_INVALID, E_CAPACITY, E_STATE = S.E_INVALID, S.E_CAPACITY, S.E_STATE
MERGE_SOURCES = ("text", "samples_pageable", "samples_pinned", "samples_dev", "chunks_host", "chunks_dev")
EXPORT_M = (1, 7, 120, 65535)
CHUNK_M = (1, 7, 120)

FAILURES = {
    "remap_range_host": E_INVALID,    # a host map entry >= the old rows
    "remap_range_dev": E_INVALID,     # the same, a device map
    "remap_twice_host": E_INVALID,    # an old row named twice, host map
    "remap_twice_dev": E_INVALID,     # the same, a device map
    "remap_no_ring": E_STATE,         # gpr_resident_remap before any ring
    "live_bad_kind": E_INVALID,       # gpr_resident_live_rows with mem_kind 7
    "live_no_ring": E_STATE,          # gpr_resident_live_rows before any ring
    "export_capacity": E_CAPACITY,    # one capacity one short: the true counts, no array written
    "export_no_power": E_STATE,       # plane 1 of a ring without a power plane
    "export_bad_T": E_INVALID,        # grid.n_samples != T
    "merge_bad_row": E_INVALID,       # a series row >= grid.n_rows (samples or chunks)
    "merge_truncated": E_INVALID,     # a chunk one byte short: named as the first bad chunk
    "merge_no_power": E_STATE,        # the power plane of a ring without one
    "merge_rows_over": E_INVALID,     # grid.n_rows > P * G right after a shrinking remap
    "decide_stale": E_STATE,          # gpr_decide_resident after a merge, before gpr_resident_reindex
}
NO_RING = ("remap_no_ring", "live_no_ring")
KINDS = ("async", "init", "append", "advance", "merge", "plant", "live_rows", "remap", "export", "restore",
         "ring_async", "sync", "reindex", "decide_resident", "fail")
TRANSITIONS = (
    "ring rewritten while a ring_async result is pending",
    "a stale index remapped, then reindexed",
    "live_rows on a current index right after a remap",
    "live_rows on a stale index",
    "live_rows on a stale index that merges have overtaken",
    "live_rows on a current index after an advance emptied rows",
    "live_rows with a row alive only in the power plane",
    "export right after a remap with the head not 0",
    "restore into another shape",
    "merge right after a shrinking remap",
    "export of a ring with empty rows",
    "chunks straddling the window's lower edge",
)
WRITES_RING = ("init", "append", "advance", "merge", "plant", "remap")


# ---- slices ------------------------------------------------------------------------------------------------------
def _slice_values(rng, n, plane, chunks):
    """f64 bit patterns: the ring pools' cells (quiet and loud), SPECIAL, integers, Prometheus' staleness marker"""
    quiet, loud = RS.POOLS[(plane, False)], RS.POOLS[(plane, True)]
    pool = np.concatenate([quiet.view(np.float32).astype(np.float64), loud.view(np.float32).astype(np.float64),
                           SPECIAL]).view(np.uint64)
    bits = pool[rng.integers(0, pool.size, n)]
    plain = rng.random(n) < 0.5
    bits[plain] = rng.choice(np.array([0.0, 0.0, 0.0, 1.0, 3.0, 55.5, 160.0]), int(plain.sum())).view(np.uint64)
    if chunks:
        bits[rng.random(n) < 0.05] = CR.STALE_NAN_BITS
    return bits


def merge_slice(op, T, t_end):
    """the slice of a merge op: CSR (offsets u64, rows u32, ts ms i64, value bits u64); samples of a series in time
    order, mostly inside the window (t_end - window, t_end], some before it (a chunk straddles the lower edge), a few
    after t_end, at the window edges and several in one bucket"""
    rng = np.random.default_rng(op["seed"])
    window = merge_window(op, T)
    n_rows = op["n_rows"]
    n_series = int(rng.integers(1, min(40, 2 * n_rows) + 1))
    rows = rng.integers(0, n_rows, n_series).astype(np.uint32)
    if op.get("revive"):
        k = min(len(op["revive"]), n_series)
        rows[:k] = op["revive"][:k]
    lengths = rng.integers(1, min(3 * window // STEP + 3, 120) + 1, n_series)
    ts, bits = [], []
    t_hi = t_end * 1000
    t_lo = (t_end - window) * 1000
    for s in range(n_series):
        n = int(lengths[s])
        t = t_hi - rng.integers(0, window * 1000, n)
        edge = rng.random(n)
        t[edge < 0.05] = t_lo + 1
        t[(edge >= 0.05) & (edge < 0.1)] = t_hi
        t[(edge >= 0.1) & (edge < 0.15)] = t_lo                       # just outside: the window is left-open
        old = (edge >= 0.15) & (edge < 0.3)
        t[old] = t_lo - rng.integers(1, 3 * STEP * 1000, int(old.sum()))
        t[(edge >= 0.3) & (edge < 0.32)] = t_hi + 1
        ts.append(np.sort(t))
        bits.append(_slice_values(rng, n, op["plane"], op["src"].startswith("chunks")))
    offsets = np.concatenate([[0], np.cumsum(lengths)]).astype(np.uint64)
    return offsets, rows, np.concatenate(ts).astype(np.int64), np.concatenate(bits).astype(np.uint64)


def merge_window(op, T):
    return min(op["n_new"], T) * STEP


def slice_chunks(op, offsets, ts, bits):
    """the slice as XOR chunks of at most op["M"] samples: (series_chunks, chunk_bytes, data)"""
    series = []
    for s in range(len(offsets) - 1):
        a, b = int(offsets[s]), int(offsets[s + 1])
        series.append(CR.split(ts[a:b].tolist(), [int(x) for x in bits[a:b]], op["M"]))
    return CR.batch(series)


def truncate_chunk(sc, cb, data, c):
    """chunk c one byte short (every later chunk moved up by a byte): its decode runs past its bytes"""
    lo, hi = int(cb[c]), int(cb[c + 1])
    data = np.concatenate([data[:hi - 1], data[hi:]]).astype(np.uint8)
    cb = cb.copy()
    cb[c + 1:] -= np.uint64(1)
    assert lo < hi - 1
    return sc, cb, data


def samples_batch(op, offsets, rows, ts, bits, plane, T, t_end, col_end):
    """the batch tests/test_samples_emul.py's model takes, on the given plane"""
    window = merge_window(op, T)
    return dict(offsets=offsets, rows=rows, ts=ts, values=bits.view(np.float64), T=T, t_end=t_end * 1000,
                t_lo=(t_end - window) * 1000, step=STEP * 1000, col_end=col_end,
                thr=op["thr"] if op["plane"] == 1 else None, plane=plane)


def text_of(offsets, rows, ts, bits):
    """the slice as a matrix response (tests/test_gpu_samples.py's rendering): (bytes, row of each span)"""
    from test_gpu_samples import _render
    return _render(offsets, rows, ts, bits.view(np.float64))


# ---- planted cells -----------------------------------------------------------------------------------------------
def plant_cells(op, ring):
    """new planes for a ring: per row one of
      0  quiet cells, and in most blocks the opened positions touch one loud cell at one of them;
      1  samples only at the opened positions (the row is empty once they are opened);
      2  util empty, power quiet with loud cells away from the opened positions (alive only in the power plane);
      3  empty in both planes (a merge revives it)
    The opened positions are those of the next advance or merge (op["open"]), or a random set before a remap."""
    rng = np.random.default_rng(op["seed"])
    T, rows = ring.T, ring.rows
    if op["open"]:
        _, pos = ring.span(op["open"])
    else:
        pos = np.unique(rng.integers(0, T, max(1, T // 8)))
    away = np.setdiff1d(np.arange(T), pos)
    cat = rng.choice(4, rows, p=[0.5, 0.2, 0.15, 0.15])
    planes = []
    for pl in range(len(ring.planes)):
        quiet, loud = RS.POOLS[(pl, False)], RS.POOLS[(pl, True)]
        c = quiet[rng.integers(0, quiet.size, (rows, T))]
        for r in range(rows):
            k = cat[r]
            if k == 3 or (k == 2 and pl == 0) or (k == 2 and len(ring.planes) == 1):
                c[r] = RS.NO_SAMPLE
                continue
            if k == 1:
                keep = c[r, pos].copy()
                c[r] = RS.NO_SAMPLE
                c[r, pos] = keep
            where = pos if k != 2 else away
            if where.size == 0:
                c[r] = RS.NO_SAMPLE
                continue
            for b in np.unique(where // RS.BLOCK):
                if rng.random() < 0.8:
                    c[r, rng.choice(where[where // RS.BLOCK == b])] = loud[rng.integers(0, loud.size)]
        planes.append(c)
    return planes


def append_columns(op, rows):
    """append columns [rows, n_new] as f32 bits: the ring pools, mostly quiet (util, power or None)"""
    rng = np.random.default_rng(op["seed"])
    n = op["n_new"]
    u = RS._mixed(rng, 0, rows, n)
    p = RS._mixed(rng, 1, rows, n) if op["power_cols"] else None
    return u, p


# ---- the model ---------------------------------------------------------------------------------------------------
class Model:
    """the context as the plans see it: the ring (tests/ring_scripts.py's Ring), its index state, the pending results
    (all, and those enqueued on the ring's planes), the time of the newest bucket, and the transitions reached"""

    def __init__(self):
        self.ring = None
        self.stale = False
        self.t_end = T_END
        self.pending = 0
        self.ring_pending = 0
        self.seen = set()
        self.fails_pending = set()
        self.prev = None              # the previous op, for the transitions that need it
        self.stale_remapped = False
        self.idx_live = None          # the rows a stale index would call live (None: unknown)
        self.emptied = False          # an advance on a current index has emptied rows since the last live_rows

    # what every op leaves behind; returns what the op must give
    def apply(self, op):
        k = op["kind"]
        m = self.ring
        out = {}
        if k in ("append", "advance", "merge", "remap") and self.ring_pending:
            self.seen.add("ring rewritten while a ring_async result is pending")
        if k == "async":
            self.pending += 1
        elif k == "ring_async":
            out["window"] = (m.window(0).copy(), m.window(1).copy() if len(m.planes) > 1 else None)
            self.pending += len(op["calls"])
            self.ring_pending += len(op["calls"])
        elif k in ("sync", "decide_resident"):
            if k == "decide_resident":
                assert not (m.index and self.stale)
            self.pending = self.ring_pending = 0
        elif k == "init":
            r = op["ring"]
            self.ring = RS.Ring(r["P"], r["G"], r["T"], (1 if r["power"] else 0) | (2 if r["index"] else 0))
            self.stale = self.emptied = False
            self.idx_live = None
        elif k == "append":
            before = live_model(m.planes)
            u, p = append_columns(op, m.rows)
            m.append(op["n_new"], u, p)
            self._after_write(before)
        elif k == "advance":
            before = live_model(m.planes)
            m.advance(op["n_new"])
            self._after_write(before)
        elif k == "merge":
            out.update(self._merge(op))
        elif k == "plant":
            m.planes = plant_cells(op, m)
            self.emptied = False
            if m.index:
                self.stale = False
            self.idx_live = live_model(m.planes)
        elif k == "reindex":
            if m.index and self.stale_remapped and self.stale:
                self.seen.add("a stale index remapped, then reindexed")
            self.stale = False
            self.stale_remapped = False
            self.emptied = False
            self.idx_live = live_model(m.planes)
        elif k == "live_rows":
            live = live_model(m.planes)
            out["live"] = live
            if m.index and not self.stale:
                if self.prev is not None and self.prev["kind"] == "remap":
                    self.seen.add("live_rows on a current index right after a remap")
                if self.emptied:
                    self.seen.add("live_rows on a current index after an advance emptied rows")
            if m.index and self.stale:
                self.seen.add("live_rows on a stale index")
                if self.idx_live is not None and not np.array_equal(self.idx_live, live):
                    self.seen.add("live_rows on a stale index that merges have overtaken")
            if len(m.planes) > 1 and (live_model(m.planes[1:]) & ~live_model(m.planes[:1])).any():
                self.seen.add("live_rows with a row alive only in the power plane")
            self.emptied = False
        elif k == "remap":
            src = np.asarray(op["src"], np.uint64).astype(np.uint32)
            n = RS.Ring(op["P"], op["G"], m.T, m.flags)
            n.planes, n.head = remap_model(m.planes, src), m.head
            if op["P"] * op["G"] < m.rows:
                op_shrink = True
            else:
                op_shrink = False
            if self.idx_live is not None:
                self.idx_live = remap_model([self.idx_live.astype(np.uint32)[:, None]], src)[0][:, 0] == 1
            if m.index and self.stale:
                self.stale_remapped = True
            self.ring = n
            out["shrink"] = op_shrink
        elif k == "export":
            if self.prev is not None and self.prev["kind"] == "remap" and m.head != 0:
                self.seen.add("export right after a remap with the head not 0")
            if not live_model(m.planes[op["plane"]:op["plane"] + 1]).all():
                self.seen.add("export of a ring with empty rows")
            out["export"] = X.export(m.planes[op["plane"]], m.head, self.t_end, STEP, op["M"])
        elif k == "restore":
            out.update(self._restore(op))
        elif k == "fail":
            out.update(self._fail(op))
        self.prev = op
        return out

    def _after_write(self, live_before):
        m = self.ring
        if m.index and not self.stale:
            self.idx_live = live_model(m.planes)
            if (live_before & ~self.idx_live).any():
                self.emptied = True
        else:
            self.idx_live = None          # an append or advance rewrote blocks of a stale index

    def _merge(self, op, advance=True):
        m = self.ring
        if advance:
            before = live_model(m.planes)
            m.advance(op["n_new"])
            self._after_write(before)
            self.t_end += op["n_new"] * STEP
        offsets, rows, ts, bits = merge_slice(op, m.T, self.t_end)
        if self.prev is not None and self.prev["kind"] == "remap" and self.prev.get("shrink"):
            self.seen.add("merge right after a shrinking remap")
        b = samples_batch(op, offsets, rows, ts, bits, m.planes[op["plane"]], m.T, self.t_end, (m.head + m.T - 1) % m.T)
        plane, n_oow, n_tiny = samples_model(b)
        if op["src"].startswith("chunks") and (ts <= b["t_lo"]).any():
            self.seen.add("chunks straddling the window's lower edge")
        m.planes[op["plane"]] = plane
        if m.index:
            self.stale = True
            self.emptied = False
        return {"stats": (len(ts), n_oow, n_tiny)}

    def _restore(self, op):
        m = self.ring
        if (op["P"], op["G"]) != (m.P, m.G):
            self.seen.add("restore into another shape")
        out = {"exports": [X.export(p, m.head, self.t_end, STEP, 120) for p in m.planes]}
        twin = RS.Ring(op["P"], op["G"], m.T, m.flags & 1 | (2 if op["index"] else 0))
        new_row = twin_rows(op, m)
        for pl, p in enumerate(m.planes):
            canon = X.canonical(X.unroll(p, m.head))
            keep = new_row != NONE
            twin.planes[pl][new_row[keep].astype(np.int64)] = canon[keep]
        out["twin"] = twin
        return out

    def _fail(self, op):
        f = op["fail"]
        m = self.ring
        if self.pending:
            self.fails_pending.add(f)
        out = {}
        if f == "merge_bad_row" or f == "merge_truncated" or f == "merge_no_power":
            before = live_model(m.planes)
            m.advance(op["n_new"])
            self._after_write(before)
            self.t_end += op["n_new"] * STEP
        if f == "export_capacity":
            out["export"] = X.export(m.planes[op["plane"]], m.head, self.t_end, STEP, op["M"])
        if f in ("remap_range_host", "remap_range_dev", "remap_twice_host", "remap_twice_dev"):
            out["first_bad"] = first_bad(np.asarray(op["src"], np.uint64).astype(np.uint32), m.rows)
        if f == "merge_truncated":
            offsets, rows, ts, bits = merge_slice(op, m.T, self.t_end)
            sc, cb, data = slice_chunks(op, offsets, ts, bits)
            sc, cb, data = truncate_chunk(sc, cb, data, op["chunk"])
            assert CR.decode(bytes(data[int(cb[op["chunk"]]):int(cb[op["chunk"] + 1])]))[2] == "overrun"
            out["batch"] = (sc, rows, cb, data)
        return out


def twin_rows(op, m):
    """old row -> twin row (NONE: not restored) through the restore op's pod table"""
    table = np.asarray(op["pods"], np.int64)          # old pod -> twin pod, -1 = dropped
    new_row = np.full(m.rows, NONE, np.uint32)
    for p in range(m.P):
        if table[p] < 0:
            continue
        for g in range(min(m.G, op["G"])):
            new_row[p * m.G + g] = table[p] * op["G"] + g
    return new_row


# ---- the generator -----------------------------------------------------------------------------------------------
def _ring_spec(rng, power=None, index=None):
    while True:
        P, G, T = int(rng.choice(PS)), int(rng.choice(GS)), int(rng.choice(TS))
        if P * G * T <= MAX_RING_CELLS:
            break
    return dict(P=P, G=G, T=T, power=bool(rng.random() < 0.65) if power is None else power,
                index=bool(rng.random() < 0.65) if index is None else index)


def _n_new(rng, T):
    return int(rng.choice([1, max(1, T - 1), T, T + 5]))


def _shape(rng, T):
    while True:
        P, G = int(rng.choice(PS + [int(rng.integers(1, 60))])), int(rng.choice(GS))
        if P * G * T <= MAX_RING_CELLS:
            return P, G


def _recipe_map(rng, md):
    """gpr.h's recipe: keep every pod with a live row (and some that a slice would bring), add head-room, widen G,
    shuffle the pods"""
    m = md.ring
    live = live_model(m.planes).reshape(m.P, m.G).any(axis=1)
    kept = np.flatnonzero(live | (rng.random(m.P) < 0.3))
    if kept.size == 0:
        kept = np.array([int(rng.integers(0, m.P))])
    G = m.G + int(rng.integers(0, 2))
    P = kept.size + int(rng.integers(0, 4))
    while P * G * m.T > MAX_RING_CELLS:
        if G > m.G:
            G -= 1
        else:
            P -= 1
            kept = kept[:P]
    order = rng.permutation(kept)
    src = np.full((P, G), NONE, np.uint32)
    for i, p in enumerate(order):
        src[i, :m.G] = np.arange(p * m.G, (p + 1) * m.G, dtype=np.uint32)
    return P, G, src.ravel()


def _random_map(rng, md, shrink=False):
    m = md.ring
    while True:
        P, G = _shape(rng, m.T)
        if not shrink or P * G < m.rows:
            break
        if m.rows == 1:
            P, G = 1, 1
            break
    n = P * G
    src = np.full(n, NONE, np.uint32)
    k = min(n, m.rows) * 3 // 4 if rng.random() < 0.7 else min(n, m.rows)
    if k:
        src[rng.choice(n, k, replace=False)] = rng.choice(m.rows, k, replace=False)
    return P, G, src


def plan_ring(seed, n_ops=N_OPS):
    """the operations of sequence `seed`"""
    rng = np.random.default_rng([seed, 0x21A6])
    md = Model()
    ops = []

    def add(op):
        out = md.apply(op)
        if op["kind"] == "remap":
            op["shrink"] = bool(out["shrink"])
        ops.append(op)

    def seed_():
        return int(rng.integers(1 << 31))

    def async_():
        add(dict(kind="async", win=S.draw_window(rng, False, src="dev", table=False, small=True)))

    def ring_async():
        m = md.ring
        calls = []
        for _ in range(int(rng.integers(1, 5))):
            thr = float(rng.choice(edges.THRESHOLDS)) if len(m.planes) > 1 and rng.random() < 0.7 else None
            calls.append(dict(thr=thr, gates=bool(rng.random() < 0.5), table=bool(m.G > 1 and rng.random() < 0.4),
                              outs={k: bool(rng.random() < 0.5) for k in S.OUTPUTS},
                              out_kind=str(rng.choice(["host", "dev"])), seed=seed_()))
        add(dict(kind="ring_async", calls=calls))

    def init(power=None, index=None):
        add(dict(kind="init", ring=_ring_spec(rng, power, index)))
        if rng.random() < 0.7:            # most rings start full
            m = md.ring
            add(dict(kind="append", n_new=m.T, src=str(rng.choice(["host", "dev"])), power_cols=len(m.planes) > 1,
                     stride=0, seed=seed_()))

    def merge(n_new=None, plane=None, src=None, revive=None):
        m = md.ring
        plane = plane if plane is not None else int(len(m.planes) > 1 and rng.random() < 0.4)
        src = src or str(rng.choice(MERGE_SOURCES))
        n_rows = m.rows if rng.random() < 0.7 else int(rng.integers(1, m.rows + 1))
        if revive is None:   # rows that are empty now: the merge brings them back to life
            dead = np.flatnonzero(~live_model(m.planes))
            dead = dead[dead < n_rows]
            revive = [int(x) for x in rng.permutation(dead)[:3]]
        return dict(kind="merge", n_new=n_new or _n_new(rng, m.T), plane=plane, src=src, n_rows=n_rows,
                    thr=float(rng.choice(edges.THRESHOLDS)), M=int(rng.choice(CHUNK_M)), seed=seed_(), revive=revive)

    def decide_resident():
        m = md.ring
        if m.index and md.stale:
            add(dict(kind="reindex"))
        add(dict(kind="decide_resident", mode=str(rng.choice(["whole", "early"])),
                 table=bool(m.G > 1 and rng.random() < 0.5), gates=bool(rng.random() < 0.5),
                 thr=float(rng.choice(edges.THRESHOLDS)) if len(m.planes) > 1 and rng.random() < 0.7 else None,
                 gates_kind=str(rng.choice(["host", "dev"])), seed=seed_()))

    def remap(kind=None, shrink=False):
        kind = kind or ("recipe" if rng.random() < 0.5 else "random")
        if kind == "recipe" and not shrink:
            P, G, src = _recipe_map(rng, md)
        else:
            P, G, src = _random_map(rng, md, shrink)
        add(dict(kind="remap", how=kind, P=P, G=G, src=[int(x) for x in src], mem=str(rng.choice(["host", "dev"]))))

    def ensure_pending():
        if md.pending == 0:
            if md.ring is not None and rng.random() < 0.8:
                ring_async()
            else:
                async_()

    def export():
        add(dict(kind="export", plane=int(len(md.ring.planes) > 1 and rng.random() < 0.5),
                 M=int(rng.choice(EXPORT_M))))

    def failure(f):
        m = md.ring
        if f in ("export_no_power", "merge_no_power") and len(m.planes) > 1:
            init(power=False)
        m = md.ring
        if f == "merge_rows_over":
            while md.ring.rows == 1:
                init()
            rows_before = md.ring.rows
            ensure_pending()
            remap(shrink=True)
            op = dict(kind="fail", fail=f, code=FAILURES[f], n_rows=rows_before, n_new=1, plane=0,
                      src=str(rng.choice(["samples_pageable", "samples_dev", "chunks_host", "chunks_dev", "text"])),
                      thr=150.0, M=120, seed=seed_(), revive=None)
            if op["src"] == "text":
                op["src"] = "samples_pinned"
            add(op)
            return
        if f == "export_capacity":
            pls = [pl for pl in range(len(m.planes)) if live_model(m.planes[pl:pl + 1]).any()]
            if not pls:
                add(dict(kind="append", n_new=m.T, src="host", power_cols=len(m.planes) > 1, stride=0, seed=seed_()))
                pls = [0]
        if f == "decide_stale" and not (m.index and md.stale):
            if not m.index:
                init(index=True)
            add(merge())
        ensure_pending()
        m = md.ring
        op = dict(kind="fail", fail=f, code=FAILURES[f])
        if f in ("remap_range_host", "remap_range_dev", "remap_twice_host", "remap_twice_dev"):
            P, G, src = _random_map(rng, md)
            src = src.copy()
            i = int(rng.integers(0, src.size))
            if "range" in f:
                src[i] = m.rows + int(rng.integers(0, 3)) if rng.random() < 0.7 else 0x7FFFFFFF
            else:
                if src.size == 1:
                    P, G, src = 2, 1, np.array([NONE, NONE], np.uint32)
                    i = 1
                j = int(rng.choice([x for x in range(src.size) if x != i]))
                src[i] = src[j] = int(rng.integers(0, m.rows))
            op.update(P=P, G=G, src=[int(x) for x in src])
        elif f == "export_capacity":
            op.update(plane=int(rng.choice(pls)), M=int(rng.choice(EXPORT_M)), short=str(rng.choice(
                ["series", "chunks", "bytes"])))
        elif f == "export_bad_T":
            op.update(plane=0, M=120, T=m.T + 1 if rng.random() < 0.5 or m.T == 1 else m.T - 1)
        elif f == "export_no_power":
            op.update(plane=1, M=120)
        elif f in ("merge_bad_row", "merge_truncated", "merge_no_power"):
            src = {"merge_bad_row": str(rng.choice(["samples_pageable", "samples_pinned", "samples_dev",
                                                     "chunks_host", "chunks_dev"])),
                   "merge_truncated": str(rng.choice(["chunks_host", "chunks_dev"])),
                   "merge_no_power": str(rng.choice(["samples_pageable", "chunks_host"]))}[f]
            op.update(merge(plane=1 if f == "merge_no_power" else 0, src=src))
            op.update(kind="fail", fail=f, code=FAILURES[f], revive=None)
            if f == "merge_truncated":
                op["M"] = 7
            if f == "merge_bad_row" or f == "merge_truncated":
                # the chunk or row at fault: drawn once the slice is known
                T, t_end = m.T, md.t_end + op["n_new"] * STEP
                offsets, rows, ts, bits = merge_slice(op, T, t_end)
                if f == "merge_bad_row":
                    op["bad_series"] = int(rng.integers(0, len(rows)))
                else:
                    sc, cb, _ = slice_chunks(op, offsets, ts, bits)
                    long_ = [c for c in range(len(cb) - 1) if int(cb[c + 1] - cb[c]) > 3]
                    op["chunk"] = int(rng.choice(long_))
        add(op)

    fails = [f for f in FAILURES if f not in NO_RING]
    rng.shuffle(fails)
    slots = sorted(rng.choice(np.arange(3, n_ops - 2), size=len(fails), replace=False).tolist())
    scheduled = dict(zip(slots, fails))
    for f in NO_RING:                 # before any ring, with a plain result pending
        async_()
        add(dict(kind="fail", fail=f, code=FAILURES[f], P=2, G=2, src=[0, 1, 2, 3]))
    init()
    i = 0
    while len(ops) < n_ops or i <= max(scheduled):
        f = scheduled.get(i)
        i += 1
        m = md.ring
        if md.pending > MAX_PENDING - 10:
            add(dict(kind="sync"))
            continue
        if f is not None:
            failure(f)
            continue
        prev = ops[-1]["kind"]
        r = rng.random()
        if prev == "remap" and r < 0.6:      # what a remap carries into: live rows, an export, a merge
            q = rng.random()
            if ops[-1]["shrink"] and q < 0.5:
                add(merge())
            elif q < 0.4:
                add(dict(kind="live_rows", out=str(rng.choice(["host", "dev"]))))
            elif q < 0.7:
                export()
            else:
                add(merge())
            continue
        if r < 0.10:
            add(dict(kind="append", n_new=_n_new(rng, m.T), src=str(rng.choice(["host", "dev"])),
                     power_cols=bool(len(m.planes) > 1 and rng.random() < 0.7), stride=int(rng.choice([0, 0, 3])),
                     seed=seed_()))
        elif r < 0.15:
            add(dict(kind="advance", n_new=_n_new(rng, m.T)))
        elif r < 0.30:
            add(merge())
            if rng.random() < 0.3:
                add(dict(kind="live_rows", out=str(rng.choice(["host", "dev"]))))
        elif r < 0.42:
            # plant, then the op it was planted for
            then = str(rng.choice(["advance", "merge", "remap"], p=[0.5, 0.25, 0.25]))
            n_new = 0 if then == "remap" else _n_new(rng, m.T) if rng.random() < 0.3 else int(
                rng.choice([1, max(1, m.T - 1), max(1, m.T // 3)]))
            if m.index and md.stale and rng.random() < 0.5:
                add(dict(kind="reindex"))
            add(dict(kind="plant", seed=seed_(), open=n_new))
            if rng.random() < 0.4:
                ensure_pending()
            if then == "advance":
                add(dict(kind="advance", n_new=n_new))
                if rng.random() < 0.6:
                    add(dict(kind="live_rows", out=str(rng.choice(["host", "dev"]))))
                else:
                    decide_resident()
            elif then == "merge":
                add(merge(n_new=n_new))
            else:
                remap()
        elif r < 0.49:
            add(dict(kind="live_rows", out=str(rng.choice(["host", "dev"]))))
        elif r < 0.57:
            remap()
        elif r < 0.63:
            export()
        elif r < 0.67:
            same = rng.random() < 0.3
            P, G = (m.P, m.G) if same else _shape(rng, m.T)
            pods = np.full(m.P, -1, np.int64)
            take = rng.permutation(m.P)[:min(m.P, P)]
            pods[take] = rng.permutation(P)[:take.size]
            if same:
                pods = np.arange(m.P)
            add(dict(kind="restore", P=P, G=G, pods=[int(x) for x in pods], index=bool(rng.random() < 0.5)))
        elif r < 0.79:
            ring_async()
        elif r < 0.84:
            add(dict(kind="sync"))
        elif r < 0.93:
            decide_resident()
        elif r < 0.96:
            init()
        else:
            add(dict(kind="reindex"))
    return ops


def replay(ops):
    """(op, what it must give, the model after it) for every op of a plan"""
    md = Model()
    for op in ops:
        out = md.apply(op)
        yield op, out, md


def transitions(ops):
    md = Model()
    for op in ops:
        md.apply(op)
    return md.seen | {"fail " + f + " with results pending" for f in md.fails_pending}
