"""Scripts of resident-ring operations and the plain numpy model of the ring they are checked against.  TEST
INFRASTRUCTURE, shared by tests/test_ring_emul.py (the ring kernels' source on the CPU) and tests/test_gpu_resident.py
(libgpr.so on an H100).

The model is the ring as gpr.h describes it: one uint32 cell per (row, position), a head, and an append of n_new
columns that writes source column skip + j to position (head + skip + j) % T, skip = max(0, n_new - T).  The block
index it implies is np.fmax.reduce over positions [64 b, min(T, 64 b + 64)) of each row.

The scripts are built so that a kernel that skips a block recompute gives a wrong index and a wrong verdict: before
most operations the ring is rewritten so that the only non-zero sample (or the only power reading at or above the
threshold) of every block the operation touches sits at a position the operation overwrites or opens.
"""
from __future__ import annotations

import dataclasses

import numpy as np

import edges

BLOCK = 64
NO_SAMPLE = 0xFFFFFFFF   # what gpr_resident_init and the opened buckets hold
QNAN = 0x7FC00000
THR = 150.0


def _bits(vals):
    return np.asarray(vals, np.float32).view(np.uint32)


def power_cell(x: float) -> np.float32:
    """the f32 a power reading x is stored as (the POWER RULE of gpr.h) for the threshold THR"""
    up = np.float32(edges.f32_up(THR))
    f = np.float32(x)
    if x >= THR and f < up:
        f = up
    if x < THR and f >= up:
        f = np.nextafter(up, np.float32(-np.inf))
    return f


_Z = np.asarray(edges.ZEROISH, np.float32)
# util: "quiet" cells leave a block idle-or-absent (max <= 0 or NaN), "loud" ones make it busy
UTIL_QUIET = np.unique(np.concatenate([_bits(_Z[_Z <= 0]), _bits([0.0, -0.0, -np.inf, -3.0]),
                                       np.array([NO_SAMPLE, QNAN, 0xFFC00000], np.uint32)]))
UTIL_LOUD = np.unique(np.concatenate([_bits(_Z[_Z > 0]), _bits([5.0, 100.0, np.inf]),
                                      np.array([0x00000001], np.uint32)]))   # the smallest denormal
_PW = np.array([power_cell(x) for x in edges.power_edges(THR)], np.float32)
POWER_QUIET = np.unique(np.concatenate([_bits(_PW[_PW < THR]), _bits([55.5, -np.inf, 0.0, -0.0]),
                                        np.array([NO_SAMPLE, QNAN], np.uint32)]))
POWER_LOUD = np.unique(np.concatenate([_bits(_PW[_PW >= THR]), _bits([200.0, np.inf])]))
POOLS = {(0, False): UTIL_QUIET, (0, True): UTIL_LOUD, (1, False): POWER_QUIET, (1, True): POWER_LOUD}


def index_ld(T):
    return ((T + BLOCK - 1) // BLOCK + 3) & ~3


class Ring:
    def __init__(self, P, G, T, flags):
        self.P, self.G, self.T, self.flags = P, G, T, flags
        self.rows = P * G
        self.index = bool(flags & 2)
        self.planes = [np.full((self.rows, T), NO_SAMPLE, np.uint32) for _ in range(2 if flags & 1 else 1)]
        self.head = 0

    def span(self, n_new):
        """(skip, ring positions) of the columns an append of n_new writes"""
        skip = max(0, n_new - self.T)
        return skip, (self.head + skip + np.arange(n_new - skip)) % self.T

    def append(self, n_new, util, power):
        skip, pos = self.span(n_new)
        self.planes[0][:, pos] = util[:, skip:skip + len(pos)]
        if len(self.planes) > 1:
            self.planes[1][:, pos] = power[:, skip:skip + len(pos)] if power is not None else NO_SAMPLE
        self.head = (self.head + n_new) % self.T

    def advance(self, n):
        _, pos = self.span(n)
        for p in self.planes:
            p[:, pos] = NO_SAMPLE
        self.head = (self.head + n) % self.T

    def write(self, pl, cells):
        self.planes[pl] = cells.copy()

    def window(self, pl):
        """the unrolled window [P, G, T] (oldest bucket first)"""
        return np.roll(self.planes[pl].view(np.float32), -self.head, axis=1).reshape(self.P, self.G, self.T)

    def block_max(self, pl):
        """[rows, idx_ld] float32: np.fmax.reduce of every block, NaN padding; and [rows, blocks] mixed-zero flags"""
        v = self.planes[pl].view(np.float32)
        nb = (self.T + BLOCK - 1) // BLOCK
        out = np.full((self.rows, index_ld(self.T)), np.nan, np.float32)
        mixed = np.zeros((self.rows, nb), bool)
        for b in range(nb):
            blk = v[:, b * BLOCK:min(self.T, b * BLOCK + BLOCK)]
            out[:, b] = np.fmax.reduce(blk, axis=1)
            z = blk == 0
            mixed[:, b] = (z & np.signbit(blk)).any(axis=1) & (z & ~np.signbit(blk)).any(axis=1)
        return out, mixed


def index_matches(got_bits, model: Ring, pl):
    """the index bits equal the model's block maxima: same value or both NaN, equal bits unless the block holds zeros
    of both signs (fmaxf may return either), NaN in the padding.  Returns a description of the first mismatch."""
    want, mixed = model.block_max(pl)
    got = got_bits.view(np.float32).reshape(want.shape)
    nan_ok = np.isnan(got) & np.isnan(want)
    same_bits = got.view(np.uint32) == want.view(np.uint32)
    same_value = got == want
    nb = mixed.shape[1]
    ok = nan_ok.copy()
    ok[:, :nb] |= np.where(mixed, same_value[:, :nb], same_bits[:, :nb])
    if ok.all():
        return None
    r, b = np.argwhere(~ok)[0]
    return f"row {r} block {b}: got {got[r, b]!r} ({got.view(np.uint32)[r, b]:#010x}), want {want[r, b]!r}"


@dataclasses.dataclass
class Case:
    name: str
    sm: int
    P: int
    G: int
    T: int
    flags: int
    ops: list
    regimes: set          # what the case was built for; asserted against what its operations reached
    hit: set = dataclasses.field(default_factory=set)


def _cells(rng, plane, rows, n, loud=False):
    pool = POOLS[(plane, loud)]
    return pool[rng.integers(0, len(pool), (rows, n))]


def _mixed(rng, plane, rows, n):
    c = _cells(rng, plane, rows, n)
    busy = rng.random((rows, n)) < 0.05
    c[busy] = _cells(rng, plane, rows, n, True)[busy]
    return c


def _regimes(model: Ring, op, sm):
    out = set()
    if model.rows > 16 * sm:
        out.add("CTA row loop strides")
    kind = op[0]
    if kind not in ("append", "advance"):
        return out
    n_new = op[1]
    T = model.T
    skip, pos = model.span(n_new)
    start, n = int(pos[0]), len(pos)
    if start % BLOCK:
        out.add("head not block-aligned")
    if start + n > T:
        out.add("span wraps")
        if start // BLOCK <= (start + n - T - 1) // BLOCK:
            out.add("a block in both runs")
    if T % BLOCK and (start + n > T or (start + n - 1) // BLOCK == (T - 1) // BLOCK):
        out.add("partial last block")
    if (T + BLOCK - 1) // BLOCK > 4:
        out.add("more blocks than warps")
    if skip:
        out.add("n_new > T")
    if kind == "append":
        ld = op[2]
        if ld > n_new:
            out.add("strided source")
            if skip:
                out.add("n_new > T, strided")
        if len(model.planes) > 1 and op[4] is None:
            out.add("power NULL with a power plane")
        if len(model.planes) == 1:
            out.add("no power plane")
    elif model.index:
        out.add("advance on an index ring")
    return out


def run_model(case: Case):
    """yields (op, model after op) for every operation of the case"""
    m = None
    for op in case.ops:
        if op[0] == "init":
            m = Ring(*op[1:])
        elif op[0] == "append":
            m.append(op[1], op[3], op[4])
        elif op[0] == "advance":
            m.advance(op[1])
        elif op[0] == "write":
            m.write(op[1], op[2])
        yield op, m


def build_case(name, T, P=3, G=1, flags=3, sm=1, seed=0, regimes=(), heads=None, nnew=None):
    """The head visits every position of `heads` (default 0, 1, 63, 64, 65, T - 1); from each, every n_new of `nnew`
    (default 1, 63, 64, 65, T - 1, T, T + 1, 2T + 3) is applied once, as an append with the power columns, an append
    with power_cols NULL and a strided source, a strided append, or an advance, in turn.  Before each, the blocks it
    touches are rewritten so that their only busy sample is one it overwrites."""
    rng = np.random.default_rng(seed)
    rows = P * G
    ops = [("init", P, G, T, flags)]
    m = Ring(P, G, T, flags)
    npl = len(m.planes)
    hit = set()
    heads = sorted({h for h in (heads or (0, 1, 63, 64, 65, T - 1)) if 0 <= h < T})
    nnew = sorted({n for n in (nnew or (1, 63, 64, 65, T - 1, T, T + 1, 2 * T + 3)) if n >= 1})

    def do(op):
        hit.update(_regimes(m, op, sm))
        ops.append(op)
        if op[0] == "append":
            m.append(op[1], op[3], op[4])
        elif op[0] == "advance":
            m.advance(op[1])
        elif op[0] == "write":
            m.write(op[1], op[2])

    k = 0
    for h in heads:
        for n in nnew:
            d = (h - m.head) % T
            if d:   # bring the head to h over ordinary traffic
                if k % 5 == 4:
                    do(("advance", d))
                else:
                    do(("append", d, d, _mixed(rng, 0, rows, d), _mixed(rng, 1, rows, d) if npl > 1 else None))
            # the only busy sample of every block n touches is at a position n overwrites
            _, pos = m.span(n)
            for pl in range(npl):
                cells = _cells(rng, pl, rows, T)
                for b in np.unique(pos // BLOCK):
                    mine = pos[pos // BLOCK == b]
                    for r in range(rows):
                        if rng.random() < 0.8:
                            cells[r, rng.choice(mine)] = _cells(rng, pl, 1, 1, True)[0, 0]
                do(("write", pl, cells))
            if m.index:
                do(("reindex",))
            kind = k % 4
            if kind == 3:
                do(("advance", n))
            else:
                ld = n if kind == 0 else n + (5 if kind == 1 else 3)
                util = _cells(rng, 0, rows, ld)
                power = _cells(rng, 1, rows, ld) if npl > 1 and kind != 1 else None
                do(("append", n, ld, util, power))
            k += 1
    return Case(name, sm, P, G, T, flags, ops, set(regimes), hit)


TS = [1, 2, 3, 4, 5, 63, 64, 65, 127, 128, 129, 191, 192, 193, 240, 1800]
# the regimes every case with an index and a power plane reaches, whatever its T
_COMMON = {"n_new > T", "strided source", "n_new > T, strided", "power NULL with a power plane",
           "advance on an index ring"}


def cases():
    out = []
    for i, T in enumerate(TS):
        want = set(_COMMON)
        if T > 1:
            want |= {"span wraps"}
        if T > 64:
            want |= {"head not block-aligned", "a block in both runs"}
        if T % BLOCK:
            want.add("partial last block")
        if T > 4 * BLOCK:
            want.add("more blocks than warps")
        out.append(build_case(f"T={T}", T, seed=100 + i, regimes=want))
    out.append(build_case("no power plane", 193, P=2, G=3, flags=2, seed=7,
                          regimes={"no power plane", "partial last block", "a block in both runs"}))
    out.append(build_case("no index", 129, P=2, G=2, flags=1, seed=8,
                          regimes={"power NULL with a power plane", "span wraps"}))
    out.append(build_case("row loop, 1 SM", 129, P=9, G=2, flags=3, sm=1, seed=9, heads=(0, 65, 128),
                          nnew=(64, 129, 261), regimes={"CTA row loop strides", "a block in both runs"}))
    out.append(build_case("row loop, 2 SMs", 65, P=11, G=3, flags=3, sm=2, seed=10, heads=(1, 64),
                          nnew=(63, 65, 133), regimes={"CTA row loop strides", "partial last block"}))
    return out


ALL_REGIMES = _COMMON | {"span wraps", "head not block-aligned", "a block in both runs", "partial last block",
                         "more blocks than warps", "no power plane", "CTA row loop strides"}
