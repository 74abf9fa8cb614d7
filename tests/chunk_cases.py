"""Seeded cases for the Prometheus XOR chunk codec (TEST INFRASTRUCTURE), shared by tests/test_chunk_cases.py (the
kernels' source on the CPU) and tests/test_gpu_chunk_codec.py (the H100).  Every case comes from a seed.

  known_answers(t_end, step, T)      [(name, chunk)]: chunks written bit by bit (BitWriter, not the encoder) whose
                                     samples land inside the window [t_end - T * step, t_end] (ms), one column apart:
                                     both ends of every delta-of-delta bucket, the 64-bit bucket, the leading-zero
                                     clamp, 64 significant bits written as 0, window reuse, a window wider than 64
                                     bits, 10-byte varints, first timestamps negative or near INT64_MAX, timestamps
                                     that wrap int64, counts of 0, 1, 2 and 65535, special values
  random_series(rng, n, t_end, step, T) -> (ts, bits): any-bit values and jittery timestamps
  corrupted(rng, chunk, other)       [(how, chunk)]: a valid chunk with bits flipped, cut short, recounted or spliced
  verdict(chunk)                     (ts, bits, fault bit): tests/chunks_ref.py's decode, the fault as the ABI's bit
  coverage(chunk)                    the set of format paths the decode of `chunk` takes (PATHS)
  decoder_plan(seed, ...) / corrupt_plan(seed, ...)   the cases both test files run
"""
import functools
import hashlib

import numpy as np

import chunks_ref as R
from chunks_ref import MASK64, BitWriter, f2b
from test_chunks_ref import DOD_CASES

FAULT_BIT = {None: 0, "short": 32, "overrun": 64, "no_window": 128, "varint": 256}
# the message gpr_chunks_scatter gives for a batch's fault bits: the first kind of this list that is set
FAULT_TEXT = ((32, "shorter than its 2-byte header"), (64, "its samples run past its bytes"),
              (128, "a value reuses the XOR window before one was set"), (256, "a varint overflows 64 bits"))

BUCKETS = {14: "10", 17: "110", 20: "1110", 64: "1111"}
PATHS = frozenset(
    ["dod0", "dod64", "dod64_neg", "clamp", "sig64", "reuse", "wide_window", "varint10", "ts_wrap", "count0",
     "count65535", "short", "overrun", "no_window", "varint"]
    + [f"dod{sz}{end}" for sz in (14, 17, 20) for end in ("", "_top", "_bottom")])


def i64(x):
    x &= MASK64
    return x - (1 << 64) if x >> 63 else x


def _start(t0, v0):
    """a chunk's first sample: zigzag varint timestamp, 64 raw bits"""
    return BitWriter().varint(i64(t0)).put(v0 & MASK64, 64)


def _window(w, x, lead, sig):
    """x in a new XOR window of `lead` leading and `sig` significant bits, as written ('11' + 5 + 6 + bits)"""
    trail = 64 - lead - sig
    return w.string("11").put(lead, 5).put(sig & 63, 6).put(x >> trail, sig)


# ---- known answers ------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def known_answers(t_end, step, T):
    """[(name, chunk bytes)], each chunk's landing samples inside the window (ms)"""
    cases = []
    top = [t_end - k * step for k in range(T)]   # column tops, newest first
    v0, v2 = f2b(1.0), f2b(0.5)                   # 1.0 ^ 0.5 = one exponent bit: lead 11, sig 1

    def land(k, edge):
        """the timestamp in column k from the newest, at the top (edge 0) or bottom (edge 1) of the column"""
        return top[1 + k % (T - 2)] - edge * (step - 1)

    # every bucket's payloads: both ends, one past each end (DOD_CASES), 1 and -1 written in every bucket, 0 in a
    # payload; sample 2 lands in the window (t0 and t1 wherever the dod puts them), sample 3 follows at dod 0
    payloads = [(dod & ((1 << sz) - 1) if sz else 0, prefix, sz) for dod, prefix, sz in DOD_CASES]
    for sz in (14, 17, 20, 64):
        m = (1 << sz) - 1
        payloads += [(1, BUCKETS[sz], sz), (m, BUCKETS[sz], sz), (0, BUCKETS[sz], sz)]
        if sz < 64:
            payloads += [(1 << (sz - 1), BUCKETS[sz], sz), ((1 << (sz - 1)) + 1, BUCKETS[sz], sz)]
    payloads += [((-(1 << 62) + 12345) & MASK64, "1111", 64), (1 << 63, "1111", 64), (MASK64 >> 1, "1111", 64)]
    for k, (payload, prefix, sz) in enumerate(payloads):
        if sz == 64:
            dod = i64(payload)
        else:
            dod = payload - (1 << sz) if sz and payload > (1 << (sz - 1)) else payload
        for edge in (0, 1):
            t2 = land(k, edge)
            d1 = step
            t0 = i64(t2 - 2 * d1 - dod)
            w = _start(t0, v0).uvarint(d1).bit(0).string(prefix)
            if sz:
                w.put(payload, sz)
            _window(w, v0 ^ v2, 11, 1)
            w.bit(0).bit(0)
            cases.append((f"dod payload {payload:#x} in {sz or 0} bits, edge {edge}", w.chunk(4)))

    # a first timestamp negative, INT64_MIN (a 10-byte zigzag varint) or near INT64_MAX; a delta of 2^64 - 1 (the last
    # legal 10-byte uvarint) and deltas that wrap int64 back into the window
    t = land(3, 0)
    for t0 in (-5000, -(1 << 63), (1 << 63) - 1 - 10, (1 << 63) - 1):
        w = _start(t0, v0).uvarint((t - t0) & MASK64)
        _window(w, v0 ^ v2, 11, 1)
        cases.append((f"first timestamp {t0}", w.chunk(2)))
    w = _start(t + 1, v0).uvarint(MASK64)   # t + 1 + (2^64 - 1) = t
    cases.append(("delta 2^64 - 1", _window(w, v0 ^ v2, 11, 1).chunk(2)))

    # counts 0, 1, 2 (bytes after the last sample unread) and 65535
    cases.append(("count 0", b"\x00\x00"))
    cases.append(("count 0, bytes after it", b"\x00\x00\xff\xff\x01"))
    cases.append(("count 1", _start(land(4, 1), f2b(42.0)).chunk(1) + b"\xff"))
    cases.append(("count 2", _window(_start(land(5, 0), v0).uvarint(step), v0 ^ v2, 11, 1).chunk(2)))
    n = 65535
    ts = [t_end - n + 1 + 2 * i - (i * 7 % 5) for i in range(n)]
    cases.append(("count 65535", R.encode(ts, [float(i % 97) for i in range(n)])))

    # XOR windows: the leading-zero clamp (x = bits 29..31, lead 32 written as 31 with 4 significant bits); 64
    # significant bits written as 0; reuse, then a new window; a window of lead + sig > 64 that reads its bits and
    # changes nothing (Go's uint8 arithmetic), reused, then a real window
    ts = [land(6 + k, 0) for k in range(4)][::-1]
    x = 0x00000000E0000000
    w = _start(ts[0], v0).uvarint(ts[1] - ts[0]).string("11").put(31, 5).put(4, 6).put(x >> 29, 4)
    cases.append(("lead clamp at 31", w.chunk(2)))
    x = 0x8000000020000001
    w = _start(ts[0], v0).uvarint(ts[1] - ts[0]).string("11").put(0, 5).put(0, 6).put(x, 64)
    cases.append(("64 significant bits written as 0", w.chunk(2)))
    a = 0x4059000000000000
    x1, x2, x3 = 0x000ABC0000000000, 0x0008040000000000, 0x00000000E0000000
    w = _start(ts[0], a).uvarint(ts[1] - ts[0])
    _window(w, x1, 12, 10).bit(0).bit(1).bit(0).put(x2 >> 42, 10)
    w.bit(0).string("11").put(31, 5).put(4, 6).put(x3 >> 29, 4)
    cases.append(("window reuse and a new window", w.chunk(4)))
    for lead, sig in ((31, 40), (31, 0), (1, 64), (20, 45)):
        w = _start(ts[0], a).uvarint(ts[1] - ts[0])
        w.string("11").put(lead, 5).put(sig & 63, 6).put((1 << (sig or 64)) - 1, sig or 64)
        w.bit(0).string("10").put(12345, sig or 64)
        _window(w.bit(0), x1, 12, 10)
        cases.append((f"window lead {lead} sig {sig or 64}", w.chunk(4)))

    # special values through the reference encoder (its bytes are held to hand-written chunks in test_chunks_ref.py)
    special = [R.STALE_NAN_BITS, f2b(float("inf")), f2b(-0.0), f2b(float("-inf")), f2b(0.0), 0x7FF8000000000001,
               0xFFF0000000000001, f2b(5e-324), f2b(-1e-310), f2b(150.0), f2b(float(np.float32(150) + 0)),
               f2b(float(np.nextafter(np.float32(150), np.float32(0)))), f2b(7.0)]
    cases.append(("special values", R.encode([land(10 + k, k & 1) for k in range(len(special))][::-1], special)))
    return cases


# ---- random series ------------------------------------------------------------------------------------------------
F150 = np.float32(150)
NEAR150 = [f2b(float(x)) for x in (np.nextafter(F150, np.float32(0)), F150, np.nextafter(F150, np.float32(1e9)))]
NEAR150 += [f2b(150.0 - 2 ** -45), f2b(150.0 + 2 ** -45), f2b(149.99), f2b(149.99000000000001)]
ODD_BITS = [R.STALE_NAN_BITS, 0x7FF8000000000000, 0x7FF8000000000001, 0xFFF8000000000000, 0x7FF0000000000001,
            0x7FF0000000000000, 0xFFF0000000000000, 0, 1 << 63, 1, 0x000FFFFFFFFFFFFF, 0x8000000000000001]
DOD_EDGES = [8192, -8191, 8193, -8192, 65536, -65535, 65537, -65536, 524288, -524287, 524289, -524288, 1 << 33,
             -(1 << 40)]


def random_series(rng, n, t_end, step, T):
    """one series of n samples: (ts list, value bits list).  Values: any 64 bits, the staleness marker, NaN payloads,
    +-0, subnormals, and f32 neighbours of 150 W.  Timestamps: a scrape every `step` ms from a little before the
    window, with jitter at several scales and one-sample jumps by the delta-of-delta buckets' edges and far away."""
    bits = rng.integers(0, 1 << 64, n, dtype=np.uint64)
    pick = rng.random(n)
    bits[pick < 0.15] = rng.choice(np.array(ODD_BITS, np.uint64), int((pick < 0.15).sum()))
    near = (pick >= 0.15) & (pick < 0.3)
    bits[near] = rng.choice(np.array(NEAR150, np.uint64), int(near.sum()))
    sub = (pick >= 0.3) & (pick < 0.35)
    bits[sub] = rng.integers(1, 1 << 52, int(sub.sum()), dtype=np.uint64) | (rng.integers(0, 2, int(sub.sum()),
                                                                                           dtype=np.uint64) << 63)
    small = (pick >= 0.35) & (pick < 0.6)    # values that survive f32: repeats and neighbours make XOR windows reuse
    bits[small] = rng.integers(0, 300, int(small.sum())).astype(np.float64).view(np.uint64)
    deltas = np.full(n, step, np.int64)
    scale = int(rng.choice([0, 3, 900, 20_000]))
    deltas += rng.integers(-scale, scale + 1, n)
    for i in np.flatnonzero(rng.random(n) < 0.08):
        e = int(rng.choice(DOD_EDGES))
        deltas[i] += e
        if i + 1 < n:
            deltas[i + 1] -= e
    t0 = t_end - (T + 2) * step + int(rng.integers(-3 * step, 3 * step))
    ts = t0 + np.concatenate([[0], np.cumsum(deltas[1:])])
    return [int(t) for t in ts], [int(b) for b in bits]


# ---- corrupted chunks -----------------------------------------------------------------------------------------------
def corrupted(rng, chunk, other, every_cut=False):
    """[(how, bytes)]: `chunk` with 1-3 bits flipped (header included), cut short (at every length, or one), its count
    raised or lowered, and spliced with `other`"""
    out = []
    for _ in range(2):
        b = bytearray(chunk)
        for bit in rng.choice(8 * len(b), min(int(rng.integers(1, 4)), 8 * len(b)), replace=False):
            b[bit >> 3] ^= 0x80 >> (bit & 7)
        out.append(("flip", bytes(b)))
    cuts = range(len(chunk)) if every_cut else [int(rng.integers(0, len(chunk)))]
    out += [(f"cut {k}", chunk[:k]) for k in cuts]
    count = int.from_bytes(chunk[:2], "big")
    for d in (1, int(rng.integers(2, 40)), -1, -int(rng.integers(2, 40))):
        c = count + d
        if 0 <= c <= 0xFFFF and len(chunk) >= 2:
            out.append((f"count {d:+d}", c.to_bytes(2, "big") + chunk[2:]))
    i, j = int(rng.integers(0, len(chunk) + 1)), int(rng.integers(0, len(other) + 1))
    out.append(("splice", chunk[:i] + other[j:]))
    return out


def bad_varints():
    """[(how, chunk)]: varints one past the last legal 10-byte value, and 11 bytes long, in the first timestamp and in
    the first delta"""
    nine = BitWriter().put((1 << 72) - 1, 72)
    first = [("timestamp varint, tenth byte 2", nine.byte(2).put(0, 64).chunk(1)),
             ("timestamp varint of 11 bytes", BitWriter().put((1 << 80) - 1, 80).byte(1).put(0, 64).chunk(1))]
    delta = [(f"delta varint, tenth byte {b}", BitWriter().varint(5).put(0, 64).put((1 << 72) - 1, 72).byte(b)
              .bit(0).chunk(2)) for b in (2, 0x7F)]
    return first + delta


def verdict(chunk):
    ts, vals, fault = R.decode(chunk)
    return ts, vals, FAULT_BIT[fault]


def fault_text(bits):
    return next(t for b, t in FAULT_TEXT if bits & b)


# ---- which format paths a chunk takes ------------------------------------------------------------------------------
class _Trace(R._Reader):
    def uvarint(self):
        start = self.pos
        x = super().uvarint()
        self.long = (self.pos - start) == 80
        return x


def coverage(chunk):
    """the format paths (PATHS) the decode of `chunk` takes, up to its first fault; also -> the decode itself, which
    must equal tests/chunks_ref.py's"""
    chunk = bytes(chunk)
    seen = set()
    if len(chunk) < 2:
        return {"short"}, ([], [], "short")
    count = int.from_bytes(chunk[:2], "big")
    seen |= {"count0"} if count == 0 else {"count65535"} if count == 0xFFFF else set()
    r = _Trace(chunk[2:])
    ts, vals = [], []
    t = delta = v = 0
    sig = trail = None
    fault = None
    try:
        for i in range(count):
            if i == 0:
                u = r.uvarint()
                seen |= {"varint10"} if r.long else set()
                t = (u >> 1) ^ (-(u & 1) & MASK64)
                v = r.take(64)
            else:
                if i == 1:
                    delta = r.uvarint()
                    seen |= {"varint10"} if r.long else set()
                else:
                    sz = 0
                    if r.take(1):
                        sz = 14 if not r.take(1) else 17 if not r.take(1) else 20 if not r.take(1) else 64
                    dod = r.take(sz) if sz else 0
                    if sz == 0:
                        seen.add("dod0")
                    elif sz == 64:
                        seen.add("dod64")
                        seen |= {"dod64_neg"} if dod >> 63 else set()
                    else:
                        half = 1 << (sz - 1)
                        seen.add(f"dod{sz}" + ("_top" if dod == half else "_bottom" if dod == half + 1 else ""))
                        if dod > half:
                            dod -= 1 << sz
                    delta = (delta + dod) & MASK64
                if i64(t) + i64(delta) != i64(t + delta):
                    seen.add("ts_wrap")
                t = (t + delta) & MASK64
                if r.take(1):
                    if r.take(1):
                        lead = r.take(5)
                        m = r.take(6)
                        sig = m or 64
                        seen |= {"sig64"} if m == 0 else set()
                        trail = (64 - lead - sig) & 0xFF
                        if lead + sig > 64:
                            seen.add("wide_window")
                        x = r.take(sig)
                        if lead == 31 and sig < 64 and x >> (sig - 1) == 0:
                            seen.add("clamp")
                    elif sig is None:
                        fault = "no_window"
                        break
                    else:
                        seen.add("reuse")
                        x = r.take(sig)
                    if trail < 64:
                        v ^= (x << trail) & MASK64
            ts.append(i64(t))
            vals.append(v)
    except EOFError:
        fault = "overrun"
    except OverflowError:
        fault = "varint"
    if fault:
        seen.add(fault)
    return seen, (ts, vals, fault)


# ---- plans ----------------------------------------------------------------------------------------------------------
def decoder_plan(seed, t_end, step, T, n_random=120, max_len=300):
    """[(name, [chunks of one series])]: every known answer as its own series, then random series cut into chunks of
    1, 2, 7 or 120 samples"""
    rng = np.random.default_rng(seed)
    plan = [(name, [c]) for name, c in known_answers(t_end, step, T)]
    for k in range(n_random):
        ts, bits = random_series(rng, int(rng.integers(1, max_len)), t_end, step, T)
        plan.append((f"random {k}", R.split(ts, bits, int(rng.choice([1, 2, 7, 120])))))
    return plan


def corrupt_plan(seed, t_end, step, T, n_chunks=2000):
    """[(how, chunk, (ts, bits, fault bit))] of some n_chunks corrupted chunks: short random series and the known
    answers, each corrupted every way; the first few cut at every length"""
    rng = np.random.default_rng(seed)
    kat = [c for name, c in known_answers(t_end, step, T) if len(c) < 200]
    out = [(how, c, verdict(c)) for how, c in bad_varints()]
    k = 0
    while len(out) < n_chunks:
        if k < len(kat):
            good = kat[k]
        else:
            good = R.encode(*random_series(rng, int(rng.integers(1, 12)), t_end, step, T))
        other = kat[int(rng.integers(0, len(kat)))] if rng.random() < 0.5 else R.encode(
            *random_series(rng, int(rng.integers(1, 6)), t_end, step, T))
        for how, c in corrupted(rng, good, other, every_cut=k < 8):
            out.append((how, c, verdict(c)))
        k += 1
    return out


def digest(chunks):
    """sha256 of a list of chunks, each with its length: a plan's fingerprint"""
    h = hashlib.sha256()
    for c in chunks:
        h.update(len(c).to_bytes(4, "little") + bytes(c))
    return h.hexdigest()
