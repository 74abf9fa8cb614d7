"""Prometheus XOR chunks (tsdb/chunkenc/xor.go) in plain Python, written from the format as include/gpr.h and
gpu-pruner_b200/csrc/gpr_chunks.cuh state it: the reference the tests hold gpr_chunks_scatter to.

  encode(ts, values)  -> bytes     the chunk Prometheus' appender writes: its delta-of-delta bucket choice, its XOR
                                   window reuse rule and its clamp of leading zeros to 31
  decode(chunk)       -> (ts, values, fault)   the decoder; fault is None or one of FAULTS
  BitWriter                        hand-written chunks, bit by bit, for the known-answer tests
  batch(series)                    CSR arrays (series_chunks, chunk_bytes, data) of a list of chunk lists
  encode_native(...)               the same encoder in C++ (tests/cpp/chunks_encode.cpp), for C2-sized batches
"""
import os
import struct
import subprocess
import tempfile

import numpy as np

MASK64 = (1 << 64) - 1
STALE_NAN_BITS = 0x7FF0000000000002          # Prometheus' staleness marker
FAULTS = ("short", "overrun", "no_window", "varint")


def f2b(x):
    return struct.unpack("<Q", struct.pack("<d", x))[0]


def b2f(b):
    return struct.unpack("<d", struct.pack("<Q", b & MASK64))[0]


class BitWriter:
    """An MSB-first bit stream after the 2-byte sample count (the count is set by header())."""

    def __init__(self):
        self.bits = []

    def bit(self, b):
        self.bits.append(1 if b else 0)
        return self

    def put(self, value, n):
        for k in range(n - 1, -1, -1):
            self.bits.append((value >> k) & 1)
        return self

    def string(self, s):
        """bits written as a string of '0' / '1' (spaces ignored)"""
        for ch in s.replace(" ", ""):
            self.bits.append(int(ch))
        return self

    def byte(self, b):
        return self.put(b & 0xFF, 8)

    def uvarint(self, x):
        x &= MASK64
        while x >= 0x80:
            self.byte((x & 0x7F) | 0x80)
            x >>= 7
        return self.byte(x)

    def varint(self, x):
        return self.uvarint(((x << 1) ^ (x >> 63)) & MASK64)   # zigzag, as binary.PutVarint

    def chunk(self, count):
        bits = self.bits + [0] * (-len(self.bits) % 8)
        body = bytes(int("".join(map(str, bits[i:i + 8])), 2) for i in range(0, len(bits), 8))
        return struct.pack(">H", count) + body


class _Reader:
    def __init__(self, data):
        self.data, self.pos = data, 0        # pos in bits

    def take(self, n):
        if self.pos + n > 8 * len(self.data):
            raise EOFError
        v = 0
        for _ in range(n):
            v = (v << 1) | ((self.data[self.pos >> 3] >> (7 - (self.pos & 7))) & 1)
            self.pos += 1
        return v

    def uvarint(self):
        x, s = 0, 0
        for i in range(10):
            b = self.take(8)
            if b < 0x80:
                if i == 9 and b > 1:
                    raise OverflowError
                return x | (b << s)
            x |= (b & 0x7F) << s
            s += 7
        raise OverflowError


def decode(chunk):
    """-> (ts list of int64 ms, value list of float64 bit patterns, fault or None): the samples before a fault"""
    chunk = bytes(chunk)
    if len(chunk) < 2:
        return [], [], "short"
    count = struct.unpack(">H", chunk[:2])[0]
    r = _Reader(chunk[2:])
    ts, vals = [], []
    t = delta = v = 0
    sig = trail = None
    try:
        for i in range(count):
            if i == 0:
                u = r.uvarint()
                t = (u >> 1) ^ (-(u & 1) & MASK64)
                v = r.take(64)
            else:
                if i == 1:
                    delta = r.uvarint()
                else:
                    sz = 0
                    if r.take(1):
                        sz = 14 if not r.take(1) else 17 if not r.take(1) else 20 if not r.take(1) else 64
                    if sz:
                        dod = r.take(sz)
                        if sz < 64 and dod > (1 << (sz - 1)):
                            dod -= 1 << sz
                        delta = (delta + dod) & MASK64
                t = (t + delta) & MASK64
                if r.take(1):
                    if r.take(1):
                        lead = r.take(5)
                        sig = r.take(6) or 64
                        trail = (64 - lead - sig) & 0xFF     # Go's uint8 arithmetic
                    elif sig is None:
                        return ts, vals, "no_window"
                    x = r.take(sig)
                    if trail < 64:
                        v ^= (x << trail) & MASK64
            ts.append(t - (1 << 64) if t >> 63 else t)
            vals.append(v)
    except EOFError:
        return ts, vals, "overrun"
    except OverflowError:
        return ts, vals, "varint"
    return ts, vals, None


def _bit_range(x, n):
    return -((1 << (n - 1)) - 1) <= x <= (1 << (n - 1))


def encode(ts, values):
    """the chunk Prometheus' XOR appender writes for these samples (ts int ms, values float or bit patterns as int)"""
    w = BitWriter()
    t_prev = delta_prev = 0
    v_prev = 0
    lead = 0xFF
    trail = 0
    for i, (t, v) in enumerate(zip(ts, values)):
        t = int(t)
        vb = v if isinstance(v, (int, np.integer)) and not isinstance(v, bool) else f2b(float(v))
        vb = int(vb) & MASK64
        if i == 0:
            w.varint(t)
            w.put(vb, 64)
        else:
            delta = (t - t_prev) & MASK64
            if i == 1:
                w.uvarint(delta)
            else:
                dod = (delta - delta_prev) & MASK64
                dod = dod - (1 << 64) if dod >> 63 else dod
                if dod == 0:
                    w.bit(0)
                elif _bit_range(dod, 14):
                    w.put(0b10, 2).put(dod & 0x3FFF, 14)
                elif _bit_range(dod, 17):
                    w.put(0b110, 3).put(dod & 0x1FFFF, 17)
                elif _bit_range(dod, 20):
                    w.put(0b1110, 4).put(dod & 0xFFFFF, 20)
                else:
                    w.put(0b1111, 4).put(dod & MASK64, 64)
            delta_prev = delta
            x = vb ^ v_prev
            if x == 0:
                w.bit(0)
            else:
                w.bit(1)
                new_lead = min(64 - x.bit_length(), 31)
                new_trail = (x & -x).bit_length() - 1
                if lead != 0xFF and new_lead >= lead and new_trail >= trail:
                    w.bit(0).put(x >> trail, 64 - lead - trail)
                else:
                    lead, trail = new_lead, new_trail
                    sig = 64 - lead - trail
                    w.bit(1).put(lead, 5).put(sig & 63, 6).put(x >> trail, sig)
        t_prev, v_prev = t, vb
    return w.chunk(len(ts))


def batch(series):
    """series: a list (one per series) of lists of chunk bytes -> (series_chunks u64, chunk_bytes u64, data u8)"""
    chunks = [c for s in series for c in s]
    series_chunks = np.concatenate([[0], np.cumsum([len(s) for s in series])]).astype(np.uint64)
    chunk_bytes = np.concatenate([[0], np.cumsum([len(c) for c in chunks])]).astype(np.uint64)
    data = np.frombuffer(b"".join(chunks), np.uint8).copy() if chunks else np.zeros(0, np.uint8)
    return series_chunks, chunk_bytes, data


def split(ts, values, per_chunk=120):
    """one series' samples as chunks of at most per_chunk samples, as Prometheus cuts them"""
    return [encode(ts[i:i + per_chunk], values[i:i + per_chunk]) for i in range(0, len(ts), per_chunk)]


def build_native(d):
    """the C++ encoder (tests/cpp/chunks_encode.cpp) built with g++ into directory d -> its path"""
    src = os.path.join(os.path.dirname(os.path.abspath(__file__)), "cpp", "chunks_encode.cpp")
    exe = os.path.join(d, "chunks_encode")
    subprocess.run(["g++", "-O2", "-std=c++17", "-Wall", "-Werror", src, "-o", exe], check=True,
                   capture_output=True, text=True)
    return exe


def encode_native(offsets, ts, bits, per_chunk=120, exe=None):
    """CSR samples (offsets u64, ts i64 ms, bits u64) -> (series_chunks, chunk_bytes, data) by the C++ encoder (`exe`
    from build_native, or built with g++ into a temporary directory)"""
    with tempfile.TemporaryDirectory() as d:
        exe = exe or build_native(d)
        np.ascontiguousarray(offsets, np.uint64).tofile(os.path.join(d, "offsets.u64"))
        np.ascontiguousarray(ts, np.int64).tofile(os.path.join(d, "ts.i64"))
        np.ascontiguousarray(bits, np.uint64).tofile(os.path.join(d, "bits.u64"))
        subprocess.run([exe, d, str(per_chunk)], check=True)
        return (np.fromfile(os.path.join(d, "series_chunks.u64"), np.uint64),
                np.fromfile(os.path.join(d, "chunk_bytes.u64"), np.uint64),
                np.fromfile(os.path.join(d, "data.u8"), np.uint8))
