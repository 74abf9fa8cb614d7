"""CPU: the XOR chunk reference of tests/chunks_ref.py against chunks written out bit by bit from the format
(include/gpr.h, Prometheus tsdb/chunkenc/xor.go), then encoder and decoder round-tripped on random series.  The
device decoder (gpu-pruner_b200/csrc/gpr_chunks.cuh) is held to this reference by tests/test_chunks_emul.py and
tests/test_gpu_chunks.py."""
import struct

import numpy as np
import pytest

import chunks_ref as R
from chunks_ref import BitWriter


def _two(t0, v0):
    """the first sample of a chunk: zigzag varint timestamp, 64 raw bits"""
    return BitWriter().varint(t0).put(R.f2b(v0), 64)


def test_empty_one_and_two_sample_chunks():
    assert R.encode([], []) == b"\x00\x00"
    assert R.decode(b"\x00\x00") == ([], [], None)
    # t = 1000 ms -> zigzag 2000 -> uvarint d0 0f; 1.0 = 3ff0000000000000
    one = bytes.fromhex("0001" "d00f" "3ff0000000000000")
    assert R.encode([1000], [1.0]) == one
    assert R.decode(one) == ([1000], [R.f2b(1.0)], None)
    # + 15 ms (uvarint 0f), the same value ('0'), padded to a byte
    two = bytes.fromhex("0002" "d00f" "3ff0000000000000" "0f" "00")
    assert R.encode([1000, 1015], [1.0, 1.0]) == two
    assert R.decode(two) == ([1000, 1015], [R.f2b(1.0)] * 2, None)
    # bytes after the last sample are not read
    assert R.decode(two + b"\xff\xff") == R.decode(two)


def test_negative_first_timestamp():
    # -1 -> zigzag 1; -1000 -> zigzag 1999 -> cf 0f
    assert R.encode([-1], [0.0])[2:3] == b"\x01"
    c = bytes.fromhex("0001" "cf0f" "0000000000000000")
    assert R.encode([-1000], [0.0]) == c
    assert R.decode(c) == ([-1000], [0], None)
    ts = [-5000, -4000, -2500, 10]
    assert R.decode(R.encode(ts, [1.0] * 4))[0] == ts


# (dod, prefix, payload bits): both ends of every bucket and the first value past each end
DOD_CASES = [
    (0, "0", 0), (1, "10", 14), (-1, "10", 14),
    (8192, "10", 14), (-8191, "10", 14), (8193, "110", 17), (-8192, "110", 17),
    (65536, "110", 17), (-65535, "110", 17), (65537, "1110", 20), (-65536, "1110", 20),
    (524288, "1110", 20), (-524287, "1110", 20), (524289, "1111", 64), (-524288, "1111", 64),
    (1 << 40, "1111", 64), (-(1 << 40), "1111", 64),
]


@pytest.mark.parametrize("dod,prefix,sz", DOD_CASES)
def test_every_dod_bucket_at_both_ends(dod, prefix, sz):
    """the encoder picks the bucket Prometheus picks, and a hand-written chunk of that bucket decodes to dod: a
    payload of exactly 2^(sz-1) is positive, one above it negative"""
    t0, d1 = 1_700_000_000_000, 15_000
    ts = [t0, t0 + d1, t0 + 2 * d1 + dod]
    w = _two(t0, 5.0).uvarint(d1).bit(0).string(prefix)
    if sz:
        w.put(dod & ((1 << sz) - 1), sz)
    w.bit(0)
    hand = w.chunk(3)
    assert R.encode(ts, [5.0] * 3) == hand
    assert R.decode(hand) == (ts, [R.f2b(5.0)] * 3, None)


def test_dod_payload_edges_by_hand():
    """payloads written directly: 0b10 0000 0000 0000 (2^13) is +8192, 0b10 0000 0000 0001 is -8191, all ones -1;
    the same edges for 17 and 20 bits"""
    for prefix, sz in (("10", 14), ("110", 17), ("1110", 20)):
        half = 1 << (sz - 1)
        for payload, want in ((half, half), (half + 1, half + 1 - (1 << sz)), ((1 << sz) - 1, -1), (1, 1)):
            c = _two(0, 1.0).uvarint(100).bit(0).string(prefix).put(payload, sz).bit(0).chunk(3)
            ts, _, fault = R.decode(c)
            assert fault is None and ts[2] - ts[1] - 100 == want, (sz, payload)


def test_64_bit_dod():
    dod = -(1 << 62) + 12345
    c = _two(0, 1.0).uvarint(10).bit(0).string("1111").put(dod & R.MASK64, 64).bit(0).chunk(3)
    ts, _, fault = R.decode(c)
    assert fault is None and ts == [0, 10, 20 + dod]


def test_leading_zeros_clamp_at_31():
    """xor 0x0000_0000_00f0_0000 has 40 leading zeros: written as 31, with 13 significant bits"""
    v1 = 0x0000000000F00000
    c = R.encode([0, 1], [0, v1])
    hand = BitWriter().varint(0).put(0, 64).uvarint(1).string("11" "11111" "001101").put(v1 >> 20, 13).chunk(2)
    assert c == hand
    assert R.decode(hand)[1] == [0, v1]


def test_64_significant_bits_written_as_0():
    v1 = 0x8000000000000001
    hand = BitWriter().varint(0).put(0, 64).uvarint(1).string("11" "00000" "000000").put(v1, 64).chunk(2)
    assert R.encode([0, 1], [0, v1]) == hand
    assert R.decode(hand) == ([0, 1], [0, v1], None)


def test_window_reuse_and_new_window():
    """v1 opens a window (lead 12, trail 40); v2's xor fits it: '10' + 12 bits; v3's xor has fewer trailing zeros: a
    new window '11'"""
    v0 = 0x4059000000000000                       # 100.0
    x1 = 0x000ABC0000000000                       # lead 12, trail 42 -> window lead 12, sig 10
    x2 = 0x0008040000000000                       # lead 12, trail 42: fits
    x3 = 0x0000000000000F00                       # trail 8: new window, lead 31 (clamped from 52)
    vals = [v0, v0 ^ x1, v0 ^ x1 ^ x2, v0 ^ x1 ^ x2 ^ x3]
    hand = (BitWriter().varint(0).put(v0, 64).uvarint(1000)
            .string("11").put(12, 5).put(10, 6).put(x1 >> 42, 10)
            .bit(0).string("10").put(x2 >> 42, 10)
            .bit(0).string("11").put(31, 5).put(25, 6).put(x3 >> 8, 25)
            .chunk(4))
    assert R.encode([0, 1000, 2000, 3000], vals) == hand
    assert R.decode(hand) == ([0, 1000, 2000, 3000], vals, None)


def test_special_values_keep_their_bits():
    special = [R.STALE_NAN_BITS, R.f2b(float("inf")), R.f2b(float("-inf")), R.f2b(-0.0), R.f2b(0.0),
               0x7FF8000000000001, R.f2b(5e-324), R.f2b(-1.5), R.STALE_NAN_BITS]
    ts = list(range(0, 15_000 * len(special), 15_000))
    ts_d, vals, fault = R.decode(R.encode(ts, special))
    assert fault is None and ts_d == ts and vals == special


def test_65535_samples_in_one_chunk():
    rng = np.random.default_rng(1)
    n = 65535
    ts = (1_700_000_000_000 + np.cumsum(rng.integers(14_000, 16_000, n))).tolist()
    vals = rng.integers(0, 101, n).astype(float).tolist()
    c = R.encode(ts, vals)
    assert c[:2] == b"\xff\xff"
    ts_d, v_d, fault = R.decode(c)
    assert fault is None and ts_d == ts and v_d == [R.f2b(v) for v in vals]


def test_malformed_chunks():
    good = R.encode([0, 1000, 2000], [1.0, 2.0, 2.0])
    assert R.decode(good)[2] is None
    assert R.decode(b"")[2] == "short" and R.decode(b"\x00")[2] == "short"
    for cut in range(2, len(good) - 1):
        # a chunk that ends mid-sample
        assert R.decode(good[:cut])[2] == "overrun", cut
    assert R.decode(struct.pack(">H", 40) + good[2:])[2] == "overrun"   # a count larger than the stream
    reuse = BitWriter().varint(0).put(0, 64).uvarint(1).string("10").put(0, 8).chunk(2)
    assert R.decode(reuse)[2] == "no_window"
    long = BitWriter().put(0xFFFFFFFFFFFFFFFFFFFF, 80).byte(0x01).put(0, 64).chunk(1)
    assert R.decode(long)[2] == "varint"
    tenth = BitWriter().put(0xFFFFFFFFFFFFFFFFFF, 72).byte(0x02).put(0, 64).chunk(1)
    assert R.decode(tenth)[2] == "varint"


def test_round_trip_random_series():
    rng = np.random.default_rng(2)
    for k in range(200):
        n = int(rng.integers(1, 300))
        step = int(rng.choice([1000, 15_000, 60_000]))
        jitter = rng.integers(-int(rng.choice([0, 5, 3000, 600_000])), 1 + int(rng.choice([0, 5, 3000, 600_000])), n)
        ts = (int(rng.integers(-10**13, 10**13)) + np.arange(n) * step + jitter).tolist()
        kind = k % 4
        if kind == 0:
            vals = rng.integers(0, 101, n).astype(float)
        elif kind == 1:
            vals = rng.random(n)
        elif kind == 2:
            vals = rng.choice([0.0, -0.0, np.inf, -np.inf, np.nan, 150.0, 149.999999, 1e-300, -3.5], n)
        else:
            vals = rng.integers(0, 1 << 64, n, dtype=np.uint64).view(np.float64)
        bits = vals.view(np.uint64).tolist()
        if kind == 2:
            bits = [R.STALE_NAN_BITS if rng.random() < 0.1 else b for b in bits]
        for c in R.split(ts, bits, int(rng.choice([1, 2, 120, 300]))):
            got_t, got_v, fault = R.decode(c)
            assert fault is None
        dec_t, dec_v = [], []
        for c in R.split(ts, bits):
            t, v, _ = R.decode(c)
            dec_t += t
            dec_v += v
        assert dec_t == ts and dec_v == bits, k
