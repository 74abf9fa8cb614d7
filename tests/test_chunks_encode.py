"""CPU: the C++ XOR encoder of tests/cpp/chunks_encode.cpp, which the GPU tests and tools/chunks_bench.py use for
C2-sized batches, writes the same bytes as the Python reference encoder of tests/chunks_ref.py."""
import numpy as np

import chunks_ref as R


def test_native_encoder_matches_the_reference():
    rng = np.random.default_rng(3)
    lengths = rng.integers(0, 400, 60)
    offsets = np.concatenate([[0], np.cumsum(lengths)]).astype(np.uint64)
    n = int(offsets[-1])
    ts = np.cumsum(rng.choice([15_000, 15_001, 14_000, 1 << 21, -(1 << 21)], n)) + int(rng.integers(-10**12, 10**12))
    v = rng.integers(0, 101, n).astype(np.float64)
    ratio = rng.random(n) < 0.2
    v[ratio] = rng.random(int(ratio.sum()))
    bits = v.view(np.uint64).copy()
    bits[rng.random(n) < 0.05] = R.STALE_NAN_BITS
    wild = rng.random(n) < 0.05
    bits[wild] = rng.integers(0, 1 << 64, int(wild.sum()), dtype=np.uint64)
    for per in (1, 7, 120):
        sc, cb, data = R.encode_native(offsets, ts, bits, per)
        want = [R.split(ts[int(offsets[s]):int(offsets[s + 1])].tolist(), bits[int(offsets[s]):int(offsets[s + 1])].tolist(),
                        per) for s in range(len(lengths))]
        w_sc, w_cb, w_data = R.batch(want)
        assert np.array_equal(sc, w_sc) and np.array_equal(cb, w_cb) and np.array_equal(data, w_data), per
