"""What gpr_resident_export must write for a ring, built from tests/chunks_ref.py's encoder (TEST INFRASTRUCTURE).

  series_of(plane, head, t_end, step)     per row: (ts list in ms, value bits list) of its present cells, oldest first
  export(plane, head, t_end, step, M)     -> (series_chunks, rows, chunk_bytes, data, n_samples) as the C ABI fills them
  export_native(...)                      the same through tests/cpp/chunks_encode.cpp, for C2-sized rings
  unroll(plane, head)                     the ring's cells oldest first
  restore(batch, T, t_end, step)          the unrolled ring the reference decoder gives back from an export
"""
import numpy as np

import chunks_ref as R

FILL = 0xFFFFFFFF


def unroll(plane, head):
    """plane: [rows][T] uint32 f32 bits -> the same cells oldest first"""
    T = plane.shape[1]
    return plane[:, (head + np.arange(T)) % T]


def _present(cells):
    return (cells & 0x7FFFFFFF) <= 0x7F800000


def flat(plane, head, t_end, step):
    """-> (rows with a sample, offsets u64, ts i64, value bits u64): the present cells as CSR samples"""
    u = unroll(np.asarray(plane, np.uint32), head)
    T = u.shape[1]
    pres = _present(u)
    counts = pres.sum(axis=1)
    rows = np.nonzero(counts)[0].astype(np.uint32)
    ts_col = np.int64(t_end) * 1000 - (T - 1 - np.arange(T, dtype=np.int64)) * np.int64(step) * 1000
    r_idx, j_idx = np.nonzero(pres[rows]) if rows.size else (np.zeros(0, int), np.zeros(0, int))
    ts = ts_col[j_idx]
    bits = u[rows][r_idx, j_idx].view(np.float32).astype(np.float64).view(np.uint64)
    offsets = np.concatenate([[0], np.cumsum(counts[rows])]).astype(np.uint64)
    return rows, offsets, ts, bits


def export(plane, head, t_end, step, M):
    rows, offsets, ts, bits = flat(plane, head, t_end, step)
    series = []
    for s in range(rows.size):
        a, b = int(offsets[s]), int(offsets[s + 1])
        series.append(R.split(ts[a:b].tolist(), [int(x) for x in bits[a:b]], M))
    sc, cb, data = R.batch(series)
    return sc, rows, cb, data, int(offsets[-1])


def export_native(plane, head, t_end, step, M, exe=None):
    rows, offsets, ts, bits = flat(plane, head, t_end, step)
    sc, cb, data = R.encode_native(offsets, ts, bits, M, exe)
    return sc, rows, cb, data, int(offsets[-1])


def restore(sc, rows, cb, data, n_rows, T, t_end, step):
    """the reference decoder's view of an export: [n_rows][T] cells oldest first, FILL where no sample came back"""
    out = np.full((n_rows, T), FILL, np.uint32)
    for s in range(len(rows)):
        for c in range(int(sc[s]), int(sc[s + 1])):
            ts, vals, fault = R.decode(bytes(data[int(cb[c]):int(cb[c + 1])]))
            assert fault is None
            for t, v in zip(ts, vals):
                back, rem = divmod(int(t_end) * 1000 - t, int(step) * 1000)
                assert rem == 0 and 0 <= back < T
                f = np.array([v], np.uint64).view(np.float64).astype(np.float32)
                assert f.astype(np.float64).view(np.uint64)[0] == v   # an f32 exactly
                out[rows[s], T - 1 - back] = f.view(np.uint32)[0]
    return out


def canonical(cells):
    """every NaN as the fill: what a restore gives back"""
    cells = np.array(cells, np.uint32)
    cells[~_present(cells)] = FILL
    return cells
