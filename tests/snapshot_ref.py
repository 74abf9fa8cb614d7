"""A reader of daemon mode's snapshot file, written from DESIGN.md §8i (TEST INFRASTRUCTURE): the binary's writer and
reader are gpu-pruner_b200/host/snapshot.cpp; this one is independent of them.

read(blob) -> dict with the fingerprint, t_end, the session, the planes (gpr_chunk_export's CSR as numpy arrays, ready
for tests/chunks_ref.py) and `sections`: [(name, begin, end)] in file order.  Raises ValueError on anything malformed."""
import struct

import numpy as np

MAGIC = b"GPRSNAP\0"
VERSION = 1


def crc32c(data, crc=0):
    """bitwise CRC32C (Castagnoli, reflected, init and xor-out 0xFFFFFFFF)"""
    c = crc ^ 0xFFFFFFFF
    for b in data:
        c ^= b
        for _ in range(8):
            c = (c >> 1) ^ (0x82F63B78 if c & 1 else 0)
    return c ^ 0xFFFFFFFF


def crc32c_fast(data):
    """the same through a byte table (for files of megabytes)"""
    tab = []
    for i in range(256):
        c = i
        for _ in range(8):
            c = (c >> 1) ^ (0x82F63B78 if c & 1 else 0)
        tab.append(c)
    c = 0xFFFFFFFF
    for b in bytes(data):
        c = tab[(c ^ b) & 0xFF] ^ (c >> 8)
    return c ^ 0xFFFFFFFF


class _In:
    def __init__(self, b, end):
        self.b, self.at, self.end = b, 0, end

    def take(self, n):
        if n < 0 or self.at + n > self.end:
            raise ValueError("truncated at %d (+%d)" % (self.at, n))
        v = self.b[self.at:self.at + n]
        self.at += n
        return v

    def u(self, fmt):
        return struct.unpack("<" + fmt, self.take(struct.calcsize("<" + fmt)))[0]

    def s(self):
        return self.take(self.u("I")).decode()

    def pad8(self):
        self.take((8 - self.at % 8) % 8)

    def arr(self, dtype, n):
        return np.frombuffer(self.take(n * np.dtype(dtype).itemsize), dtype=dtype)


def read(blob, check_crc=True):
    blob = bytes(blob)
    if blob[:8] != MAGIC:
        raise ValueError("magic")
    if struct.unpack_from("<I", blob, 8)[0] != VERSION:
        raise ValueError("version")
    total, crc = struct.unpack_from("<QI", blob, len(blob) - 12)
    if total != len(blob):
        raise ValueError("length")
    if check_crc and crc32c_fast(blob[:-4]) != crc:
        raise ValueError("crc")
    r = _In(blob, len(blob) - 12)
    out, sections = {}, []
    r.take(16)
    flags = struct.unpack_from("<I", blob, 12)[0]
    out["power"] = bool(flags & 1)
    sections.append(("header", 0, 16))
    b0 = r.at
    out["span"], out["step"], out["T"], out["pods_cap"], out["G"], _ = struct.unpack("<qqIIII", r.take(32))
    out["power_threshold"] = r.u("d")
    out["selectors"] = [r.s() for _ in range(3)]
    sections.append(("fingerprint", b0, r.at))
    b0 = r.at
    out["t_end"] = r.u("q")
    sections.append(("t_end", b0, r.at))
    b0 = r.at
    pods = []
    for _ in range(r.u("I")):
        pod = {"name": r.s(), "ns": r.s(), "power_slots": r.u("I"), "has_groups": r.u("B")}
        pod["slots"] = [{"hostname": r.s(), "container": r.s(), "gpu": r.s(), "model": r.s(), "node_type": r.s(),
                         "from_prof": r.u("B"), "group": r.u("I")} for _ in range(r.u("I"))]
        pods.append(pod)
    out["pods"] = pods
    out["known"] = [struct.unpack("<QQIII", r.take(28)) for _ in range(r.u("Q"))]
    out["power_keys"] = [list(r.arr("<u8", r.u("I"))) for _ in pods]
    sigs = []
    for _ in range(r.u("I")):
        pod, grp, n = struct.unpack("<III", r.take(12))
        sigs.append(((pod, grp), [r.s() for _ in range(n)]))
    out["prof_sigs"] = sigs
    n = r.u("I")
    out["prof_rows"] = [tuple(x) for x in r.arr("<u4", 2 * n).reshape(-1, 2)]
    r.pad8()
    sections.append(("session", b0, r.at))
    planes = []
    for k in range(2 if out["power"] else 1):
        b0 = r.at
        ns, nc, nb = struct.unpack("<QQQ", r.take(24))
        p = {"series_chunks": r.arr("<u8", ns + 1), "rows": r.arr("<u4", ns)}
        r.pad8()
        p["chunk_bytes_at"] = r.at
        p["chunk_bytes"] = r.arr("<u8", nc + 1)
        p["data_at"] = r.at
        p["data"] = r.arr("u1", nb)
        r.pad8()
        planes.append(p)
        sections.append(("plane%d" % k, b0, r.at))
    if r.at != r.end:
        raise ValueError("bytes after the planes")
    sections.append(("trailer", r.end, len(blob)))
    out["planes"], out["sections"] = planes, sections
    return out


def reseal(blob):
    """the same bytes with the trailer's CRC recomputed (a corruption the checksum does not see)"""
    blob = bytearray(blob)
    struct.pack_into("<I", blob, len(blob) - 4, crc32c_fast(blob[:-4]))
    return bytes(blob)
