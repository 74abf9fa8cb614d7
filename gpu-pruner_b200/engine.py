"""Thin object wrapper over the C ABI (include/gpr.h) for Python callers, tests and bench.py.

The product is libgpr.so; this file only marshals arguments.  It mirrors the seam of the
reference at ``gpu-pruner/src/main.rs:397-437`` ("run the aggregation, get
back the candidate set"): :meth:`IdleEngine.decide` takes the window matrix and returns the
packed decision bitmap plus the ``QueryResponse``-style counts (``lib.rs:131-134``).

There is no CPU fallback anywhere in this module: if libgpr.so or a CUDA device is missing the
constructor raises.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass
from typing import Optional

import numpy as np

from . import ffi

_KERNELS = {"auto": ffi.GPR_KERNEL_AUTO, "ldg": ffi.GPR_KERNEL_LDG, "tma": ffi.GPR_KERNEL_TMA}


class GprError(RuntimeError):
    """Non-zero status from libgpr.so (the Rust wrapper would turn this into ``anyhow!``,
    feeding the failure counter at main.rs:310-321)."""

    def __init__(self, code: int, message: str):
        super().__init__(f"{ffi.ERROR_NAMES.get(code, code)}: {message}")
        self.code = code
        self.message = message


@dataclass
class Decision:
    n_pods: int
    decision_bits: np.ndarray            # uint32[ceil(P/32)] (x world with a communicator)
    candidate_bits: Optional[np.ndarray]
    series_max: Optional[np.ndarray]     # float32[P, G]
    n_series: int                        # QueryResponse.num_pods (series, pre-dedup; main.rs:418)
    n_candidates: int
    n_decisions: int
    kernel_ms: float
    veto_bits: Optional[np.ndarray] = None   # uint32[ceil(P/32)]: pods vetoed by the power clause (this rank's pods)
    idle_slots: Optional[np.ndarray] = None  # uint32[P, ceil(G/32)]: slots that start an idle element

    def pods(self, bits: Optional[np.ndarray] = None) -> np.ndarray:
        """Indices of set bits (the idle-pod set), ascending."""
        w = self.decision_bits if bits is None else bits
        flat = np.unpackbits(np.ascontiguousarray(w, dtype="<u4").view(np.uint8), bitorder="little")
        return np.flatnonzero(flat)


def to_biased_u8(util: np.ndarray) -> np.ndarray:
    """f32 window (NaN = no sample) -> GPR_FMT_U8B bytes (0 = no sample, b = value + 1).  Raises if a
    sample is not an integer in 0..254 (DCGM_FI_DEV_GPU_UTIL is an integer percentage)."""
    util = np.asarray(util, dtype=np.float32)
    present = ~np.isnan(util)
    v = np.where(present, util, 0.0)
    if not np.all((v >= 0) & (v <= 254) & (v == np.floor(v))):
        raise ValueError("window is not representable in GPR_FMT_U8B (integers 0..254 or NaN)")
    return np.where(present, v + 1, 0).astype(np.uint8)


def from_biased_u8(b: np.ndarray) -> np.ndarray:
    b = np.asarray(b, dtype=np.uint8)
    return np.where(b == 0, np.float32("nan"), b.astype(np.float32) - 1).astype(np.float32)


def _ptr(x) -> Optional[int]:
    """numpy array / torch tensor / int address / None -> address."""
    if x is None:
        return None
    if isinstance(x, int):
        return x
    if isinstance(x, np.ndarray):
        return x.ctypes.data
    if hasattr(x, "data_ptr"):
        return x.data_ptr()
    raise TypeError(f"cannot take the address of {type(x)!r}")


def _n_series(n_series: Optional[int], rows, mem_kind: int) -> int:
    """a batch's series count: as given, or for host arrays the length of ``rows``"""
    if n_series is not None:
        return int(n_series)
    if mem_kind != ffi.GPR_MEM_HOST:
        raise ValueError("n_series is required for device arrays")
    return rows.size


def _text_grid(t_end: int, step: int, T: int, n_rows: int = 0, window_seconds: Optional[int] = None,
               power_threshold: Optional[float] = 0.0, fill: bool = False, resident: bool = False) -> ffi.gpr_text_grid:
    """the time axis and destination of a merge or an export; ``window_seconds`` defaults to ``T * step``"""
    g = ffi.gpr_text_grid()
    g.struct_size = C.sizeof(ffi.gpr_text_grid)
    g.flags = (ffi.GPR_TEXT_FILL if fill and not resident else 0) | (ffi.GPR_TEXT_RESIDENT if resident else 0)
    g.t_end, g.step = int(t_end), int(step)
    g.window_seconds = int(T) * int(step) if window_seconds is None else int(window_seconds)
    g.n_samples, g.n_rows = int(T), int(n_rows)
    g.power_threshold = 0.0 if power_threshold is None else float(power_threshold)
    return g


class IdleEngine:
    """One context = one GPU.  Not re-entrant (one call at a time), thread-agnostic."""

    def __init__(self, device: int = 0, max_pods: int = 0, max_gpus: int = 0, max_samples: int = 0,
                 power_plane: bool = False, kernel: str = "auto", stream: Optional[int] = None):
        self._lib = ffi.load()
        cfg = ffi.gpr_config()
        cfg.struct_size = C.sizeof(ffi.gpr_config)
        cfg.device = device
        cfg.max_pods, cfg.max_gpus, cfg.max_samples = max_pods, max_gpus, max_samples
        cfg.flags = ffi.GPR_F_POWER_PLANE if power_plane else 0
        cfg.kernel_variant = _KERNELS[kernel]
        cfg.stream = stream
        h = C.c_void_p()
        rc = self._lib.gpr_create(C.byref(cfg), C.byref(h))
        if rc != ffi.GPR_OK:
            raise GprError(rc, (self._lib.gpr_last_error(None) or b"").decode())
        self._h = h
        self.device = device
        self._keep = []  # result structs / arrays referenced by outstanding async calls
        self._host_arrays = []  # pinned allocations handed out by host_array(), freed in close()

    # ---- plumbing ---------------------------------------------------------------------------
    def _check(self, rc: int):
        if rc != ffi.GPR_OK:
            raise GprError(rc, (self._lib.gpr_last_error(self._h) or b"").decode())

    def close(self):
        if getattr(self, "_h", None):
            for ptr in getattr(self, "_host_arrays", []):
                self._lib.gpr_host_free(self._h, ptr)
            self._host_arrays = []
            self._lib.gpr_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    @property
    def handle(self):
        return self._h

    # ---- hot path ---------------------------------------------------------------------------
    def _window(self, util, power, eligible, created_ts, cutoff_ts, P, G, T, row_stride,
                power_threshold, mem_kind, util_format: int = ffi.GPR_FMT_F32, groups=None) -> ffi.gpr_window:
        w = ffi.gpr_window()
        w.groups = _ptr(groups)
        w.util_format = util_format
        w.struct_size = C.sizeof(ffi.gpr_window)
        w.mem_kind = mem_kind
        w.util, w.power = _ptr(util), _ptr(power)
        w.eligible, w.created_ts = _ptr(eligible), _ptr(created_ts)
        w.cutoff_ts = int(cutoff_ts)
        w.n_pods, w.n_gpus, w.n_samples = P, G, T
        w.row_stride = row_stride
        w.power_threshold = float(power_threshold) if power_threshold is not None else 0.0
        return w

    def decide(self, util: np.ndarray, power: Optional[np.ndarray] = None,
               eligible: Optional[np.ndarray] = None, created_ts: Optional[np.ndarray] = None,
               cutoff_ts: int = 0, power_threshold: Optional[float] = 0.0,
               want_candidates: bool = True, want_series_max: bool = False,
               world: int = 1, want_veto: bool = False, groups: Optional[np.ndarray] = None,
               want_idle_slots: bool = False) -> Decision:
        """Blocking decision over a HOST window ``util[P, G, T]`` (float32, NaN = no sample; or
        uint8 in the biased byte format GPR_FMT_U8B, see :func:`to_biased_u8`).  ``groups``: the
        ``sum by`` group table ``uint32[P, G]`` (include/gpr.h, gpr_window.groups)."""
        fmt = ffi.GPR_FMT_U8B if getattr(util, "dtype", None) == np.uint8 else ffi.GPR_FMT_F32
        util = np.ascontiguousarray(util, dtype=np.uint8 if fmt else np.float32)
        if util.ndim != 3:
            raise ValueError("util must be [pods, gpus, samples]")
        P, G, T = util.shape
        if power is not None:
            power = np.ascontiguousarray(power, dtype=np.float32)
            if power.shape != util.shape:
                raise ValueError("power must have util's shape")
        if eligible is not None:
            eligible = np.ascontiguousarray(eligible, dtype=np.uint8)
        if created_ts is not None:
            created_ts = np.ascontiguousarray(created_ts, dtype=np.int64)
        if groups is not None:
            groups = np.ascontiguousarray(groups, dtype=np.uint32)
            if groups.shape != (P, G):
                raise ValueError("groups must be [pods, gpus]")
        w = self._window(util, power, eligible, created_ts, cutoff_ts, P, G, T, 0,
                         power_threshold, ffi.GPR_MEM_HOST, fmt, groups)
        W = (P + 31) // 32 * world
        islots = np.zeros((max(P, 1), (G + 31) // 32), dtype=np.uint32) if want_idle_slots else None
        dbits = np.zeros(max(W, 1), dtype=np.uint32)
        cbits = np.zeros(max(W, 1), dtype=np.uint32) if want_candidates else None
        smax = np.zeros((P, G), dtype=np.float32) if want_series_max else None
        vbits = np.zeros(max((P + 31) // 32, 1), dtype=np.uint32) if want_veto else None
        r = ffi.gpr_result()
        r.struct_size = C.sizeof(ffi.gpr_result)
        r.out_mem_kind = ffi.GPR_MEM_HOST
        r.decision_bits, r.candidate_bits, r.series_max = _ptr(dbits), _ptr(cbits), _ptr(smax)
        r.veto_bits = _ptr(vbits)
        r.idle_slots = _ptr(islots)
        self._check(self._lib.gpr_decide(self._h, C.byref(w), C.byref(r)))
        d = Decision(P, dbits[:W], None if cbits is None else cbits[:W], smax, r.n_series,
                     r.n_candidates, r.n_decisions, r.kernel_ms)
        d.veto_bits = None if vbits is None else vbits[:(P + 31) // 32]
        d.idle_slots = None if islots is None else islots[:P]
        return d

    def decide_ptr(self, util, P: int, G: int, T: int, decision_bits, *, power=None, eligible=None,
                   created_ts=None, cutoff_ts: int = 0, power_threshold: Optional[float] = 0.0,
                   candidate_bits=None, series_max=None, veto_bits=None, row_stride: int = 0,
                   in_kind: int = ffi.GPR_MEM_DEVICE, out_kind: int = ffi.GPR_MEM_DEVICE,
                   blocking: bool = True, resident: bool = False,
                   util_format: int = ffi.GPR_FMT_F32, groups=None, idle_slots=None) -> ffi.gpr_result:
        """Raw-pointer form (device tensors, pinned host buffers).  With ``blocking=False`` the
        call only enqueues; counters in the returned struct are valid after :meth:`sync`.
        ``groups`` (where ``in_kind`` says) and ``idle_slots`` (where ``out_kind`` says): see
        include/gpr.h; ``resident=True`` is gpr_decide_resident."""
        w = self._window(util, power, eligible, created_ts, cutoff_ts, P, G, T, row_stride,
                         power_threshold, in_kind, util_format, groups)
        r = ffi.gpr_result()
        r.struct_size = C.sizeof(ffi.gpr_result)
        r.out_mem_kind = out_kind
        r.decision_bits, r.candidate_bits, r.series_max = (_ptr(decision_bits), _ptr(candidate_bits),
                                                           _ptr(series_max))
        r.veto_bits = _ptr(veto_bits)
        r.idle_slots = _ptr(idle_slots)
        if resident:
            self._check(self._lib.gpr_decide_resident(self._h, C.byref(w), C.byref(r)))
        elif blocking:
            self._check(self._lib.gpr_decide(self._h, C.byref(w), C.byref(r)))
        else:
            self._keep.append((w, r))
            self._check(self._lib.gpr_decide_async(self._h, C.byref(w), C.byref(r)))
        return r

    def make_batch(self, calls):
        """Pre-marshal a list of decide_ptr-style keyword dicts into contiguous gpr_window /
        gpr_result arrays for :meth:`decide_batch_async` (build once, enqueue many times)."""
        n = len(calls)
        wins = (ffi.gpr_window * n)()
        ress = (ffi.gpr_result * n)()
        for i, kw in enumerate(calls):
            w = self._window(kw["util"], kw.get("power"), kw.get("eligible"), kw.get("created_ts"),
                             kw.get("cutoff_ts", 0), kw["P"], kw["G"], kw["T"], kw.get("row_stride", 0),
                             kw.get("power_threshold", 0.0), kw.get("in_kind", ffi.GPR_MEM_DEVICE),
                             kw.get("util_format", ffi.GPR_FMT_F32), kw.get("groups"))
            C.memmove(C.byref(wins, i * C.sizeof(ffi.gpr_window)), C.byref(w), C.sizeof(ffi.gpr_window))
            r = ress[i]
            r.struct_size = C.sizeof(ffi.gpr_result)
            r.out_mem_kind = kw.get("out_kind", ffi.GPR_MEM_DEVICE)
            r.decision_bits = _ptr(kw["decision_bits"])
            r.candidate_bits = _ptr(kw.get("candidate_bits"))
            r.series_max = _ptr(kw.get("series_max"))
            r.veto_bits = _ptr(kw.get("veto_bits"))
            r.idle_slots = _ptr(kw.get("idle_slots"))
        return wins, ress, calls   # `calls` keeps the tensors alive

    def decide_batch_async(self, batch, n: Optional[int] = None):
        wins, ress, _ = batch
        n = len(wins) if n is None else n
        self._check(self._lib.gpr_decide_batch_async(self._h, wins, ress, n))
        return ress

    def sync(self):
        self._check(self._lib.gpr_sync(self._h))
        self._keep.clear()

    # ---- resident window (daemon mode) --------------------------------------------------------
    def resident_init(self, P: int, G: int, T: int, power_plane: bool = False, block_index: bool = False):
        flags = (ffi.GPR_F_POWER_PLANE if power_plane else 0) | (ffi.GPR_F_BLOCK_INDEX if block_index else 0)
        self._check(self._lib.gpr_resident_init(self._h, P, G, T, flags))
        self._res_rows = int(P) * int(G)

    def resident_reindex(self):
        self._check(self._lib.gpr_resident_reindex(self._h))

    def append(self, util_cols, power_cols=None, n_new: Optional[int] = None, row_stride: int = 0,
               mem_kind: int = ffi.GPR_MEM_HOST):
        if isinstance(util_cols, np.ndarray):
            util_cols = np.ascontiguousarray(util_cols, dtype=np.float32)
            n_new = util_cols.shape[-1]
            if power_cols is not None:
                power_cols = np.ascontiguousarray(power_cols, dtype=np.float32)
        self._check(self._lib.gpr_append(self._h, _ptr(util_cols), _ptr(power_cols), n_new,
                                         row_stride, mem_kind))  # blocking: the columns are consumed

    def resident_planes(self):
        u, p, ld = C.c_void_p(), C.c_void_p(), C.c_uint64()
        self._check(self._lib.gpr_resident_planes(self._h, C.byref(u), C.byref(p), C.byref(ld)))
        return u.value, p.value, ld.value

    # ---- multi-GPU ------------------------------------------------------------------------------
    def comm_unique_id(self) -> bytes:
        buf = C.create_string_buffer(ffi.GPR_UNIQUE_ID_BYTES)
        rc = self._lib.gpr_comm_unique_id(buf)
        if rc != ffi.GPR_OK:
            raise GprError(rc, (self._lib.gpr_last_error(None) or b"").decode())
        return buf.raw

    def comm_init(self, unique_id: bytes, rank: int, world: int):
        buf = C.create_string_buffer(unique_id, ffi.GPR_UNIQUE_ID_BYTES)
        self._check(self._lib.gpr_comm_init(self._h, buf, rank, world))

    def p2p_init(self, rank: int, world: int, max_pods_per_rank: int) -> bytes:
        """allocate this rank's exchange block; returns the 64-byte CUDA IPC handle to publish"""
        buf = C.create_string_buffer(ffi.GPR_P2P_HANDLE_BYTES)
        self._check(self._lib.gpr_p2p_init(self._h, rank, world, max_pods_per_rank, buf))
        return buf.raw

    def p2p_attach(self, handles):
        """handles: the world handles in rank order (bytes each); enables the fused exchange"""
        blob = b"".join(handles)
        self._check(self._lib.gpr_p2p_attach(self._h, C.create_string_buffer(blob, len(blob))))

    def comm_destroy(self):
        self._check(self._lib.gpr_comm_destroy(self._h))

    # ---- memory / measurement helpers -------------------------------------------------------------
    def host_alloc(self, nbytes: int) -> int:
        p = C.c_void_p()
        self._check(self._lib.gpr_host_alloc(self._h, nbytes, C.byref(p)))
        return p.value

    def host_free(self, ptr: int):
        self._check(self._lib.gpr_host_free(self._h, ptr))

    def host_array(self, shape, dtype) -> np.ndarray:
        """numpy view over freshly allocated PINNED host memory (freed with the engine)."""
        dtype = np.dtype(dtype)
        n = int(np.prod(shape)) * dtype.itemsize
        ptr = self.host_alloc(max(n, 1))
        self._host_arrays.append(ptr)
        buf = (C.c_char * max(n, 1)).from_address(ptr)
        arr = np.frombuffer(buf, dtype=dtype, count=int(np.prod(shape))).reshape(shape)
        return arr

    def device_alloc(self, nbytes: int) -> int:
        p = C.c_void_p()
        self._check(self._lib.gpr_device_alloc(self._h, nbytes, C.byref(p)))
        return p.value

    def device_free(self, ptr: int):
        self._check(self._lib.gpr_device_free(self._h, ptr))

    def memcpy(self, dst, src, nbytes: int, dst_kind: int, src_kind: int):
        self._check(self._lib.gpr_memcpy(self._h, _ptr(dst), _ptr(src), nbytes, dst_kind, src_kind))

    def timer_begin(self):
        self._check(self._lib.gpr_timer_begin(self._h))

    def timer_end(self) -> float:
        ms = C.c_double()
        self._check(self._lib.gpr_timer_end(self._h, C.byref(ms)))
        return ms.value

    def step_stamps(self):
        """(begin_ns, ns[]) — device %globaltimer at the last timer_begin and at the completion of every
        decision retired by the last sync / blocking call"""
        n, t0 = C.c_uint32(), C.c_uint64()
        self._check(self._lib.gpr_step_stamps(self._h, None, 0, C.byref(n), C.byref(t0)))
        out = np.zeros(max(n.value, 1), np.uint64)
        self._check(self._lib.gpr_step_stamps(self._h, _ptr(out), n.value, C.byref(n), C.byref(t0)))
        return int(t0.value), out[:n.value]

    def phase_stamps(self) -> np.ndarray:
        """[n, 4] ns: fold start, folded, flags raised, peers arrived — per decision retired by the last sync"""
        n = C.c_uint32()
        self._check(self._lib.gpr_phase_stamps(self._h, None, 0, C.byref(n)))
        out = np.zeros(max(n.value, 4), np.uint64)
        self._check(self._lib.gpr_phase_stamps(self._h, _ptr(out), n.value, C.byref(n)))
        return out[:n.value].reshape(-1, 4)

    def p2p_debug(self, mode: int):
        self._check(self._lib.gpr_p2p_debug(self._h, mode))

    def flush_l2(self):
        self._check(self._lib.gpr_flush_l2(self._h))

    def launch_count(self) -> int:
        n = C.c_uint64()
        self._check(self._lib.gpr_launch_count(self._h, C.byref(n)))
        return n.value

    def device_info(self) -> dict:
        info = ffi.gpr_device_info()
        info.struct_size = C.sizeof(ffi.gpr_device_info)
        self._check(self._lib.gpr_get_device_info(self._h, C.byref(info)))
        return {"name": info.name.decode(errors="replace"), "sm_count": info.sm_count,
                "cc": (info.cc_major, info.cc_minor), "l2_bytes": info.l2_bytes,
                "hbm_bytes": info.hbm_bytes}

    # ---- device-side ingest of the response text ------------------------------------------------
    SPAN_DTYPE = np.dtype([("begin", "<u8"), ("end", "<u8"), ("row", "<u4"), ("flags", "<u4"),
                           ("n_in", "<u4"), ("n_oow", "<u4"), ("n_tiny", "<u4"), ("reserved", "<u4")])

    def text_scan(self, text, slot: int = 0, n_bytes: Optional[int] = None, mem_kind: int = ffi.GPR_MEM_HOST):
        """Upload response text (bytes, or a pinned uint8 array from :meth:`host_array`) into ``slot`` and
        return the sorted offsets of every ``},"values":[`` and ``"]]``."""
        if isinstance(text, (bytes, bytearray)):
            buf = np.frombuffer(text, dtype=np.uint8)
        else:
            buf = text
        n = int(buf.size if n_bytes is None else n_bytes)
        cap = max(1024, n // 256)
        while True:
            opens = np.empty(cap, np.uint64)
            closes = np.empty(cap, np.uint64)
            no, nc = C.c_uint64(0), C.c_uint64(0)
            rc = self._lib.gpr_text_scan(self._h, slot, _ptr(buf), n, mem_kind, _ptr(opens), _ptr(closes), cap,
                                         C.byref(no), C.byref(nc))
            if rc == ffi.GPR_E_CAPACITY and max(no.value, nc.value) > cap:   # our cap was short: ask again
                cap = int(max(no.value, nc.value)) + 16
                continue
            # (otherwise a piece of the text held more markers than the scan has room for: raise)
            self._check(rc)
            return np.sort(opens[:no.value]), np.sort(closes[:nc.value])

    def text_scan_chunks(self, text, slot: int = 0, n_bytes: Optional[int] = None, mem_kind: int = ffi.GPR_MEM_HOST):
        """generator over the pipelined scan: yields (opens, closes, bytes_done) per piece of at most 2 MB while later chunks are
        still being uploaded (gpr_text_scan_begin / gpr_text_scan_next)"""
        buf = np.frombuffer(text, dtype=np.uint8) if isinstance(text, (bytes, bytearray)) else text
        n = int(buf.size if n_bytes is None else n_bytes)
        self._check(self._lib.gpr_text_scan_begin(self._h, slot, _ptr(buf), n, mem_kind))
        cap = 1 << 14
        opens, closes = np.empty(cap, np.uint64), np.empty(cap, np.uint64)
        no, nc, done, more = C.c_uint64(0), C.c_uint64(0), C.c_uint64(0), C.c_int32(1)
        while more.value:
            self._check(self._lib.gpr_text_scan_next(self._h, _ptr(opens), _ptr(closes), cap, C.byref(no), C.byref(nc),
                                                     C.byref(done), C.byref(more)))
            yield opens[:no.value].copy(), closes[:nc.value].copy(), done.value

    def text_parse(self, spans: np.ndarray, t_end: int, step: int, T: int, n_rows: int, slot: int = 0,
                   plane: int = 0, fill: bool = True, window_seconds: Optional[int] = None,
                   resident: bool = False, power_threshold: Optional[float] = 0.0) -> np.ndarray:
        """Parse the samples of ``spans`` (structured array of SPAN_DTYPE, sorted by begin) of the text in
        ``slot`` into the context's plane (or, ``resident=True``, the resident ring); returns the spans with
        their out-fields filled.  ``window_seconds`` defaults to ``T * step``.  ``power_threshold``: for the
        power plane, the threshold it will be decided with (samples are snapped to it, include/gpr.h)."""
        spans = np.ascontiguousarray(spans, dtype=self.SPAN_DTYPE)
        g = _text_grid(t_end, step, T, n_rows, window_seconds, power_threshold, fill, resident)
        self._check(self._lib.gpr_text_parse(self._h, slot, _ptr(spans), len(spans), C.byref(g), plane))
        return spans

    def samples_scatter(self, offsets, rows, ts_ms, values, t_end: int, step: int, T: int, n_rows: int, *,
                        window_seconds: Optional[int] = None, plane: int = 0, resident: bool = False,
                        fill: bool = True, power_threshold: Optional[float] = 0.0, mem_kind: int = ffi.GPR_MEM_HOST,
                        n_series: Optional[int] = None) -> dict:
        """Merge decoded samples into the context's plane (or, ``resident=True``, the resident ring), exactly as
        :meth:`text_parse` merges the same samples written as text.  CSR form: series s owns samples
        ``offsets[s]:offsets[s+1]`` (uint64) of ``ts_ms`` (int64 Unix milliseconds) and ``values`` (float64) and
        feeds row ``rows[s]`` (uint32).  Host arrays (numpy; pinned ones from :meth:`host_array` upload fastest) are
        converted to those dtypes; with ``mem_kind=GPR_MEM_DEVICE`` pass device addresses / tensors and
        ``n_series``.  Returns the counts ``{"n_in", "n_oow", "n_tiny"}``."""
        if mem_kind == ffi.GPR_MEM_HOST:
            offsets = np.ascontiguousarray(offsets, dtype=np.uint64)
            rows = np.ascontiguousarray(rows, dtype=np.uint32)
            ts_ms = np.ascontiguousarray(ts_ms, dtype=np.int64)
            values = np.ascontiguousarray(values, dtype=np.float64)
        n_series = _n_series(n_series, rows, mem_kind)
        b = ffi.gpr_sample_batch()
        b.struct_size = C.sizeof(ffi.gpr_sample_batch)
        b.mem_kind = mem_kind
        b.offsets, b.rows, b.ts_ms, b.values = _ptr(offsets), _ptr(rows), _ptr(ts_ms), _ptr(values)
        b.n_series = n_series
        g = _text_grid(t_end, step, T, n_rows, window_seconds, power_threshold, fill, resident)
        st = ffi.gpr_sample_stats()
        self._check(self._lib.gpr_samples_scatter(self._h, C.byref(b), C.byref(g), plane, C.byref(st)))
        return {"n_in": st.n_in, "n_oow": st.n_oow, "n_tiny": st.n_tiny}

    def chunks_scatter(self, series_chunks, rows, chunk_bytes, data, t_end: int, step: int, T: int, n_rows: int, *,
                       window_seconds: Optional[int] = None, plane: int = 0, resident: bool = False,
                       fill: bool = True, power_threshold: Optional[float] = 0.0, mem_kind: int = ffi.GPR_MEM_HOST,
                       n_series: Optional[int] = None) -> dict:
        """Decode Prometheus XOR chunks and merge their samples into the context's plane (or, ``resident=True``, the
        resident ring), exactly as :meth:`samples_scatter` merges the same decoded samples.  CSR over chunks: series
        s owns chunks ``series_chunks[s]:series_chunks[s+1]`` (uint64) and feeds row ``rows[s]`` (uint32); chunk c is
        ``data[chunk_bytes[c]:chunk_bytes[c+1]]`` (uint64 offsets into the uint8 ``data``).  Host arrays (numpy) are
        converted to those dtypes; with ``mem_kind=GPR_MEM_DEVICE`` pass device addresses / tensors and
        ``n_series``.  Returns the counts ``{"n_in", "n_oow", "n_tiny"}``."""
        if mem_kind == ffi.GPR_MEM_HOST:
            series_chunks = np.ascontiguousarray(series_chunks, dtype=np.uint64)
            rows = np.ascontiguousarray(rows, dtype=np.uint32)
            chunk_bytes = np.ascontiguousarray(chunk_bytes, dtype=np.uint64)
            data = np.ascontiguousarray(np.frombuffer(data, np.uint8) if isinstance(data, (bytes, bytearray))
                                        else data, dtype=np.uint8)
        n_series = _n_series(n_series, rows, mem_kind)
        b = ffi.gpr_chunk_batch()
        b.struct_size = C.sizeof(ffi.gpr_chunk_batch)
        b.mem_kind = mem_kind
        b.series_chunks, b.rows, b.chunk_bytes, b.data = _ptr(series_chunks), _ptr(rows), _ptr(chunk_bytes), _ptr(data)
        b.n_series = n_series
        g = _text_grid(t_end, step, T, n_rows, window_seconds, power_threshold, fill, resident)
        st = ffi.gpr_sample_stats()
        self._check(self._lib.gpr_chunks_scatter(self._h, C.byref(b), C.byref(g), plane, C.byref(st)))
        return {"n_in": st.n_in, "n_oow": st.n_oow, "n_tiny": st.n_tiny}

    def resident_export(self, t_end: int, step: int, *, plane: int = 0, max_per_chunk: int = 120,
                        window_seconds: Optional[int] = None, power_threshold: Optional[float] = 0.0) -> dict:
        """Encode one plane of the resident ring (0 = util, 1 = power) as Prometheus XOR chunks on the GPU
        (gpr_resident_export): every row with a sample is a series, its cells oldest first at
        ``t_end - (T - 1 - j) * step`` seconds.  Returns numpy arrays ready for :meth:`chunks_scatter`
        (``series_chunks``, ``rows``, ``chunk_bytes``, ``data``), the counts ``n_samples``, and the ``grid`` to
        restore with: ``chunks_scatter(..., **out["grid"], resident=True)`` into a ring of the same T."""
        T = int(self.resident_planes()[2])
        g = _text_grid(t_end, step, T, window_seconds=window_seconds, power_threshold=power_threshold)
        o = ffi.gpr_chunk_export()
        o.struct_size = C.sizeof(ffi.gpr_chunk_export)
        o.mem_kind = ffi.GPR_MEM_HOST
        arrays = None
        for _ in range(2):   # the sizes, then the chunks
            if arrays is None:
                arrays = (np.zeros(1, np.uint64), np.zeros(0, np.uint32), np.zeros(1, np.uint64), np.zeros(0, np.uint8))
            o.series_chunks, o.rows, o.chunk_bytes, o.data = (_ptr(a) if a.size else None for a in arrays)
            o.cap_series, o.cap_chunks, o.cap_bytes = arrays[1].size, arrays[2].size - 1, arrays[3].size
            rc = self._lib.gpr_resident_export(self._h, C.byref(g), int(plane), int(max_per_chunk), C.byref(o))
            if rc != ffi.GPR_E_CAPACITY:
                break
            arrays = (np.zeros(o.n_series + 1, np.uint64), np.zeros(o.n_series, np.uint32),
                      np.zeros(o.n_chunks + 1, np.uint64), np.zeros(o.n_bytes, np.uint8))
        self._check(rc)
        return {"series_chunks": arrays[0], "rows": arrays[1], "chunk_bytes": arrays[2], "data": arrays[3],
                "n_samples": int(o.n_samples),
                "grid": {"t_end": int(t_end), "step": int(step), "T": T, "window_seconds": int(g.window_seconds),
                         "plane": int(plane), "power_threshold": g.power_threshold}}

    def resident_head(self) -> int:
        h = C.c_uint32()
        self._check(self._lib.gpr_resident_head(self._h, C.byref(h)))
        return h.value

    def resident_advance(self, n_new: int):
        """open the next ``n_new`` buckets of the resident ring without data (all rows: no sample)"""
        self._check(self._lib.gpr_resident_advance(self._h, int(n_new)))

    def resident_remap(self, P: int, G: int, src_rows):
        """Give the resident ring the shape ``[P][G][T]`` without losing its history: new row ``i`` holds old row
        ``src_rows[i]`` (uint32, ``P * G`` entries), or no sample for ``ffi.GPR_ROW_NONE``.  ``src_rows`` is a
        numpy array (host) or a contiguous int32 / uint32 CUDA tensor on the engine's device (read in place; as
        int32, ``GPR_ROW_NONE`` is -1)."""
        if hasattr(src_rows, "is_cuda") and src_rows.is_cuda:
            import torch
            if src_rows.dtype not in (torch.int32, torch.uint32):
                raise ValueError(f"src_rows must be an int32 or uint32 tensor, not {src_rows.dtype}")
            if src_rows.device.index != self.device:
                raise ValueError(f"src_rows is on {src_rows.device}, the engine on cuda:{self.device}")
            if not src_rows.is_contiguous() or src_rows.numel() != P * G:
                raise ValueError(f"src_rows must be a contiguous tensor of P * G = {P * G} entries")
            self._check(self._lib.gpr_resident_remap(self._h, int(P), int(G), src_rows.data_ptr(),
                                                     ffi.GPR_MEM_DEVICE))
            self._res_rows = int(P) * int(G)
            return
        rows = np.ascontiguousarray(src_rows, dtype=np.uint32).ravel()
        if rows.size != P * G:
            raise ValueError(f"src_rows has {rows.size} entries, not P * G = {P * G}")
        self._check(self._lib.gpr_resident_remap(self._h, int(P), int(G), rows.ctypes.data, ffi.GPR_MEM_HOST))
        self._res_rows = int(P) * int(G)

    def resident_live_rows(self) -> np.ndarray:
        """Which rows of the resident ring hold at least one sample (any non-NaN cell) in the util plane or the power
        plane (gpr_resident_live_rows): a bool array of ``P * G`` entries, row ``pod * G + slot``.  What a caller of
        :meth:`resident_remap` reads to choose which pods to keep."""
        rows = getattr(self, "_res_rows", None)
        if rows is None:
            raise RuntimeError("no resident window (resident_init)")
        words = np.zeros(max(1, (rows + 31) // 32), np.uint32)
        self._check(self._lib.gpr_resident_live_rows(self._h, words.ctypes.data, ffi.GPR_MEM_HOST))
        return np.unpackbits(words.view(np.uint8), bitorder="little")[:rows].astype(bool)

    def resident_retime(self, n_keep: int, factor: int):
        """Put the resident ring on a coarser or shorter grid (gpr_resident_retime): its newest ``n_keep`` buckets
        merged ``factor`` to a bucket, newest first, into ``ceil(n_keep / factor)`` buckets; the head becomes 0 and a
        block index is rebuilt.  ``gpr::retime_plan`` (csrc/gpr_retime.h) says which grid changes this makes exact."""
        self._check(self._lib.gpr_resident_retime(self._h, int(n_keep), int(factor)))

    def resident_cols(self, plane: int, newer: int, n_cols: int) -> np.ndarray:
        """A band of the resident ring (gpr_resident_cols): the ``n_cols`` buckets that end ``newer`` buckets before
        the newest, oldest first, of plane ``plane`` (0 util, 1 power) for every row — a float32 array
        ``[P * G, n_cols]``, row ``pod * G + slot``, NaN where a bucket holds no sample."""
        rows = getattr(self, "_res_rows", None)
        if rows is None:
            raise RuntimeError("no resident window (resident_init)")
        out = np.empty((rows, max(0, int(n_cols))), np.float32)
        self._check(self._lib.gpr_resident_cols(self._h, int(plane), int(newer), int(n_cols), out.ctypes.data,
                                                ffi.GPR_MEM_HOST))
        return out

    def text_planes(self):
        u, w = C.c_void_p(), C.c_void_p()
        self._check(self._lib.gpr_text_planes(self._h, C.byref(u), C.byref(w)))
        return u.value, w.value

    def synth_fill(self, seed: int, plane: int, dst, pod_offset: int, P: int, G: int, T: int,
                   row_stride: int = 0):
        self._check(self._lib.gpr_synth_fill(self._h, seed, plane, _ptr(dst), pod_offset, P, G, T,
                                             row_stride))

    def synth_eligible(self, seed: int, dst, pod_offset: int, P: int):
        self._check(self._lib.gpr_synth_eligible(self._h, seed, _ptr(dst), pod_offset, P))
