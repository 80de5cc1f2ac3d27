"""ctypes binding of the CPU oracle (oracle/dnz_oracle.c).

TEST INFRASTRUCTURE ONLY: imported by tests/, __graft_entry__.smoke() and bench.py's CPU-baseline legs.
Nothing in denormalized_b200/ may import this package.  PARITY UNPINNED -- see dnz_oracle.h.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
from dataclasses import dataclass

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "_build", "libdnz_oracle.so")

OPS = {">": 0, ">=": 1, "<": 2, "<=": 3, "==": 4, "!=": 5}
COLS = {"count": 0, "min": 1, "max": 2, "average": 3, "avg": 3, "sum": 4}


def build(force: bool = False) -> str:
    """Compile oracle/dnz_oracle.c with gcc (recipe: oracle/Makefile)."""
    src = os.path.join(_HERE, "dnz_oracle.c")
    if force or not os.path.exists(_SO) or os.path.getmtime(_SO) < max(
        os.path.getmtime(src), os.path.getmtime(os.path.join(_HERE, "dnz_oracle.h"))
    ):
        subprocess.check_call(["make", "-C", _HERE, "-s"])
    return _SO


class _Config(C.Structure):
    _fields_ = [("window_ms", C.c_int64), ("slide_ms", C.c_int64), ("has_filter", C.c_int32),
                ("filter_col", C.c_int32), ("filter_op", C.c_int32), ("reserved", C.c_int32),
                ("filter_lit", C.c_double)]


class _Batch(C.Structure):
    _fields_ = [("n", C.c_int64), ("ts", C.c_void_p), ("ts_valid", C.c_void_p), ("val", C.c_void_p),
                ("val_valid", C.c_void_p), ("key_off", C.c_void_p), ("key_bytes", C.c_void_p),
                ("key_valid", C.c_void_p), ("occurred_at", C.c_void_p), ("barrier_off", C.c_void_p),
                ("barrier_bytes", C.c_void_p)]


class _Result(C.Structure):
    _fields_ = [("n", C.c_int64), ("key_off", C.c_void_p), ("key_bytes", C.c_void_p), ("key_isnull", C.c_void_p),
                ("count", C.c_void_p), ("min", C.c_void_p), ("max", C.c_void_p), ("avg", C.c_void_p),
                ("agg_isnull", C.c_void_p), ("window_start_ms", C.c_void_p), ("window_end_ms", C.c_void_p),
                ("emit_seq", C.c_void_p), ("sum", C.c_void_p)]


_lib = None


def lib():
    global _lib
    if _lib is None:
        build()
        L = C.CDLL(_SO)
        L.orc_create.restype = C.c_void_p
        L.orc_create.argtypes = [C.POINTER(_Config)]
        L.orc_destroy.argtypes = [C.c_void_p]
        L.orc_push.restype = C.c_int64
        L.orc_push.argtypes = [C.c_void_p, C.POINTER(_Batch)]
        L.orc_get_results.argtypes = [C.c_void_p, C.POINTER(_Result)]
        L.orc_clear_results.argtypes = [C.c_void_p]
        L.orc_open_frames.restype = C.c_int64
        L.orc_open_frames.argtypes = [C.c_void_p]
        L.orc_watermark.restype = C.c_int64
        L.orc_watermark.argtypes = [C.c_void_p]
        L.orc_last_error.restype = C.c_char_p
        L.orc_last_error.argtypes = [C.c_void_p]
        L.orc_mt_create.restype = C.c_void_p
        L.orc_mt_create.argtypes = [C.POINTER(_Config), C.c_int]
        L.orc_mt_destroy.argtypes = [C.c_void_p]
        L.orc_mt_push_many.restype = C.c_int64
        L.orc_mt_push_many.argtypes = [C.c_void_p, C.POINTER(_Batch), C.c_int64]
        L.orc_mt_num_results.restype = C.c_int64
        L.orc_mt_num_results.argtypes = [C.c_void_p]
        L.orc_mt_get_results.argtypes = [C.c_void_p, C.c_int, C.POINTER(_Result)]
        L.orc_mt_clear_results.argtypes = [C.c_void_p]
        L.orc_synth_fill.restype = C.c_int64
        L.orc_synth_fill.argtypes = [C.c_int64, C.c_int64, C.c_uint64, C.c_int64, C.c_int64, C.c_int64, C.c_int32, C.c_int64, C.c_int64,
                                     C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        L.orc_u_create.restype = C.c_void_p
        L.orc_u_create.argtypes = [C.POINTER(_Config)]
        L.orc_u_destroy.argtypes = [C.c_void_p]
        L.orc_u_push.restype = C.c_int64
        L.orc_u_push.argtypes = [C.c_void_p, C.POINTER(_Batch)]
        L.orc_u_get_results.argtypes = [C.c_void_p, C.POINTER(_Result)]
        L.orc_u_clear_results.argtypes = [C.c_void_p]
        L.orc_u_last_error.restype = C.c_char_p
        L.orc_u_last_error.argtypes = [C.c_void_p]
        L.orc_ts_convert.restype = C.c_int64
        L.orc_ts_convert.argtypes = [C.c_int32, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_char_p, C.c_void_p]
        _lib = L
    return _lib


@dataclass
class Batch:
    """Needed columns of one canonical-schema RecordBatch as numpy arrays (validity = Arrow LSB bitmaps or None)."""
    ts: np.ndarray
    val: np.ndarray
    key_off: np.ndarray
    key_bytes: np.ndarray
    ts_valid: np.ndarray | None = None
    val_valid: np.ndarray | None = None
    key_valid: np.ndarray | None = None
    occurred_at: np.ndarray | None = None
    barrier_off: np.ndarray | None = None
    barrier_bytes: np.ndarray | None = None

    @property
    def n(self) -> int:
        return int(self.ts.shape[0])

    def _c(self) -> _Batch:
        def p(a):
            return None if a is None else a.ctypes.data
        assert self.ts.dtype == np.int64 and self.val.dtype == np.float64 and self.key_off.dtype == np.int32
        return _Batch(self.n, p(self.ts), p(self.ts_valid), p(self.val), p(self.val_valid), p(self.key_off),
                      p(self.key_bytes), p(self.key_valid), p(self.occurred_at), p(self.barrier_off),
                      p(self.barrier_bytes))


def _mkcfg(window_ms, slide_ms=0, filt=None) -> _Config:
    c = _Config(int(window_ms), int(slide_ms or 0), 0, 0, 0, 0, 0.0)
    if filt is not None:
        col, op, lit = filt
        c.has_filter, c.filter_col, c.filter_op, c.filter_lit = 1, COLS[col], OPS[op], float(lit)
    return c


def _rows(res: _Result, with_sum=False):
    """-> list of tuples (window_start, window_end, key(bytes|None), count, min|None, max|None, avg|None, emit_seq), with sum|None
    appended at index 8 when `with_sum`"""
    n = res.n
    if n == 0:
        return []

    def arr(ptr, dt, m):
        return np.ctypeslib.as_array(C.cast(ptr, C.POINTER(C.c_uint8)), shape=(m * np.dtype(dt).itemsize,)).view(dt).copy()
    off = arr(res.key_off, np.int32, n + 1)
    kb = arr(res.key_bytes, np.uint8, max(int(off[-1]), 1)).tobytes() if res.key_bytes else b""
    knull = arr(res.key_isnull, np.uint8, n)
    cnt = arr(res.count, np.int64, n)
    mn, mx, av = arr(res.min, np.float64, n), arr(res.max, np.float64, n), arr(res.avg, np.float64, n)
    anull = arr(res.agg_isnull, np.uint8, n)
    ws, we, seq = arr(res.window_start_ms, np.int64, n), arr(res.window_end_ms, np.int64, n), arr(res.emit_seq, np.int64, n)
    sm = arr(res.sum, np.float64, n) if with_sum else None
    out = []
    for i in range(n):
        key = None if knull[i] else kb[off[i]:off[i + 1]]
        if anull[i]:
            r = (int(ws[i]), int(we[i]), key, int(cnt[i]), None, None, None, int(seq[i]))
        else:
            r = (int(ws[i]), int(we[i]), key, int(cnt[i]), float(mn[i]), float(mx[i]), float(av[i]), int(seq[i]))
        if with_sum:
            r += (None if anull[i] else float(sm[i]),)
        out.append(r)
    return out


def _arrays(res: _Result) -> dict:
    """Result set as numpy arrays (copies): key_off[n+1], key_bytes, key_isnull, count, min, max, avg, sum, agg_isnull, window_start,
    window_end.  For large outputs (millions of rows), where the tuple list of _rows() would take minutes."""
    n = int(res.n)

    def arr(ptr, dt, m):
        if m == 0:
            return np.zeros(0, dt)
        return np.ctypeslib.as_array(C.cast(ptr, C.POINTER(C.c_uint8)), shape=(m * np.dtype(dt).itemsize,)).view(dt).copy()
    off = arr(res.key_off, np.int32, n + 1) if n else np.zeros(1, np.int32)
    return {"n": n, "key_off": off, "key_bytes": arr(res.key_bytes, np.uint8, int(off[-1])), "key_isnull": arr(res.key_isnull, np.uint8, n),
            "count": arr(res.count, np.int64, n), "min": arr(res.min, np.float64, n), "max": arr(res.max, np.float64, n),
            "avg": arr(res.avg, np.float64, n), "sum": arr(res.sum, np.float64, n), "agg_isnull": arr(res.agg_isnull, np.uint8, n),
            "window_start": arr(res.window_start_ms, np.int64, n), "window_end": arr(res.window_end_ms, np.int64, n)}


class OracleWindow:
    """Single-partition GroupedWindowAggStream (+ FilterExec) -- the ground truth."""

    def __init__(self, window_ms, slide_ms=0, filt=None):
        self._L = lib()
        cfg = _mkcfg(window_ms, slide_ms, filt)
        self._h = self._L.orc_create(C.byref(cfg))

    def push(self, b: Batch) -> int:
        cb = b._c()
        r = self._L.orc_push(self._h, C.byref(cb))
        if r < 0:
            raise RuntimeError(self._L.orc_last_error(self._h).decode())
        return int(r)

    def results(self, clear=True, with_sum=False):
        """Emitted rows (see _rows); `with_sum` appends sum at index 8."""
        res = _Result()
        self._L.orc_get_results(self._h, C.byref(res))
        rows = _rows(res, with_sum)
        if clear:
            self._L.orc_clear_results(self._h)
        return rows

    @property
    def open_frames(self) -> int:
        return int(self._L.orc_open_frames(self._h))

    @property
    def watermark(self):
        v = int(self._L.orc_watermark(self._h))
        return None if v == -(2 ** 63) else v

    def close(self):
        if self._h:
            self._L.orc_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class OracleUngrouped:
    """`.window([], aggs, ..)`: one partition of the Partial -> Final chain (rows: key is always None)."""

    def __init__(self, window_ms, slide_ms=0):
        self._L = lib()
        cfg = _mkcfg(window_ms, slide_ms, None)
        self._h = self._L.orc_u_create(C.byref(cfg))

    def push(self, b: Batch) -> int:
        cb = b._c()
        r = self._L.orc_u_push(self._h, C.byref(cb))
        if r < 0:
            raise RuntimeError(self._L.orc_u_last_error(self._h).decode())
        return int(r)

    def results(self, clear=True, with_sum=False):
        res = _Result()
        self._L.orc_u_get_results(self._h, C.byref(res))
        rows = _rows(res, with_sum)
        if clear:
            self._L.orc_u_clear_results(self._h)
        return rows

    def close(self):
        if self._h:
            self._L.orc_u_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class OracleMT:
    """Hash-partitioned multi-threaded mode: the timed CPU baseline."""

    def __init__(self, window_ms, slide_ms=0, filt=None, partitions=1):
        self._L = lib()
        cfg = _mkcfg(window_ms, slide_ms, filt)
        self.partitions = partitions
        self._h = self._L.orc_mt_create(C.byref(cfg), partitions)

    def push_many(self, batches) -> int:
        arr = (_Batch * len(batches))(*[b._c() for b in batches])
        r = self._L.orc_mt_push_many(self._h, arr, len(batches))
        if r < 0:
            raise RuntimeError(f"oracle mt error {r}")
        return int(r)

    def num_results(self) -> int:
        return int(self._L.orc_mt_num_results(self._h))

    def results(self, clear=True, with_sum=False):
        rows = []
        for p in range(self.partitions):
            res = _Result()
            self._L.orc_mt_get_results(self._h, p, C.byref(res))
            rows += _rows(res, with_sum)
        if clear:
            self._L.orc_mt_clear_results(self._h)
        return rows

    def results_arrays(self, clear=True):
        """One dict of numpy arrays per partition (see _arrays)."""
        out = []
        for p in range(self.partitions):
            res = _Result()
            self._L.orc_mt_get_results(self._h, p, C.byref(res))
            out.append(_arrays(res))
        if clear:
            self._L.orc_mt_clear_results(self._h)
        return out

    def clear(self):
        self._L.orc_mt_clear_results(self._h)

    def close(self):
        if self._h:
            self._L.orc_mt_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def synth_batch(row0, n, *, seed=42, groups=1000, rows_per_ms=1000, t0_ms=1_700_000_000_000, uuid_keys=False,
                extra_columns=False, key_mul=1, key_add=0) -> Batch:
    """Rows [row0,row0+n) of the synthetic sensor stream (SURVEY.md §8d)."""
    L = lib()
    ts = np.empty(n, np.int64)
    val = np.empty(n, np.float64)
    off = np.empty(n + 1, np.int32)
    kb = np.empty(n * (36 if uuid_keys else 27) + 16, np.uint8)
    used = L.orc_synth_fill(row0, n, seed, groups, rows_per_ms, t0_ms, 1 if uuid_keys else 0, key_mul, key_add,
                            ts.ctypes.data, val.ctypes.data, off.ctypes.data, kb.ctypes.data)
    b = Batch(ts=ts, val=val, key_off=off, key_bytes=kb[:max(int(used), 1)])
    if extra_columns:
        b.occurred_at = ts.copy()
        b.barrier_off = (np.arange(n + 1, dtype=np.int32) * 10)
        b.barrier_bytes = np.frombuffer(b"no_barrier" * n, dtype=np.uint8).copy() if n else np.zeros(1, np.uint8)
    return b


def sort_rows(rows):
    """Parity is on the multiset of rows sorted by (window_start, key) (SURVEY.md §8a rule 4)."""
    return sorted(rows, key=lambda r: (r[0], r[1], r[2] is None, r[2] or b"", r[7] if len(r) > 7 else 0))


def ts_convert(unit, values=None, strings=None, fmt=None) -> np.ndarray:
    """array_to_timestamp_array (utils/time.rs:59-94): unit 1 Int64Millis, 2 Int64Seconds, 3 StringIso8601(fmt)."""
    L = lib()
    if unit in (1, 2):
        v = np.ascontiguousarray(values, np.int64)
        out = np.empty(len(v), np.int64)
        rc = L.orc_ts_convert(unit, len(v), v.ctypes.data, None, None, None, out.ctypes.data)
    else:
        bs = [x if isinstance(x, bytes) else x.encode() for x in strings]
        off = np.zeros(len(bs) + 1, np.int32)
        off[1:] = np.cumsum([len(b) for b in bs])
        kb = np.frombuffer(b"".join(bs) + b"\0", np.uint8).copy()
        out = np.empty(len(bs), np.int64)
        rc = L.orc_ts_convert(3, len(bs), None, off.ctypes.data, kb.ctypes.data, fmt.encode(), out.ctypes.data)
    if rc:
        raise ValueError(f"row {rc - 1} does not parse")
    return out
