"""ctypes binding of include/dnz_gpu.h (the drop-in boundary).  Test/bench convenience only: the reference-facing
host code is the C++ mirror in cpp/ (and the Rust shim sketched in INTEGRATION.md).

`GpuStreamingWindow` plays the role of one partition's GroupedWindowAggStream
(crates/core/src/physical_plan/continuous/grouped_window_agg_stream.rs:63-82): push RecordBatches, poll emitted
windows.  It fails loudly when the CUDA library is missing; nothing here computes on the CPU.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np
import pyarrow as pa

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "libdnz_gpu.so")

AGG_KINDS = {"count": 0, "min": 1, "max": 2, "avg": 3, "average": 3, "sum": 4}
OPS = {">": 0, ">=": 1, "<": 2, "<=": 3, "==": 4, "!=": 5}
ABI_VERSION = 2
NO_KEY = -1          # DNZ_NO_KEY: `.window([], aggs, ..)`
TS_CANONICAL, TS_INT64_MILLIS, TS_INT64_SECONDS, TS_STRING_ISO8601 = 0, 1, 2, 3
FLAG_KERNEL_TIMING = 1
FLAG_FORCE_GENERIC = 2
FLAG_NO_HINTS = 4
FLAG_NO_QUEUE = 8
FLAG_NO_PRIVATE = 16
FLAG_SYNCHRONOUS = 32
FLAG_SCALAR_PROBE = 64
FLAG_STAGE_TS = 128
INTERNAL_METADATA_COLUMN = "_streaming_internal_metadata"   # crates/common/src/lib.rs:5
SYNTH_SENSOR_KEYS, SYNTH_UUID_KEYS, SYNTH_INT64_KEYS = 0, 1, 2    # dnz_synth_generate key_kind
# integer group-key types (Arrow formats l / i / L / I) -> numpy dtype of their values
INT_KEY_DTYPES = {pa.int64(): np.int64, pa.int32(): np.int32, pa.uint64(): np.uint64, pa.uint32(): np.uint32}


class DnzError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__(f"dnz error {code}: {msg}")
        self.code = code


class ArrowSchemaC(C.Structure):
    pass


class ArrowArrayC(C.Structure):
    pass


ArrowSchemaC._fields_ = [("format", C.c_char_p), ("name", C.c_char_p), ("metadata", C.c_char_p), ("flags", C.c_int64),
                         ("n_children", C.c_int64), ("children", C.POINTER(C.POINTER(ArrowSchemaC))),
                         ("dictionary", C.POINTER(ArrowSchemaC)), ("release", C.c_void_p), ("private_data", C.c_void_p)]
ArrowArrayC._fields_ = [("length", C.c_int64), ("null_count", C.c_int64), ("offset", C.c_int64), ("n_buffers", C.c_int64),
                        ("n_children", C.c_int64), ("buffers", C.POINTER(C.c_void_p)),
                        ("children", C.POINTER(C.POINTER(ArrowArrayC))), ("dictionary", C.POINTER(ArrowArrayC)),
                        ("release", C.c_void_p), ("private_data", C.c_void_p)]


class _Agg(C.Structure):
    _fields_ = [("kind", C.c_int32), ("arg_column", C.c_int32), ("alias", C.c_char_p)]


class _Config(C.Structure):
    _fields_ = [("abi_version", C.c_uint32), ("device", C.c_int32), ("key_column", C.c_int32), ("n_aggs", C.c_int32),
                ("aggs", C.POINTER(_Agg)), ("window_ms", C.c_int64), ("slide_ms", C.c_int64), ("has_filter", C.c_int32),
                ("filter_agg", C.c_int32), ("filter_op", C.c_int32), ("flags", C.c_uint32), ("filter_literal", C.c_double),
                ("expected_groups", C.c_int64), ("max_rows_per_launch", C.c_int64), ("cuda_stream", C.c_void_p),
                ("ts_source", C.c_int32), ("ts_column", C.c_int32), ("ts_format", C.c_char_p)]


class DeviceBatchC(C.Structure):
    _fields_ = [("n_rows", C.c_int64), ("ts", C.c_void_p), ("ts_valid", C.c_void_p), ("val", C.c_void_p),
                ("val_valid", C.c_void_p), ("key_off", C.c_void_p), ("key_bytes", C.c_void_p), ("key_valid", C.c_void_p)]


class DeviceResultC(C.Structure):
    _fields_ = [("n_rows", C.c_int64), ("key_bytes_len", C.c_int64), ("key_off", C.c_void_p), ("key_bytes", C.c_void_p),
                ("key_valid", C.c_void_p), ("count", C.c_void_p), ("min", C.c_void_p), ("max", C.c_void_p),
                ("avg", C.c_void_p), ("sum", C.c_void_p), ("agg_valid", C.c_void_p), ("window_start_ms", C.c_void_p),
                ("window_end_ms", C.c_void_p)]


class PartialsC(C.Structure):
    _fields_ = [("n_entries", C.c_int64), ("entries", C.c_void_p), ("owner_counts", C.POINTER(C.c_int64)),
                ("key_bytes_len", C.c_int64), ("key_bytes", C.c_void_p), ("owner_key_bytes", C.POINTER(C.c_int64)),
                ("pane_lo", C.c_int64), ("pane_hi", C.c_int64)]


class GroupConfigC(C.Structure):
    _fields_ = [("abi_version", C.c_uint32), ("rank", C.c_int32), ("world", C.c_int32), ("device", C.c_int32),
                ("ring_entries", C.c_int64), ("ring_key_bytes", C.c_int64)]


ALLGATHER_FN = C.CFUNCTYPE(C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64)


class StatsC(C.Structure):
    _fields_ = [("rows_in", C.c_int64), ("batches_in", C.c_int64), ("rows_out", C.c_int64), ("windows_emitted", C.c_int64),
                ("groups", C.c_int64), ("agg_launches", C.c_int64), ("total_launches", C.c_int64),
                ("agg_kernel_ms", C.c_double), ("agg_algorithmic_bytes", C.c_double), ("h2d_bytes", C.c_int64),
                ("d2h_bytes", C.c_int64), ("deferred_rows", C.c_int64), ("generic_tiles", C.c_int64),
                ("fast_tiles", C.c_int64), ("late_batches", C.c_int64), ("exchanged_out", C.c_int64), ("exchanged_in", C.c_int64),
                ("h2d_pageable_bytes", C.c_int64)]

    def as_dict(self):
        return {k: getattr(self, k) for k, _ in self._fields_}


EXPORTS = ["dnz_window_create", "dnz_window_push", "dnz_window_push_device", "dnz_window_poll", "dnz_window_poll_ready",
           "dnz_window_poll_device", "dnz_window_poll_device_ready",
           "dnz_window_flush", "dnz_window_stats", "dnz_window_reset_stats", "dnz_window_watermark",
           "dnz_window_last_error", "dnz_window_destroy", "dnz_window_set_exchange", "dnz_window_reserve_input", "dnz_window_process", "dnz_window_export_partials",
           "dnz_window_import_partials", "dnz_host_alloc", "dnz_host_free", "dnz_device_alloc", "dnz_device_free",
           "dnz_device_count", "dnz_memcpy", "dnz_synth_generate", "dnz_synth_bytes", "dnz_synth_free",
           "dnz_window_checkpoint", "dnz_window_restore", "dnz_blob_free",
           "dnz_group_create", "dnz_group_create_local", "dnz_group_destroy", "dnz_group_attach", "dnz_group_step_begin",
           "dnz_group_step_pack", "dnz_group_step_finish", "dnz_group_step", "dnz_group_flush"]

_lib = None


def library_path() -> str:
    return _SO


def lib():
    """Load libdnz_gpu.so.  Raises if it has not been built: there is no fallback implementation."""
    global _lib
    if _lib is None:
        if not os.path.exists(_SO):
            raise ImportError(f"{_SO} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                              "(make -C denormalized_b200/csrc).  denormalized_b200 has no CPU fallback.")
        L = C.CDLL(_SO)
        L.dnz_window_create.restype = C.c_int32
        L.dnz_window_create.argtypes = [C.POINTER(_Config), C.POINTER(ArrowSchemaC), C.POINTER(C.c_void_p)]
        L.dnz_window_push.restype = C.c_int32
        L.dnz_window_push.argtypes = [C.c_void_p, C.POINTER(ArrowArrayC)]
        L.dnz_window_push_device.restype = C.c_int32
        L.dnz_window_push_device.argtypes = [C.c_void_p, C.POINTER(DeviceBatchC), C.c_int64]
        L.dnz_window_poll.restype = C.c_int32
        L.dnz_window_poll.argtypes = [C.c_void_p, C.POINTER(ArrowArrayC), C.POINTER(ArrowSchemaC), C.POINTER(C.c_int32)]
        L.dnz_window_poll_ready.restype = C.c_int32
        L.dnz_window_poll_ready.argtypes = [C.c_void_p, C.POINTER(ArrowArrayC), C.POINTER(ArrowSchemaC), C.POINTER(C.c_int32)]
        L.dnz_window_poll_device.restype = C.c_int32
        L.dnz_window_poll_device.argtypes = [C.c_void_p, C.POINTER(DeviceResultC)]
        L.dnz_window_poll_device_ready.restype = C.c_int32
        L.dnz_window_poll_device_ready.argtypes = [C.c_void_p, C.POINTER(DeviceResultC)]
        L.dnz_window_flush.restype = C.c_int32
        L.dnz_window_flush.argtypes = [C.c_void_p, C.c_int64]
        L.dnz_window_stats.restype = C.c_int32
        L.dnz_window_stats.argtypes = [C.c_void_p, C.POINTER(StatsC)]
        L.dnz_window_reset_stats.restype = C.c_int32
        L.dnz_window_reset_stats.argtypes = [C.c_void_p]
        L.dnz_window_watermark.restype = C.c_int64
        L.dnz_window_watermark.argtypes = [C.c_void_p]
        L.dnz_window_last_error.restype = C.c_char_p
        L.dnz_window_last_error.argtypes = [C.c_void_p]
        L.dnz_window_destroy.argtypes = [C.c_void_p]
        L.dnz_window_reserve_input.restype = C.c_int32
        L.dnz_window_reserve_input.argtypes = [C.c_void_p, C.c_int64]
        L.dnz_window_set_exchange.restype = C.c_int32
        L.dnz_window_set_exchange.argtypes = [C.c_void_p, C.c_int32, C.c_int32]
        L.dnz_window_process.restype = C.c_int32
        L.dnz_window_process.argtypes = [C.c_void_p, C.POINTER(C.c_int64)]
        L.dnz_window_export_partials.restype = C.c_int32
        L.dnz_window_export_partials.argtypes = [C.c_void_p, C.c_int64, C.POINTER(PartialsC)]
        L.dnz_window_import_partials.restype = C.c_int32
        L.dnz_window_import_partials.argtypes = [C.c_void_p, C.c_void_p, C.POINTER(C.c_int64), C.c_void_p, C.POINTER(C.c_int64),
                                                 C.c_int64, C.c_int64]
        L.dnz_host_alloc.restype = C.c_void_p
        L.dnz_host_alloc.argtypes = [C.c_int64]
        L.dnz_host_free.argtypes = [C.c_void_p]
        L.dnz_device_alloc.restype = C.c_void_p
        L.dnz_device_alloc.argtypes = [C.c_int32, C.c_int64]
        L.dnz_device_free.argtypes = [C.c_int32, C.c_void_p]
        L.dnz_device_count.restype = C.c_int32
        L.dnz_memcpy.restype = C.c_int32
        L.dnz_memcpy.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_int32]
        L.dnz_synth_generate.restype = C.c_int32
        L.dnz_synth_generate.argtypes = [C.c_int32, C.c_int64, C.c_int64, C.c_int64, C.c_uint64, C.c_int64, C.c_int64,
                                         C.c_int64, C.c_int32, C.c_int64, C.c_int64, C.POINTER(C.c_void_p), C.POINTER(DeviceBatchC), C.c_int64]
        L.dnz_window_checkpoint.restype = C.c_int32
        L.dnz_window_checkpoint.argtypes = [C.c_void_p, C.POINTER(C.c_void_p), C.POINTER(C.c_int64)]
        L.dnz_window_restore.restype = C.c_int32
        L.dnz_window_restore.argtypes = [C.c_void_p, C.c_char_p, C.c_int64]
        L.dnz_blob_free.argtypes = [C.c_void_p]
        L.dnz_group_create.restype = C.c_int32
        L.dnz_group_create.argtypes = [C.POINTER(GroupConfigC), ALLGATHER_FN, C.c_void_p, C.POINTER(C.c_void_p)]
        L.dnz_group_create_local.restype = C.c_int32
        L.dnz_group_create_local.argtypes = [C.c_int32, C.POINTER(C.c_int32), C.c_int64, C.c_int64, C.POINTER(C.c_void_p)]
        L.dnz_group_destroy.argtypes = [C.c_void_p]
        L.dnz_group_attach.restype = C.c_int32
        L.dnz_group_attach.argtypes = [C.c_void_p, C.c_void_p]
        for name in ("dnz_group_step_begin", "dnz_group_step_pack"):
            getattr(L, name).restype = C.c_int32
            getattr(L, name).argtypes = [C.c_void_p, C.c_void_p]
        for name in ("dnz_group_step_finish", "dnz_group_step", "dnz_group_flush"):
            getattr(L, name).restype = C.c_int32
            getattr(L, name).argtypes = [C.c_void_p, C.c_void_p, C.POINTER(C.c_int64)]
        L.dnz_synth_bytes.restype = C.c_int64
        L.dnz_synth_bytes.argtypes = [C.c_void_p]
        L.dnz_synth_free.argtypes = [C.c_void_p]
        _lib = L
    return _lib


def canonical_schema() -> pa.Schema:
    """The reference's canonical Kafka schema for the sensor example (kafka_config.rs:186-214)."""
    meta = pa.struct([pa.field("barrier_batch", pa.utf8(), nullable=False),
                      pa.field("canonical_timestamp", pa.timestamp("ms"))])
    return pa.schema([pa.field("occurred_at_ms", pa.int64()), pa.field("reading", pa.float64()),
                      pa.field("sensor_name", pa.utf8()), pa.field(INTERNAL_METADATA_COLUMN, meta, nullable=False)])


def _bitmap_to_mask(bm, n):
    if bm is None:
        return None
    bits = np.unpackbits(np.asarray(bm, np.uint8), bitorder="little")[:n]
    return bits == 0          # pyarrow mask: True = null


def make_record_batch(ts, val, key_off, key_bytes, ts_valid=None, val_valid=None, key_valid=None) -> pa.RecordBatch:
    """Canonical-schema RecordBatch from columnar numpy buffers (validity = Arrow LSB bitmaps or None)."""
    n = len(ts)

    def vbuf(bm):
        return None if bm is None else pa.py_buffer(np.ascontiguousarray(bm[:(n + 7) // 8 + 1]))
    ts_arr = pa.Array.from_buffers(pa.timestamp("ms"), n, [vbuf(ts_valid), pa.py_buffer(np.ascontiguousarray(ts, np.int64))])
    val_arr = pa.Array.from_buffers(pa.float64(), n, [vbuf(val_valid), pa.py_buffer(np.ascontiguousarray(val, np.float64))])
    key_arr = pa.Array.from_buffers(pa.utf8(), n, [vbuf(key_valid), pa.py_buffer(np.ascontiguousarray(key_off, np.int32)),
                                                   pa.py_buffer(np.ascontiguousarray(key_bytes, np.uint8))])
    occ = pa.array(np.where(np.ones(n, bool) if ts_valid is None else ~_bitmap_to_mask(ts_valid, n), ts, 0), pa.int64())
    barrier = pa.array(["no_barrier"] * n, pa.utf8())
    meta = pa.StructArray.from_arrays([barrier, ts_arr], fields=list(canonical_schema().field(3).type))
    return pa.RecordBatch.from_arrays([occ, val_arr, key_arr, meta], schema=canonical_schema())


class DeviceBatches:
    """Synthetic sensor batches generated directly in device memory (dnz_synth_generate).  int_keys: Int64 keys equal to the key
    id (the ids of the "sensor_<id>" keys of the default stream), key_off = NULL."""

    def __init__(self, n_rows, batch_rows=65536, *, row0=0, seed=42, groups=1000, rows_per_ms=1000,
                 t0_ms=1_700_000_000_000, uuid_keys=False, device=0, key_mul=1, key_add=0, int_keys=False):
        assert not (uuid_keys and int_keys)
        L = lib()
        self.n_batches = (n_rows + batch_rows - 1) // batch_rows
        self.n_rows = n_rows
        self.array = (DeviceBatchC * self.n_batches)()
        self._arena = C.c_void_p()
        kind = SYNTH_INT64_KEYS if int_keys else SYNTH_UUID_KEYS if uuid_keys else SYNTH_SENSOR_KEYS
        rc = L.dnz_synth_generate(device, row0, n_rows, batch_rows, seed, groups, rows_per_ms, t0_ms, kind,
                                  key_mul, key_add, C.byref(self._arena), self.array, self.n_batches)
        if rc != 0:
            raise DnzError(rc, L.dnz_window_last_error(None).decode())
        self.algorithmic_bytes = int(L.dnz_synth_bytes(self._arena))

    def free(self):
        if self._arena:
            lib().dnz_synth_free(self._arena)
            self._arena = C.c_void_p()

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


class GpuStreamingWindow:
    """One partition of the GPU streaming-window operator (StreamingWindowExec::execute ->
    GroupedWindowAggStream, streaming_window.rs:421-482) with the FilterExec above it fused in.

    aggs: list of (kind, input column name, alias); filt: (alias, op, literal) or None."""

    def __init__(self, schema: pa.Schema, key, aggs, window_ms, slide_ms=0, filt=None, *, device=0, flags=0,
                 expected_groups=0, max_rows_per_launch=0, cuda_stream=None, timestamp=None):
        self._L = lib()
        self._h = C.c_void_p()
        names = schema.names
        self._key_dtype = INT_KEY_DTYPES.get(schema.field(key).type) if key is not None else None   # None: Utf8 keys
        self._aliases = [a[2].encode() for a in aggs]
        arr = (_Agg * len(aggs))(*[_Agg(AGG_KINDS[k], names.index(col), al) for (k, col, _), al in zip(aggs, self._aliases)])
        ts_source, ts_column, ts_format = timestamp if timestamp else (0, 0, None)      # (TS_* kind, column name, chrono format)
        self._ts_format = ts_format.encode() if ts_format else None
        cfg = _Config(ABI_VERSION, device, NO_KEY if key is None else names.index(key), len(aggs), arr, int(window_ms), int(slide_ms or 0), 0, 0, 0, flags, 0.0,
                      expected_groups, max_rows_per_launch, cuda_stream, ts_source, names.index(ts_column) if ts_source else 0, self._ts_format)
        if filt is not None:
            alias, op, lit = filt
            cfg.has_filter, cfg.filter_agg, cfg.filter_op, cfg.filter_literal = 1, [a[2] for a in aggs].index(alias), OPS[op], float(lit)
        cs = ArrowSchemaC()
        schema._export_to_c(C.addressof(cs))
        try:
            rc = self._L.dnz_window_create(C.byref(cfg), C.byref(cs), C.byref(self._h))
        finally:
            if cs.release:
                C.CFUNCTYPE(None, C.POINTER(ArrowSchemaC))(cs.release)(C.byref(cs))
        if rc != 0:
            raise DnzError(rc, self._L.dnz_window_last_error(None).decode())

    def _check(self, rc):
        if rc != 0:
            raise DnzError(rc, self._L.dnz_window_last_error(self._h).decode())

    def push(self, batch: pa.RecordBatch):
        ca = ArrowArrayC()
        batch._export_to_c(C.addressof(ca))
        rc = self._L.dnz_window_push(self._h, C.byref(ca))
        if ca.release:   # not moved (error path)
            C.CFUNCTYPE(None, C.POINTER(ArrowArrayC))(ca.release)(C.byref(ca))
        self._check(rc)

    def push_device(self, batches: DeviceBatches | None = None, array=None, n=None):
        arr = batches.array if batches is not None else array
        cnt = batches.n_batches if batches is not None else n
        self._check(self._L.dnz_window_push_device(self._h, arr, cnt))

    def poll(self) -> pa.RecordBatch:
        ca, cs, has = ArrowArrayC(), ArrowSchemaC(), C.c_int32(0)
        self._check(self._L.dnz_window_poll(self._h, C.byref(ca), C.byref(cs), C.byref(has)))
        return pa.RecordBatch._import_from_c(C.addressof(ca), C.addressof(cs))

    def poll_ready(self) -> pa.RecordBatch:
        ca, cs, has = ArrowArrayC(), ArrowSchemaC(), C.c_int32(0)
        self._check(self._L.dnz_window_poll_ready(self._h, C.byref(ca), C.byref(cs), C.byref(has)))
        return pa.RecordBatch._import_from_c(C.addressof(ca), C.addressof(cs))

    def poll_device(self) -> DeviceResultC:
        r = DeviceResultC()
        self._check(self._L.dnz_window_poll_device(self._h, C.byref(r)))
        return r

    def poll_device_ready(self) -> DeviceResultC:
        r = DeviceResultC()
        self._check(self._L.dnz_window_poll_device_ready(self._h, C.byref(r)))
        return r

    def fetch_device_result(self, r: DeviceResultC, max_keys=None) -> dict:
        """Copy a device-resident result to host arrays (test helper); keys are materialised for the first max_keys rows.
        Integer keys (key_off == NULL): "key" holds Python ints (None for the NULL key) and "key_values" the value array."""
        n = r.n_rows

        def get(ptr, dt, m):
            a = np.empty(m, dt)
            if m:
                rc = self._L.dnz_memcpy(a.ctypes.data, ptr, a.nbytes, 2)
                if rc:
                    raise DnzError(rc, "memcpy")
            return a
        if not r.key_off:
            dt = np.dtype(self._key_dtype)
            assert self._key_dtype is not None and r.key_bytes_len == n * dt.itemsize, "integer key result of another layout"
            vals = get(r.key_bytes, dt, n)
            kv = get(r.key_valid, np.uint8, n)
            nk = n if max_keys is None else min(n, max_keys)
            return {"key": [int(vals[i]) if kv[i] else None for i in range(nk)], "key_values": vals, "key_valid": kv,
                    "count": get(r.count, np.int64, n), "min": get(r.min, np.float64, n), "max": get(r.max, np.float64, n),
                    "avg": get(r.avg, np.float64, n), "sum": get(r.sum, np.float64, n), "agg_valid": get(r.agg_valid, np.uint8, n),
                    "window_start": get(r.window_start_ms, np.int64, n), "window_end": get(r.window_end_ms, np.int64, n)}
        off = np.concatenate([get(r.key_off, np.int32, n), np.array([r.key_bytes_len], np.int32)])
        kb_arr = get(r.key_bytes, np.uint8, r.key_bytes_len)
        kb = kb_arr.tobytes() if (max_keys is None or max_keys > 0) else b""
        kv = get(r.key_valid, np.uint8, n)
        av = get(r.agg_valid, np.uint8, n)
        nk = n if max_keys is None else min(n, max_keys)
        return {"key": [kb[off[i]:off[i + 1]] if kv[i] else None for i in range(nk)], "key_off": off, "key_bytes": kb_arr, "key_valid": kv,
                "count": get(r.count, np.int64, n), "min": get(r.min, np.float64, n), "max": get(r.max, np.float64, n),
                "avg": get(r.avg, np.float64, n), "sum": get(r.sum, np.float64, n), "agg_valid": av,
                "window_start": get(r.window_start_ms, np.int64, n), "window_end": get(r.window_end_ms, np.int64, n)}

    def checkpoint(self) -> bytes:
        """Serialised device state (dictionary, open panes, stream clock): dnz_window_checkpoint."""
        blob, n = C.c_void_p(), C.c_int64(0)
        self._check(self._L.dnz_window_checkpoint(self._h, C.byref(blob), C.byref(n)))
        try:
            return C.string_at(blob, n.value)
        finally:
            self._L.dnz_blob_free(blob)

    def restore(self, blob: bytes):
        self._check(self._L.dnz_window_restore(self._h, blob, len(blob)))

    def flush(self, watermark_ms: int):
        self._check(self._L.dnz_window_flush(self._h, int(watermark_ms)))

    def stats(self) -> dict:
        s = StatsC()
        self._L.dnz_window_stats(self._h, C.byref(s))
        return s.as_dict()

    def reset_stats(self):
        self._L.dnz_window_reset_stats(self._h)

    @property
    def watermark(self):
        v = int(self._L.dnz_window_watermark(self._h))
        return None if v == -(2 ** 63) else v

    def reserve_input(self, bytes_per_launch):
        self._check(self._L.dnz_window_reserve_input(self._h, int(bytes_per_launch)))

    def set_exchange(self, rank, world):
        self._check(self._L.dnz_window_set_exchange(self._h, rank, world))
        self._world = world

    def process(self):
        """Aggregate everything queued; returns the local watermark (None if there is none yet)."""
        v = C.c_int64(0)
        self._check(self._L.dnz_window_process(self._h, C.byref(v)))
        return None if v.value == -(2 ** 63) else v.value

    def export_partials(self, watermark_ms):
        """-> dict(entries=(device ptr, n), keys=(device ptr, bytes), owner_counts, owner_key_bytes, pane_lo, pane_hi)."""
        p = PartialsC()
        self._check(self._L.dnz_window_export_partials(self._h, -(2 ** 63) if watermark_ms is None else int(watermark_ms), C.byref(p)))
        w = self._world
        return dict(entries=(p.entries or 0, int(p.n_entries)), keys=(p.key_bytes or 0, int(p.key_bytes_len)),
                    owner_counts=[int(p.owner_counts[i]) for i in range(w)], owner_key_bytes=[int(p.owner_key_bytes[i]) for i in range(w)],
                    pane_lo=int(p.pane_lo), pane_hi=int(p.pane_hi))

    def import_partials(self, entries_ptr, src_counts, keys_ptr, src_key_bytes, pane_lo, pane_hi):
        w = self._world
        sc = (C.c_int64 * w)(*[int(x) for x in src_counts]); sk = (C.c_int64 * w)(*[int(x) for x in src_key_bytes])
        self._check(self._L.dnz_window_import_partials(self._h, C.c_void_p(entries_ptr), sc, C.c_void_p(keys_ptr), sk, int(pane_lo), int(pane_hi)))

    def close(self):
        if getattr(self, "_h", None):
            self._L.dnz_window_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class ExchangeGroup:
    """One rank of the fused pane exchange (dnz_group): the library owns the communicator -- peer mappings of every rank's receive
    ring (CUDA IPC), remote-atomic reservations, P2P stores over NVLink, flag signalling; see include/dnz_gpu.h.

    ExchangeGroup.create(rank, world, device, allgather)  one rank per process; `allgather(bytes) -> list of bytes` is the
                                                          rendezvous helper (e.g. torch.distributed), used at creation only
    ExchangeGroup.create_local(devices)                   all ranks in this process (tests)"""

    def __init__(self, handle, rank, world, keep=None):
        self._L, self._h, self.rank, self.world, self._keep = lib(), C.c_void_p(handle), rank, world, keep

    @staticmethod
    def create(rank, world, device, allgather, ring_entries=0, ring_key_bytes=0):
        L = lib()

        def cb(_ctx, send, recv, nbytes):
            try:
                parts = allgather(C.string_at(send, nbytes))
                C.memmove(recv, b"".join(parts), nbytes * len(parts))
                return 0
            except Exception:          # noqa: BLE001 -- reported as a failed rendezvous by the library
                return 1
        fn = ALLGATHER_FN(cb)
        cfg = GroupConfigC(ABI_VERSION, rank, world, device, ring_entries, ring_key_bytes)
        h = C.c_void_p()
        rc = L.dnz_group_create(C.byref(cfg), fn, None, C.byref(h))
        if rc != 0:
            raise DnzError(rc, L.dnz_window_last_error(None).decode())
        return ExchangeGroup(h.value, rank, world, keep=fn)

    @staticmethod
    def create_local(devices, ring_entries=0, ring_key_bytes=0):
        L = lib()
        n = len(devices)
        dv = (C.c_int32 * n)(*devices)
        out = (C.c_void_p * n)()
        rc = L.dnz_group_create_local(n, dv, ring_entries, ring_key_bytes, out)
        if rc != 0:
            raise DnzError(rc, L.dnz_window_last_error(None).decode())
        return [ExchangeGroup(out[r], r, n) for r in range(n)]

    def _check(self, rc, w):
        if rc != 0:
            raise DnzError(rc, self._L.dnz_window_last_error(w._h).decode())

    def attach(self, w: GpuStreamingWindow):
        self._check(self._L.dnz_group_attach(self._h, w._h), w)
        w._world = self.world

    def step_begin(self, w):
        self._check(self._L.dnz_group_step_begin(self._h, w._h), w)

    def step_pack(self, w):
        self._check(self._L.dnz_group_step_pack(self._h, w._h), w)

    def step_finish(self, w):
        v = C.c_int64(0)
        self._check(self._L.dnz_group_step_finish(self._h, w._h, C.byref(v)), w)
        return None if v.value == -(2 ** 63) else v.value

    def step(self, w):
        """One collective exchange step; returns the global watermark (None before every rank has one)."""
        v = C.c_int64(0)
        self._check(self._L.dnz_group_step(self._h, w._h, C.byref(v)), w)
        return None if v.value == -(2 ** 63) else v.value

    def flush(self, w):
        """COLLECTIVE end of stream: process + three steps (the protocol is pipelined over three steps): everything pushed so far
        is exchanged and the windows it closes are emitted."""
        v = C.c_int64(0)
        self._check(self._L.dnz_group_flush(self._h, w._h, C.byref(v)), w)
        return None if v.value == -(2 ** 63) else v.value

    def close(self):
        if self._h:
            self._L.dnz_group_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
