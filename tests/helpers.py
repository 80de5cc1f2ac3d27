"""Shared test helpers: row-list <-> columnar batches, random streams, row comparison."""
import math
import struct

import numpy as np

from oracle import Batch


def pack_bitmap(flags):
    n = len(flags)
    bm = np.zeros((n + 7) // 8 + 1, np.uint8)
    for i, f in enumerate(flags):
        if f:
            bm[i >> 3] |= 1 << (i & 7)
    return bm


def rows_to_batch(rows, force_validity=False) -> Batch:
    """rows: list of (ts|None, val|None, key(bytes)|None)."""
    n = len(rows)
    ts = np.array([r[0] if r[0] is not None else 0 for r in rows], np.int64).reshape(n)
    val = np.array([r[1] if r[1] is not None else 0.0 for r in rows], np.float64).reshape(n)
    off = np.zeros(n + 1, np.int32)
    chunks = []
    for i, r in enumerate(rows):
        k = r[2] if r[2] is not None else b""
        chunks.append(k)
        off[i + 1] = off[i] + len(k)
    kb = np.frombuffer(b"".join(chunks) + b"\0" * 16, np.uint8).copy()
    b = Batch(ts=ts, val=val, key_off=off, key_bytes=kb)
    if force_validity or any(r[0] is None for r in rows):
        b.ts_valid = pack_bitmap([r[0] is not None for r in rows])
    if force_validity or any(r[1] is None for r in rows):
        b.val_valid = pack_bitmap([r[1] is not None for r in rows])
    if force_validity or any(r[2] is None for r in rows):
        b.key_valid = pack_bitmap([r[2] is not None for r in rows])
    return b


def batch_to_rows(b: Batch):
    out = []
    kb = b.key_bytes.tobytes()
    for i in range(b.n):
        def ok(bm):
            return bm is None or (bm[i >> 3] >> (i & 7)) & 1
        out.append((int(b.ts[i]) if ok(b.ts_valid) else None, float(b.val[i]) if ok(b.val_valid) else None,
                    kb[b.key_off[i]:b.key_off[i + 1]] if ok(b.key_valid) else None))
    return out


def bits(d):
    return None if d is None else struct.pack("<d", d)


def assert_rows_equal(got, want, rel=1e-9, check_seq=False):
    """count/min/max bit-exact, avg within `rel` relative (north_star tolerance)."""
    def key(r):
        return (r[0], r[1], r[2] is None, r[2] or b"", (r[7] if check_seq else 0))
    g, w = sorted(got, key=key), sorted(want, key=key)
    assert len(g) == len(w), f"row count {len(g)} != {len(w)}"
    for a, b in zip(g, w):
        assert a[:4] == b[:4], f"{a} != {b}"
        assert bits(a[4]) == bits(b[4]), f"min differs: {a} != {b}"
        assert bits(a[5]) == bits(b[5]), f"max differs: {a} != {b}"
        if a[6] is None or b[6] is None:
            assert a[6] is None and b[6] is None, f"{a} != {b}"
        elif math.isnan(b[6]) or math.isinf(b[6]):
            assert bits(a[6]) == bits(b[6]) or (math.isnan(a[6]) and math.isnan(b[6])), f"{a} != {b}"
        else:
            assert abs(a[6] - b[6]) <= rel * max(abs(b[6]), 1e-300), f"avg differs: {a} != {b}"
        if check_seq:
            assert a[7] == b[7], f"emit seq differs: {a} != {b}"


def random_stream(rng, n_batches, rows_per_batch, n_keys, t0=1_700_000_000_000, span_ms=400, jitter_ms=0,
                  null_frac=0.0, special_vals=False, ragged=False, late_every=0, late_shift_ms=0):
    """Mostly in-order batches of (ts,val,key) rows; jitter_ms>0 makes batches overlap / arrive late."""
    batches = []
    t = t0
    for bi in range(n_batches):
        n = int(rng.integers(0, rows_per_batch + 1)) if ragged else rows_per_batch
        rows = []
        back = late_shift_ms if (late_every and bi % late_every == late_every - 1) else 0   # a whole batch arrives late
        for _ in range(n):
            ts = t - back + int(rng.integers(0, span_ms)) - (int(rng.integers(0, jitter_ms)) if jitter_ms else 0)
            k = int(rng.integers(0, n_keys))
            key = b"sensor_%d" % k if k % 7 else b"k" * (k % 40)   # some long / empty keys
            val = float(rng.random() * 115.0)
            if special_vals:
                val = [val, 0.0, -0.0, float("nan"), float("inf"), float("-inf"), 1e308, -1e308][int(rng.integers(0, 8))]
            r = [ts, val, key]
            if null_frac:
                for j in range(3):
                    if rng.random() < null_frac:
                        r[j] = None
            rows.append(tuple(r))
        if rows and all(r[0] is None for r in rows):
            rows[0] = (t, rows[0][1], rows[0][2])
        batches.append(rows)
        t += span_ms
    return batches


# ---------------------------------------------------------------------------------------------
# GPU-side helpers (import denormalized_b200 lazily so the CPU suite does not need the CUDA library)
DEFAULT_AGGS = [("count", "reading", "count"), ("min", "reading", "min"), ("max", "reading", "max"), ("avg", "reading", "average")]


def to_record_batch(b: Batch):
    from denormalized_b200 import make_record_batch
    return make_record_batch(b.ts, b.val, b.key_off, b.key_bytes, b.ts_valid, b.val_valid, b.key_valid)


SUM_AGGS = DEFAULT_AGGS + [("sum", "reading", "sum")]


def same_f64(a, b):
    """None == None, any NaN == any NaN, otherwise the same bits (+0.0 != -0.0)."""
    if a is None or b is None:
        return a is None and b is None
    if math.isnan(a) or math.isnan(b):
        return math.isnan(a) and math.isnan(b)
    return bits(a) == bits(b)


def assert_rows_exact(got, want, check_seq=False):
    """Rows with sum at index 8 (OracleWindow.results(with_sum=True)): count / min / max / avg / sum all bit-exact, NaN as NaN."""
    def key(r):
        return (r[0], r[1], r[2] is None, r[2] or b"", (r[7] if check_seq else 0), r[3], bits(r[8]) or b"")
    g, w = sorted(got, key=key), sorted(want, key=key)
    assert len(g) == len(w), f"row count {len(g)} != {len(w)}"
    for a, b in zip(g, w):
        assert a[:4] == b[:4] and (not check_seq or a[7] == b[7]), f"{a} != {b}"
        for i, name in ((4, "min"), (5, "max"), (6, "avg"), (8, "sum")):
            assert same_f64(a[i], b[i]), f"{name} differs: {a} != {b}"


def agg_rows(rb, aliases=("count", "min", "max", "average", "sum"), seq=0):
    """Emitted RecordBatch -> rows (window_start, window_end, key, count, min, max, avg, seq, sum) read by the aliases of count, min,
    max, avg and sum; the key is None when the batch has no key column (ungrouped), bytes otherwise (an integer v as str(v))."""
    names = rb.schema.names
    col = {name: rb.column(i) for i, name in enumerate(names)}
    n = rb.num_rows
    keyed = len(names) > len(aliases) + 2
    keys = col[names[0]].cast("string").cast("binary").to_pylist() if keyed else [None] * n      # integer keys as str(v)
    c, mn, mx, av, sm = (col[a].to_pylist() for a in aliases)
    ws = col["window_start_time"].cast("int64").to_pylist()
    we = col["window_end_time"].cast("int64").to_pylist()
    return [(ws[i], we[i], keys[i], c[i], mn[i], mx[i], av[i], seq, sm[i]) for i in range(n)]


def record_batch_rows(rb, seq=0):
    """Emitted RecordBatch (key|count|min|max|average|window_start_time|window_end_time) -> oracle-style row tuples."""
    cols = {name: rb.column(i) for i, name in enumerate(rb.schema.names)}
    keys = cols[rb.schema.names[0]].cast("binary").to_pylist()
    cnt = cols["count"].to_pylist()
    mn, mx, av = cols["min"].to_pylist(), cols["max"].to_pylist(), cols["average"].to_pylist()
    ws = cols["window_start_time"].cast("int64").to_pylist()
    we = cols["window_end_time"].cast("int64").to_pylist()
    return [(ws[i], we[i], keys[i], cnt[i], mn[i], mx[i], av[i], seq) for i in range(rb.num_rows)]


def gpu_window(L, S=0, filt=None, **kw):
    from denormalized_b200 import GpuStreamingWindow, canonical_schema
    return GpuStreamingWindow(canonical_schema(), "sensor_name", DEFAULT_AGGS, L, S, filt, **kw)


def run_gpu(batches, L, S=0, filt=None, per_batch_poll=True, **kw):
    """batches: list of oracle.Batch.  Returns rows (emit seq = index of the push that emitted them when per_batch_poll)."""
    w = gpu_window(L, S, filt, **kw)
    rows = []
    for i, b in enumerate(batches):
        w.push(to_record_batch(b))
        if per_batch_poll:
            rows += record_batch_rows(w.poll(), i)
    if not per_batch_poll:
        rows += record_batch_rows(w.poll(), 0)
    st = w.stats()
    w.close()
    return rows, st


def run_oracle_batches(batches, L, S=0, filt=None):
    from oracle import OracleWindow
    o = OracleWindow(L, S, filt)
    for b in batches:
        o.push(b)
    return o.results()


# ---------------------------------------------------------------------------------------------
# kernel configurations: name -> (flags, expected_groups).  count / min / max are bit-exact by contract, so every configuration
# must emit the same bits for the same stream.
FLAG_FORCE_GENERIC, FLAG_NO_HINTS, FLAG_NO_QUEUE, FLAG_NO_PRIVATE, FLAG_SYNCHRONOUS = 2, 4, 8, 16, 32
KERNEL_PATHS = {
    "private": (0, 16),                          # 1024 groups: per-CTA private pane copies, no min/max hints
    "hinted": (0, 0),                            # 131072 groups: hints in the dictionary slots, no private copies
    "hinted_noqueue": (FLAG_NO_QUEUE, 0),        # colliding probes loop in place instead of the per-warp retry queue
    "nohints": (FLAG_NO_HINTS, 0),
    "noprivate_small": (FLAG_NO_PRIVATE, 16),    # small table without private copies: hints on a 1024-group table
    "generic": (FLAG_FORCE_GENERIC, 0),          # no TMA-staged tiles
    "sync": (FLAG_SYNCHRONOUS, 0),               # no speculative pipeline
}


def _row_order(r):
    return (r[0], r[2] is None, r[2] or b"", r[7])


def _row_bits(r):
    return (r[0], r[1], r[2], r[3], bits(r[4]), bits(r[5]), r[6] is None)


def run_paths(batches, L, S=0, filt=None, names=tuple(KERNEL_PATHS), per_batch_poll=False, want=None, **kw):
    """Runs `batches` under each named kernel configuration, compares each with the oracle and checks that count / min / max
    and the null flags are bit-identical between the configurations.  Returns {name: stats}."""
    if want is None:
        want = run_oracle_batches(batches, L, S, filt)
    stats, ref = {}, None
    for name in names:
        flags, eg = KERNEL_PATHS[name]
        got, st = run_gpu(batches, L, S, filt, per_batch_poll=per_batch_poll, flags=flags, expected_groups=eg, **kw)
        try:
            assert_rows_equal(got, want, check_seq=per_batch_poll)
        except AssertionError as e:
            raise AssertionError(f"kernel path {name!r}: {e}") from None
        got_bits = [_row_bits(r) for r in sorted(got, key=_row_order)]
        if ref is None:
            ref = (name, got_bits)
        else:
            assert got_bits == ref[1], f"kernel paths {ref[0]!r} and {name!r} emit different bits"
        stats[name] = st
    return stats


def columns_to_batch(ts, val, keys) -> Batch:
    """Batch from a timestamp array, a value array and a list of key bytes (no nulls)."""
    lens = np.fromiter((len(k) for k in keys), np.int64, len(keys))
    off = np.zeros(len(keys) + 1, np.int32)
    np.cumsum(lens, out=off[1:])
    kb = np.frombuffer(b"".join(keys) + b"\0" * 16, np.uint8).copy()
    return Batch(ts=np.ascontiguousarray(ts, np.int64), val=np.ascontiguousarray(val, np.float64), key_off=off, key_bytes=kb)


def record_batch_table(rb, tag):
    """Emitted RecordBatch -> the pyarrow Table layout of result_table(.., tag) (for assert_tables_equal)."""
    import pyarrow as pa
    col = {name: rb.column(i) for i, name in enumerate(rb.schema.names)}

    def f64_bits(name):
        return pa.array(np.asarray(col[name].fill_null(0.0).to_numpy(zero_copy_only=False), np.float64).view(np.int64))
    return pa.table({"ws": col["window_start_time"].cast(pa.int64()), "key": col[rb.schema.names[0]].cast(pa.binary()),
                     "count_" + tag: col["count"].cast(pa.int64()), "min_" + tag: f64_bits("min"), "max_" + tag: f64_bits("max"),
                     "avg_" + tag: pa.array(np.asarray(col["average"].fill_null(0.0).to_numpy(zero_copy_only=False), np.float64)),
                     "null_" + tag: col["min"].is_null()})


# ---------------------------------------------------------------------------------------------
# NumPy port of the dictionary hash of keys <= 16 B (hash_words / hash_inline in denormalized_b200/csrc/dnz_device.cuh).
# tests/test_hash_port.py pins it against the header.
def _rotl32(x, r):
    return (x << np.uint32(r)) | (x >> np.uint32(32 - r))


def hash_words(w0, w1, w2, w3, length):
    """32-bit hash of four zero-padded little-endian key words and the key length (uint32 arrays or scalars)."""
    w0, w1, w2, w3, length = (np.asarray(x, np.uint32) for x in (w0, w1, w2, w3, length))
    with np.errstate(over="ignore"):
        a, b, c = w1 * np.uint32(0xC2B2AE35), w2 * np.uint32(0x27D4EB2F), w3 * np.uint32(0x165667B1)
        h = w0 * np.uint32(0x85EBCA6B) + _rotl32(a, 13) + _rotl32(b, 21) + _rotl32(c, 5) + length * np.uint32(0x9E3779B1)
        h = h ^ (h >> np.uint32(16)); h = h * np.uint32(0x85EBCA6B)
        h = h ^ (h >> np.uint32(13)); h = h * np.uint32(0xC2B2AE35)
        h = h ^ (h >> np.uint32(16))
    return h


def hash_inline(k0, k1, length):
    k0, k1 = np.asarray(k0, np.uint64), np.asarray(k1, np.uint64)
    m = np.uint64(0xFFFFFFFF)
    return hash_words(k0 & m, k0 >> np.uint64(32), k1 & m, k1 >> np.uint64(32), length)


def key_words(keys):
    """(n, 4) uint32 words of keys <= 16 B, zero padded, as the dictionary stores them."""
    assert all(len(k) <= 16 for k in keys)
    return np.frombuffer(b"".join(k.ljust(16, b"\0") for k in keys), "<u4").reshape(len(keys), 4)


def hash_keys(keys):
    w = key_words(keys)
    return hash_words(w[:, 0], w[:, 1], w[:, 2], w[:, 3], np.fromiter((len(k) for k in keys), np.uint32, len(keys)))


# ---------------------------------------------------------------------------------------------
# large results: sort-free comparison (hash join on (window_start, key)) of column arrays instead of Python row tuples
def _binary_array(key_off, key_bytes, key_isnull=None):
    import pyarrow as pa
    n = len(key_off) - 1
    off = np.ascontiguousarray(key_off, np.int32)
    kb = np.ascontiguousarray(key_bytes, np.uint8)
    if len(kb) == 0:
        kb = np.zeros(1, np.uint8)
    arr = pa.Array.from_buffers(pa.binary(), n, [None, pa.py_buffer(off), pa.py_buffer(kb)])
    if key_isnull is not None and np.any(key_isnull):
        arr = pa.array([None if key_isnull[i] else arr[i].as_py() for i in range(n)], pa.binary()) if n < 100_000 else \
            pa.compute.if_else(pa.array(np.asarray(key_isnull, bool)), pa.scalar(None, pa.binary()), arr)
    return arr


def result_table(a, tag):
    """dict of column arrays (oracle._arrays or fetch_device_result layout) -> pyarrow Table with columns suffixed by `tag`."""
    import pyarrow as pa
    n = len(a["count"])
    if "key_isnull" in a:
        knull, anull = a["key_isnull"], a["agg_isnull"]
        ws = a["window_start"]
    else:
        knull, anull = (np.asarray(a["key_valid"]) == 0), (np.asarray(a["agg_valid"]) == 0)
        ws = a["window_start"]
    key = _binary_array(a["key_off"][: n + 1], a["key_bytes"], knull)
    anull = np.asarray(anull, bool)
    return pa.table({"ws": pa.array(np.asarray(ws, np.int64)), "key": key,
                     "count_" + tag: pa.array(np.asarray(a["count"], np.int64)),
                     "min_" + tag: pa.array(np.asarray(a["min"], np.float64).view(np.int64)),      # bit patterns: compared exactly
                     "max_" + tag: pa.array(np.asarray(a["max"], np.float64).view(np.int64)),
                     "avg_" + tag: pa.array(np.asarray(a["avg"], np.float64)),
                     "null_" + tag: pa.array(anull)})


def assert_tables_equal(got, want, rel=1e-9):
    """got / want: pyarrow Tables from result_table(.., "g") / (.., "w").  Rows must match one to one on (window_start, key)
    [valid for in-order streams: every (window, key) is emitted once]; count/min/max bit-exact, avg within `rel`."""
    assert got.num_rows == want.num_rows, f"row count {got.num_rows} != {want.num_rows}"
    if got.num_rows == 0:
        return 0
    j = got.join(want, keys=["ws", "key"], join_type="inner")
    assert j.num_rows == got.num_rows, f"only {j.num_rows} of {got.num_rows} (window, key) pairs match"
    c = {name: j.column(name).to_numpy(zero_copy_only=False) for name in j.column_names if name not in ("ws", "key")}
    assert np.array_equal(c["count_g"], c["count_w"]), "count differs"
    assert np.array_equal(c["null_g"], c["null_w"]), "null aggregates differ"
    ok = ~c["null_w"].astype(bool)
    assert np.array_equal(c["min_g"][ok], c["min_w"][ok]), "min differs (bit pattern)"
    assert np.array_equal(c["max_g"][ok], c["max_w"][ok]), "max differs (bit pattern)"
    ag, aw = c["avg_g"][ok], c["avg_w"][ok]
    fin = np.isfinite(aw)
    assert np.all(np.abs(ag[fin] - aw[fin]) <= rel * np.maximum(np.abs(aw[fin]), 1e-300)), "avg differs beyond the tolerance"
    assert np.array_equal(np.isnan(ag[~fin]), np.isnan(aw[~fin])) and np.array_equal(ag[~fin][~np.isnan(ag[~fin])], aw[~fin][~np.isnan(aw[~fin])])
    return j.num_rows


def concat_arrays(parts):
    """Concatenate several column-array dicts (e.g. the oracle's partitions, or several polls) into one."""
    parts = [p for p in parts if len(p["count"])]
    if not parts:
        z = np.zeros(0)
        return {"key_off": np.zeros(1, np.int32), "key_bytes": np.zeros(0, np.uint8), "key_isnull": np.zeros(0, np.uint8), "count": z.astype(np.int64),
                "min": z, "max": z, "avg": z, "agg_isnull": np.zeros(0, np.uint8), "window_start": z.astype(np.int64)}
    out = {}
    offs, base = [np.zeros(1, np.int64)], 0
    for p in parts:
        n = len(p["count"])
        o = np.asarray(p["key_off"][: n + 1], np.int64)
        offs.append(o[1:] - o[0] + base)
        base += int(o[-1] - o[0])
    tot = np.concatenate(offs)
    assert tot[-1] < 2 ** 31, "concatenated key bytes exceed 2 GiB: compare in pieces"
    out["key_off"] = tot.astype(np.int32)
    out["key_bytes"] = np.concatenate([np.asarray(p["key_bytes"], np.uint8)[int(p["key_off"][0]): int(p["key_off"][len(p["count"])])] for p in parts])
    for k_out, k_a, k_b in [("key_isnull", "key_isnull", "key_valid"), ("agg_isnull", "agg_isnull", "agg_valid")]:
        out[k_out] = np.concatenate([np.asarray(p[k_a], np.uint8) if k_a in p else (np.asarray(p[k_b]) == 0).astype(np.uint8) for p in parts])
    for k in ("count", "min", "max", "avg", "window_start") + (("sum",) if all("sum" in p for p in parts) else ()):
        out[k] = np.concatenate([np.asarray(p[k]) for p in parts])
    return out


def host_stream(n_rows, *, groups, rows_per_ms, uuid_keys=False, batch_rows=65536, seed=42, key_mul=1, key_add=0, threads=None, extra_columns=False):
    """Batches [0, n_rows) of the synthetic sensor stream, generated with a thread pool (ctypes releases the GIL)."""
    import os
    from concurrent.futures import ThreadPoolExecutor
    from oracle import synth_batch
    starts = list(range(0, n_rows, batch_rows))
    with ThreadPoolExecutor(max_workers=threads or min(32, os.cpu_count() or 1)) as ex:
        return list(ex.map(lambda r0: synth_batch(r0, min(batch_rows, n_rows - r0), seed=seed, groups=groups, rows_per_ms=rows_per_ms, uuid_keys=uuid_keys,
                                                  key_mul=key_mul, key_add=key_add, extra_columns=extra_columns), starts))


def oracle_mt_arrays(batches, L, S=0, filt=None, partitions=None):
    """Run the multi-threaded oracle over `batches`; returns one concatenated column-array dict."""
    import os
    from oracle import OracleMT
    m = OracleMT(L, S, filt, partitions=partitions or min(32, os.cpu_count() or 1))
    m.push_many(batches)
    parts = m.results_arrays()
    m.close()
    return concat_arrays(parts)
