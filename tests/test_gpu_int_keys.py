"""Integer group keys (Arrow Int64 / Int32 / UInt64 / UInt32) through the fixed-width instantiations of k_aggregate and every path
around them: generic and deferred rows, the retry queue, dictionary growth, emission, Arrow and device export, the checkpoint and
the pane exchange (run on an H100 with -m gpu).

The oracle groups byte-string keys.  It is fed str(v).encode() for every key v -- an injective map that keeps NULL as NULL, so
the grouping, and with it every aggregate, is the same -- and the emitted integer keys are mapped the same way before comparing:
count / min / max bit-exact, avg within 1e-9 relative."""
import ctypes as C
import math
import zlib

import numpy as np
import pyarrow as pa
import pyarrow.compute as pc
import pytest

from oracle import Batch
from tests.helpers import (DEFAULT_AGGS, KERNEL_PATHS, assert_rows_equal, assert_tables_equal, bits, hash_inline, host_stream,
                           oracle_mt_arrays, pack_bitmap, result_table, run_oracle_batches)

pytestmark = pytest.mark.gpu
T0 = 1_700_000_000_000
TILE = 416                                          # denormalized_b200/csrc/dnz_kernels.h
INT_KEY_TAG = 0x494E544B45594B31                    # denormalized_b200/csrc/dnz_device.cuh: int_key
TYPES = {"int64": pa.int64(), "int32": pa.int32(), "uint64": pa.uint64(), "uint32": pa.uint32()}
FLAG_SCALAR_PROBE, FLAG_STAGE_TS = 64, 128          # include/dnz_gpu.h
PATHS = {**KERNEL_PATHS, "scalar_probe": (FLAG_SCALAR_PROBE, 0), "stage_ts": (FLAG_STAGE_TS, 0)}
SENTINEL_KEY = 424242


def edge_keys(typ):
    """0, -1, MIN and MAX of the type (the unsigned types: 0, 1, MAX - 1, MAX; MAX has the bits of -1)."""
    info = np.iinfo(typ.to_pandas_dtype())
    ks = [0, 1, int(info.max), int(info.max) - 1, int(info.min)]
    if info.min < 0:
        ks += [-1, int(info.min) + 1]
    return sorted(set(ks))


# ---------------------------------------------------------------------------------------------------------------- batches
def int_schema(typ, key_nullable=True):
    from denormalized_b200 import canonical_schema
    meta = canonical_schema().field(3)
    return pa.schema([pa.field("id", typ, nullable=key_nullable), pa.field("reading", pa.float64()), meta])


def _meta(ts, ts_valid, n):
    from denormalized_b200 import canonical_schema
    ts_arr = pa.array(ts, pa.timestamp("ms"), mask=None if ts_valid is None else ~ts_valid)
    return pa.StructArray.from_arrays([pa.array(["no_barrier"] * n, pa.utf8()), ts_arr], fields=list(canonical_schema().field(3).type))


class IntBatch:
    """One batch as columns: timestamps, values, integer keys and their validity (bool arrays, None = no nulls)."""

    def __init__(self, ts, val, keys, typ, ts_valid=None, val_valid=None, key_valid=None):
        self.ts, self.val, self.typ = np.asarray(ts, np.int64), np.asarray(val, np.float64), typ
        self.keys = np.asarray(keys, typ.to_pandas_dtype())
        self.ts_valid, self.val_valid, self.key_valid = ts_valid, val_valid, key_valid

    @staticmethod
    def from_rows(rows, typ):
        """rows: (ts|None, val|None, key|None)"""
        n = len(rows)
        tv = np.array([r[0] is not None for r in rows], bool)
        vv = np.array([r[1] is not None for r in rows], bool)
        kv = np.array([r[2] is not None for r in rows], bool)
        return IntBatch([r[0] or 0 for r in rows], [0.0 if r[1] is None else r[1] for r in rows], [r[2] or 0 for r in rows], typ,
                        None if tv.all() else tv, None if vv.all() else vv, None if kv.all() else kv)

    def record_batch(self):
        n = len(self.ts)
        key = pa.array(self.keys, self.typ, mask=None if self.key_valid is None else ~self.key_valid)
        val = pa.array(self.val, pa.float64(), mask=None if self.val_valid is None else ~self.val_valid)
        return pa.RecordBatch.from_arrays([key, val, _meta(self.ts, self.ts_valid, n)], schema=int_schema(self.typ))

    def oracle(self):
        """The same batch with the key v as the byte string str(v)."""
        n = len(self.ts)
        s = pa.array(self.keys, self.typ).cast(pa.string())
        off = np.frombuffer(s.buffers()[1], np.int32, n + 1).copy()
        kb = np.concatenate([np.frombuffer(s.buffers()[2], np.uint8, int(off[-1])), np.zeros(16, np.uint8)])

        def bm(v):
            return None if v is None else pack_bitmap(v.tolist())
        return Batch(ts=self.ts.copy(), val=self.val.copy(), key_off=off, key_bytes=kb, ts_valid=bm(self.ts_valid),
                     val_valid=bm(self.val_valid), key_valid=bm(self.key_valid))


def sentinel(ts, typ):
    return IntBatch([ts], [1.0], [SENTINEL_KEY], typ)


def gpu_int_window(typ, L, S=0, filt=None, **kw):
    from denormalized_b200 import GpuStreamingWindow
    return GpuStreamingWindow(int_schema(typ), "id", DEFAULT_AGGS, L, S, filt, **kw)


def int_rows(rb, typ, seq=0, nullable=True):
    """Emitted RecordBatch -> oracle-style row tuples with the key mapped to str(v).encode()."""
    assert rb.schema.field(0).type == typ and rb.schema.field(0).nullable == nullable, rb.schema
    c = {name: rb.column(i).to_pylist() for i, name in enumerate(rb.schema.names)}
    keys = [None if k is None else str(k).encode() for k in c["id"]]
    ws = rb.column(rb.schema.names.index("window_start_time")).cast(pa.int64()).to_pylist()
    we = rb.column(rb.schema.names.index("window_end_time")).cast(pa.int64()).to_pylist()
    return [(ws[i], we[i], keys[i], c["count"][i], c["min"][i], c["max"][i], c["average"][i], seq) for i in range(rb.num_rows)]


def run_int(batches, typ, L, S=0, filt=None, per_batch_poll=False, **kw):
    w = gpu_int_window(typ, L, S, filt, **kw)
    rows = []
    for i, b in enumerate(batches):
        w.push(b.record_batch())
        if per_batch_poll:
            rows += int_rows(w.poll(), typ, i)
    if not per_batch_poll:
        rows += int_rows(w.poll(), typ)
    st = w.stats()
    w.close()
    return rows, st


def oracle_rows(batches, L, S=0, filt=None):
    return run_oracle_batches([b.oracle() for b in batches], L, S, filt)


def distinct_keys(batches):
    ks = set()
    for b in batches:
        live = np.ones(len(b.ts), bool) if b.ts_valid is None else b.ts_valid
        kv = np.ones(len(b.ts), bool) if b.key_valid is None else b.key_valid
        ks |= {int(x) for x in b.keys[live & kv].tolist()}
        if (live & ~kv).any():
            ks.add(None)
    return ks


def _row_bits(r):
    return (r[0], r[1], r[2] is None, r[2] or b"", r[3], bits(r[4]) or b"", bits(r[5]) or b"", r[6] is None)


def run_every_path(batches, typ, L, S=0, names=tuple(PATHS), want=None, per_batch_poll=False, **kw):
    """Runs the stream under each kernel configuration: parity with the oracle, count / min / max bit-identical across the
    configurations, and one group per distinct key.  Returns {name: stats}."""
    if want is None:
        want = oracle_rows(batches, L, S)
    n_keys = len(distinct_keys(batches))
    stats, ref = {}, None
    for name in names:
        flags, eg = PATHS[name]
        got, st = run_int(batches, typ, L, S, per_batch_poll=per_batch_poll, flags=flags, expected_groups=eg, **kw)
        try:
            assert_rows_equal(got, want, check_seq=per_batch_poll)
        except AssertionError as e:
            raise AssertionError(f"kernel path {name!r}: {e}") from None
        got_bits = sorted(_row_bits(r) for r in got)
        if ref is None:
            ref = (name, got_bits)
        else:
            assert got_bits == ref[1], f"kernel paths {ref[0]!r} and {name!r} emit different bits"
        assert st["groups"] == n_keys, (name, st["groups"], n_keys)
        stats[name] = st
    return stats


def int_stream(rng, typ, n_batches, rows, n_keys, span_ms=300, null_frac=0.0, special_vals=False, late_every=0, late_shift_ms=0,
               hot_zero=0.0):
    """Mostly in-order batches over a key pool that holds the type's edge values; whole batches may arrive late."""
    pool = np.array(sorted(set(edge_keys(typ)) | set(rng.integers(0, 1 << 20, n_keys).tolist())), object)
    out, t = [], T0
    for bi in range(n_batches):
        back = late_shift_ms if (late_every and bi % late_every == late_every - 1) else 0
        rs = []
        for _ in range(rows):
            k = int(pool[int(rng.integers(0, len(pool)))])
            if hot_zero and rng.random() < hot_zero:
                k = 0
            v = float(rng.random() * 115.0)
            if special_vals:
                v = [v, v, 0.0, -0.0, math.nan, math.inf, -math.inf, 113.0, -113.0][int(rng.integers(0, 9))]
            r = [t - back + int(rng.integers(0, span_ms)), v, k]
            if null_frac:
                for j in (1, 2):
                    if rng.random() < null_frac:
                        r[j] = None
            rs.append(tuple(r))
        out.append(IntBatch.from_rows(rs, typ))
        t += span_ms
    return out, t


# ---------------------------------------------------------------------------------------------------------------- 1. parity
@pytest.mark.parametrize("tname", list(TYPES))
@pytest.mark.parametrize("L,S,filt", [(1000, 0, None), (4000, 2000, None), (1000, 0, ("max", ">", 100.0))])
def test_parity_with_nulls_edges_specials_and_late_batches(tname, L, S, filt):
    typ = TYPES[tname]
    rng = np.random.default_rng(zlib.crc32(f"{tname}-{L}-{S}".encode()))     # the same stream in every process
    batches, t = int_stream(rng, typ, 30, 1500, 300, null_frac=0.05, special_vals=True, late_every=6, late_shift_ms=2500)
    batches.append(sentinel(t + 3 * L, typ))
    want = oracle_rows(batches, L, S, filt)
    got, st = run_int(batches, typ, L, S, filt, per_batch_poll=True)
    assert len(want) > 200 and st["late_batches"] > 0 and st["generic_tiles"] > 0    # key bitmaps: the generic path
    assert_rows_equal(got, want, check_seq=True)
    assert st["groups"] == len(distinct_keys(batches))
    emitted = {r[2] for r in got}
    assert None in emitted and all(str(k).encode() in emitted for k in edge_keys(typ))


@pytest.mark.parametrize("tname", list(TYPES))
def test_parity_on_the_staged_path(tname):
    """No bitmaps: every tile goes through the TMA-staged integer instantiation (edge keys, +-0.0, NaN, +-inf, late batches)."""
    typ = TYPES[tname]
    rng = np.random.default_rng(3)
    batches, t = int_stream(rng, typ, 30, 2000, 500, special_vals=True, late_every=7, late_shift_ms=2500)
    batches.append(sentinel(t + 3000, typ))
    want = oracle_rows(batches, 1000)
    got, st = run_int(batches, typ, 1000, per_batch_poll=True)
    assert st["fast_tiles"] > 0 and st["late_batches"] > 0
    assert_rows_equal(got, want, check_seq=True)


# ---------------------------------------------------------------------------------------------------------------- 2. + 3. paths
@pytest.mark.parametrize("tname", ["int64", "uint32"])
def test_every_kernel_path_agrees(tname):
    typ = TYPES[tname]
    rng = np.random.default_rng(21)
    batches, t = int_stream(rng, typ, 24, 4 * TILE, 3000, span_ms=250, special_vals=True)
    batches.append(sentinel(t + 5000, typ))
    st = run_every_path(batches, typ, 1000)
    assert st["hinted"]["fast_tiles"] > 0 and st["generic"]["fast_tiles"] == 0


@pytest.mark.parametrize("tname", ["int64", "int32"])
def test_hot_key_zero_on_every_path(tname):
    """Half of the rows have the key 0, whose stored form is non-zero only through int_key's tag word."""
    typ = TYPES[tname]
    rng = np.random.default_rng(5)
    batches, t = int_stream(rng, typ, 20, 4 * TILE, 800, span_ms=250, hot_zero=0.5)
    batches.append(sentinel(t + 5000, typ))
    assert sum(int((b.keys == 0).sum()) for b in batches) > 0.45 * sum(len(b.ts) for b in batches)
    run_every_path(batches, typ, 1000)


# ---------------------------------------------------------------------------------------------------------------- 4. collisions
def int_key_hash(values, width):
    """NumPy port of int_key (dnz_device.cuh) followed by hash_inline: the dictionary hash of integer keys."""
    k0 = np.asarray(values).astype(np.uint64)
    if width == 4:
        k0 = k0 & np.uint64(0xFFFFFFFF)
    return hash_inline(k0, np.full(k0.shape, INT_KEY_TAG, np.uint64), np.full(k0.shape, width, np.uint32))


def collision_int_keys(width):
    cand = np.unique(np.random.default_rng(9).integers(-(1 << 62), 1 << 62, 4_000_000)) if width == 8 else \
        np.unique(np.random.default_rng(9).integers(0, 1 << 31, 4_000_000))
    h = int_key_hash(cand, width)
    order = np.argsort(h, kind="stable")
    eq = np.nonzero(h[order][1:] == h[order][:-1])[0]
    pairs = [(int(cand[order[e]]), int(cand[order[e + 1]])) for e in eq[:40]]
    clusters = []
    for nbits, count in ((16, 6), (21, 6)):          # one home slot while the table has <= 2^nbits slots
        low = (h & np.uint32((1 << nbits) - 1)).astype(np.int64)
        cnt = np.bincount(low, minlength=1 << nbits)
        for b in np.argsort(-cnt, kind="stable")[:count]:
            clusters.append([int(x) for x in cand[np.nonzero(low == b)[0][:32]]])
    return pairs, clusters


@pytest.mark.parametrize("tname", ["int64", "int32"])
def test_colliding_keys_on_every_path(tname):
    """Int64 keys with equal 32-bit hashes (the same chain at every table size) and clusters of keys that share their home slot
    on the small and on the hinted table.  A 4-byte key's hash is a bijection of its value (one multiply plus murmur3's
    finaliser): Int32 keys collide only in their home slots."""
    typ = TYPES[tname]
    pairs, clusters = collision_int_keys(8 if tname == "int64" else 4)
    assert (len(pairs) >= 20) == (tname == "int64") and min(len(c) for c in clusters) >= 4
    keys = sorted({k for p in pairs for k in p} | {k for c in clusters for k in c})
    assert len(keys) < 900
    rng = np.random.default_rng(64)
    batches = []
    for b in range(24):
        n = 8 * TILE
        k = np.array(keys, np.int64)[rng.integers(0, len(keys), n)]
        v = rng.random(n) * 200.0 - 100.0
        batches.append(IntBatch(T0 + b * 250 + rng.integers(0, 250, n), v, k, typ))
    batches.append(sentinel(T0 + 10_000, typ))
    st = run_every_path(batches, typ, 1000, names=("private", "hinted", "hinted_noqueue", "scalar_probe", "generic"))
    for name, s in st.items():
        assert s["deferred_rows"] == 0, name


# ---------------------------------------------------------------------------------------------------------------- 5. slices
def _sliced_batch(typ, ts, val, keys, kvalid, n_junk):
    """A RecordBatch whose columns are slices with their own offsets (the key bitmap starts at a non-byte offset)."""
    n = len(ts)
    junk_k = [7] * n_junk
    key = pa.array(junk_k + list(keys), typ, mask=np.concatenate([np.zeros(n_junk, bool), ~kvalid])).slice(n_junk)
    val_a = pa.array([1e300] * (n_junk + 2) + list(val), pa.float64()).slice(n_junk + 2)
    meta = _meta(np.concatenate([np.full(n_junk + 1, 5, np.int64), ts]), None, n + n_junk + 1).slice(n_junk + 1)
    return pa.RecordBatch.from_arrays([key, val_a, meta], schema=int_schema(typ))


@pytest.mark.parametrize("tname", list(TYPES))
def test_sliced_arrow_arrays(tname):
    typ = TYPES[tname]
    rng = np.random.default_rng(17)
    ks = edge_keys(typ)
    w = gpu_int_window(typ, 1000)
    o_batches = []
    for b in range(12):
        n = 3 * TILE + 5
        keys = np.array([ks[int(x)] for x in rng.integers(0, len(ks), n)], dtype=object)
        kvalid = rng.random(n) > 0.1
        ts = T0 + b * 300 + rng.integers(0, 300, n)
        val = rng.random(n) * 100.0
        w.push(_sliced_batch(typ, ts, val, keys.tolist(), kvalid, 3 + b))
        o_batches.append(IntBatch(ts, val, keys.astype(typ.to_pandas_dtype()), typ, key_valid=kvalid))
    w.push(sentinel(T0 + 9000, typ).record_batch())
    got = int_rows(w.poll(), typ)
    w.close()
    assert_rows_equal(got, oracle_rows(o_batches + [sentinel(T0 + 9000, typ)], 1000))


def _device_copy(arr):
    from denormalized_b200 import lib
    L = lib()
    a = np.ascontiguousarray(arr)
    p = L.dnz_device_alloc(0, a.nbytes + 64)
    assert p and L.dnz_memcpy(p, a.ctypes.data, a.nbytes, 1) == 0
    return p


@pytest.mark.parametrize("tname", ["int64", "uint32"])
def test_device_values_not_16_byte_aligned_take_the_generic_path(tname):
    from denormalized_b200 import capi, lib
    typ = TYPES[tname]
    dt = np.dtype(typ.to_pandas_dtype())
    rng = np.random.default_rng(4)
    n = 6 * TILE + 3
    ts = T0 + np.sort(rng.integers(0, 2000, n)).astype(np.int64)
    val = rng.random(n) * 50.0
    keys = rng.integers(0, 300, n).astype(dt)
    bufs = [_device_copy(ts), _device_copy(val)]
    kbuf = _device_copy(np.concatenate([np.zeros(1, dt), keys]))          # the values start W bytes into the block
    bufs.append(kbuf)
    db = (capi.DeviceBatchC * 1)()
    db[0] = capi.DeviceBatchC(n, bufs[0], None, bufs[1], None, None, kbuf + dt.itemsize, None)
    w = gpu_int_window(typ, 1000)
    w.push_device(array=db, n=1)
    w.push(sentinel(T0 + 9000, typ).record_batch())
    got = int_rows(w.poll(), typ)
    st = w.stats()
    w.close()
    for p in bufs:
        lib().dnz_device_free(0, p)
    assert st["generic_tiles"] >= 7 and st["fast_tiles"] <= 1
    assert_rows_equal(got, oracle_rows([IntBatch(ts, val, keys, typ), sentinel(T0 + 9000, typ)], 1000))


# ---------------------------------------------------------------------------------------------------------------- 6. growth, storm
def test_dictionary_growth_through_8192_groups_with_replayed_rows():
    typ = pa.int64()
    rng = np.random.default_rng(12)
    batches = []
    for b in range(20):
        n = 4 * TILE
        k = rng.integers(-5000, 5000, n) * 1_000_003
        batches.append(IntBatch(T0 + b * 400 + rng.integers(0, 400, n), rng.random(n) * 100.0, k, typ))
    batches.append(sentinel(T0 + 20_000, typ))
    n_keys = len(distinct_keys(batches))
    assert n_keys > 8192
    want = oracle_rows(batches, 1000)
    for flags in (0, PATHS["generic"][0], FLAG_SCALAR_PROBE):
        got, st = run_int(batches, typ, 1000, expected_groups=16, flags=flags)
        assert st["deferred_rows"] > 0 and st["groups"] == n_keys, (flags, st)
        assert_rows_equal(got, want)


def test_insert_storm_of_new_int64_keys():
    """8 Mi rows in one launch, every key new and probed by several CTAs while it is inserted (the layout of the Utf8 storm in
    tests/test_gpu_kernel_edges.py): every key is interned exactly once."""
    typ = pa.int64()
    n_rows = 8 * 1024 * 1024 - (8 * 1024 * 1024) % (16 * TILE)
    t = np.arange(n_rows, dtype=np.int64) // TILE
    r = np.arange(n_rows, dtype=np.int64) % TILE
    u = t % 16
    kid = (t // 16) * (4 * TILE) + (u % 4) * TILE + (r + 97 * (u // 4)) % TILE
    n_keys = int(kid.max()) + 1
    keys = kid * -7_919 + (1 << 40)
    val = (np.random.default_rng(8).random(n_rows) - 0.5) * 200.0
    ts = T0 + np.arange(n_rows, dtype=np.int64) // 20_000
    batches = [IntBatch(ts[i:i + (1 << 20)], val[i:i + (1 << 20)], keys[i:i + (1 << 20)], typ) for i in range(0, n_rows, 1 << 20)]
    batches.append(sentinel(T0 + 10_000_000, typ))
    want = result_table(oracle_mt_arrays([b.oracle() for b in batches], 60_000), "w")
    for flags in (0, FLAG_SCALAR_PROBE):
        w = gpu_int_window(typ, 60_000, expected_groups=n_keys, flags=flags)
        for b in batches:
            w.push(b.record_batch())
        got = int_result_table(w.poll(), "g")
        st = w.stats()
        w.close()
        assert st["groups"] == n_keys + 1 and st["fast_tiles"] > 0.9 * n_rows / TILE, st
        assert assert_tables_equal(got, want) == want.num_rows


def int_result_table(rb, tag):
    """Emitted RecordBatch with an integer key -> the table layout of result_table (key as str(v) bytes)."""
    col = {name: rb.column(i) for i, name in enumerate(rb.schema.names)}

    def f64_bits(name):
        return pa.array(np.asarray(col[name].fill_null(0.0).to_numpy(zero_copy_only=False), np.float64).view(np.int64))
    return pa.table({"ws": col["window_start_time"].cast(pa.int64()), "key": col["id"].cast(pa.string()).cast(pa.binary()),
                     "count_" + tag: col["count"].cast(pa.int64()), "min_" + tag: f64_bits("min"), "max_" + tag: f64_bits("max"),
                     "avg_" + tag: pa.array(np.asarray(col["average"].fill_null(0.0).to_numpy(zero_copy_only=False), np.float64)),
                     "null_" + tag: col["min"].is_null()})


# ---------------------------------------------------------------------------------------------------------------- 7. checkpoint
def test_checkpoint_round_trip_and_refused_restores():
    from denormalized_b200 import DnzError
    from tests.helpers import gpu_window
    typ = pa.uint64()
    rng = np.random.default_rng(31)
    batches, t = int_stream(rng, typ, 16, 2000, 400, null_frac=0.02, special_vals=True)
    batches.append(sentinel(t + 4000, typ))
    want = oracle_rows(batches, 2000, 1000)
    w = gpu_int_window(typ, 2000, 1000)
    got = []
    for b in batches[:8]:
        w.push(b.record_batch())
        got += int_rows(w.poll(), typ)
    blob = w.checkpoint()
    w.close()
    w2 = gpu_int_window(typ, 2000, 1000)
    w2.restore(blob)
    for b in batches[8:]:
        w2.push(b.record_batch())
        got += int_rows(w2.poll(), typ)
    w2.close()
    assert_rows_equal(got, want)
    # an integer blob into a Utf8 operator, a Utf8 blob into an integer operator, Int64 into UInt64: all refused
    u = gpu_window(2000, 1000)
    with pytest.raises(DnzError) as e:
        u.restore(blob)
    assert e.value.code == -1
    u.close()
    u = gpu_window(2000, 1000)
    from tests.helpers import rows_to_batch, to_record_batch
    u.push(to_record_batch(rows_to_batch([(T0, 1.0, b"a")])))
    ublob = u.checkpoint()
    u.close()
    for t2 in (pa.uint64(), pa.int64()):
        wi = gpu_int_window(t2, 2000, 1000)
        with pytest.raises(DnzError) as e:
            wi.restore(ublob)
        assert e.value.code == -1
        wi.close()
    wi = gpu_int_window(pa.int64(), 2000, 1000)
    with pytest.raises(DnzError) as e:
        wi.restore(blob)
    assert e.value.code == -1
    wi.close()


# ---------------------------------------------------------------------------------------------------------------- 8. exchange
def _exchange_stream(typ):
    rng = np.random.default_rng(77)
    batches, t = int_stream(rng, typ, 36, 1500, 600, span_ms=200, null_frac=0.03)
    return batches, t


@pytest.mark.parametrize("world", [2, 4])
def test_fused_exchange_equals_one_operator(world):
    from denormalized_b200 import ExchangeGroup
    typ = pa.int64()
    batches, t = _exchange_stream(typ)
    close = (t // 1000 + 1) * 1000 + 2000
    want = oracle_rows(batches + [sentinel(close, typ)], 1000)
    groups = ExchangeGroup.create_local([0] * world, ring_entries=1 << 16, ring_key_bytes=4 << 20)
    wins = [gpu_int_window(typ, 1000, expected_groups=4096) for _ in range(world)]
    for g, w in zip(groups, wins):
        g.attach(w)
    got = []

    def step(force=False):
        for g, w in zip(groups, wins):
            if force:
                w.process()
            g.step_begin(w)
        for g, w in zip(groups, wins):
            g.step_pack(w)
        assert len({g.step_finish(w) for g, w in zip(groups, wins)}) == 1
        for w in wins:
            got.extend(int_rows(w.poll(), typ))
    for i, b in enumerate(batches):
        wins[i % world].push(b.record_batch())
        if i % (2 * world) == 2 * world - 1:
            step()
    for w in wins:
        w.push(sentinel(close, typ).record_batch())
    for _ in range(3):                                 # publish | pack | merge + emit
        step(force=True)
    step()
    st = [w.stats() for w in wins]
    for w in wins:
        w.close()
    for g in groups:
        g.close()
    assert sum(s["exchanged_in"] for s in st) > 500
    assert_rows_equal(got, want)
    assert len({(r[0], r[2]) for r in got}) == len(got)


def test_host_driven_exchange_equals_one_operator():
    from denormalized_b200.exchange import LocalTransport
    typ = pa.uint32()
    world = 2
    batches, t = _exchange_stream(typ)
    close = (t // 1000 + 1) * 1000 + 2000
    want = oracle_rows(batches + [sentinel(close, typ)], 1000)
    wins = [gpu_int_window(typ, 1000, expected_groups=64) for _ in range(world)]
    for r, w in enumerate(wins):
        w.set_exchange(r, world)
    lt = LocalTransport(wins)
    got = []
    for i, b in enumerate(batches):
        wins[i % world].push(b.record_batch())
        if i % 6 == 5:
            got += [r for rb in lt.exchange_all() for r in int_rows(rb, typ)]
    for w in wins:
        w.push(sentinel(close, typ).record_batch())
    got += [r for rb in lt.exchange_all() for r in int_rows(rb, typ)]
    st = [w.stats() for w in wins]
    for w in wins:
        w.close()
    assert sum(s["exchanged_out"] for s in st) == sum(s["exchanged_in"] for s in st) > 500
    assert_rows_equal(got, want)


@pytest.mark.parametrize("types", [("int64", "uint64"), ("int64", "utf8"), ("utf8", "int32")])
def test_exchange_between_key_types_is_refused(types):
    """Ranks that group by different key types (here even of the same width) cannot exchange: the owner's merge sees the
    sender's key type in the packets and the import fails with DNZ_ERR_INVALID instead of grouping foreign keys."""
    from denormalized_b200 import DnzError
    from denormalized_b200.exchange import LocalTransport
    from tests.helpers import gpu_window, rows_to_batch, to_record_batch
    wins = []
    for r, tname in enumerate(types):
        w = gpu_window(1000, expected_groups=64) if tname == "utf8" else gpu_int_window(TYPES[tname], 1000, expected_groups=64)
        w.set_exchange(r, len(types))
        wins.append(w)
    for tname, w in zip(types, wins):
        for t in (T0, T0 + 1500):
            if tname == "utf8":
                w.push(to_record_batch(rows_to_batch([(t + i, 1.0, b"%d" % i) for i in range(200)])))
            else:
                w.push(IntBatch(t + np.arange(200), np.ones(200), np.arange(200), TYPES[tname]).record_batch())
    with pytest.raises(DnzError) as e:
        LocalTransport(wins).exchange_all()
    assert e.value.code == -1 and "key type" in str(e.value)
    for w in wins:
        w.close()


# ---------------------------------------------------------------------------------------------------------------- 9. device I/O
def _device_rows(w, r, typ):
    a = w.fetch_device_result(r)
    return [(int(a["window_start"][i]), int(a["window_end"][i]), None if a["key"][i] is None else str(a["key"][i]).encode(),
             int(a["count"][i]), float(a["min"][i]) if a["agg_valid"][i] else None, float(a["max"][i]) if a["agg_valid"][i] else None,
             float(a["avg"][i]) if a["agg_valid"][i] else None, 0) for i in range(r.n_rows)]


@pytest.mark.parametrize("tname", ["int64", "int32"])
def test_device_push_and_poll(tname):
    from denormalized_b200 import DeviceBatches, DnzError, capi
    typ = TYPES[tname]
    rng = np.random.default_rng(2)
    batches, t = int_stream(rng, typ, 12, 2000, 300, null_frac=0.05)
    batches.append(sentinel(t + 3000, typ))
    want = oracle_rows(batches, 1000)
    w = gpu_int_window(typ, 1000)
    got = []
    for b in batches:
        w.push(b.record_batch())
        r = w.poll_device_ready()
        assert r.n_rows == 0 or (not r.key_off and r.key_bytes_len == r.n_rows * typ.bit_width // 8)
        got += _device_rows(w, r, typ)
    while True:
        r = w.poll_device()
        if not r.n_rows:
            break
        assert not r.key_off and r.key_bytes_len == r.n_rows * typ.bit_width // 8
        got += _device_rows(w, r, typ)
    w.close()
    assert_rows_equal(got, want)
    # device batches of an integer stream carry the values in key_bytes and no offsets
    dev = DeviceBatches(4096, 1024, groups=50, rows_per_ms=10, int_keys=True)
    bad = (capi.DeviceBatchC * 1)()
    bad[0] = dev.array[0]
    bad[0].key_off = dev.array[0].ts
    w = gpu_int_window(pa.int64(), 1000)
    with pytest.raises(DnzError) as e:
        w.push_device(array=bad, n=1)
    assert e.value.code == -1
    w.close()
    w = gpu_int_window(pa.int64(), 1000)
    w.push_device(dev)
    w.flush(T0 + 10_000)
    r = w.poll_device()
    a = w.fetch_device_result(r)
    w.close(); dev.free()
    assert r.n_rows > 0 and not r.key_off and set(a["key"]) <= set(range(50)) and int(a["count"].sum()) == 4096


# ---------------------------------------------------------------------------------------------------------------- 10. large
def test_cfg2_stream_200m_rows_with_int64_keys():
    """cfg 2's stream (100 K groups, tumbling 1 s) with synthetic Int64 keys, device resident, against the multi-threaded oracle
    over the same stream with the keys "sensor_<id>" (the same ids)."""
    from denormalized_b200 import DeviceBatches, capi
    n_rows, groups, rpm, L = 200_000_000, 100_000, 10_000, 1000
    dev = DeviceBatches(n_rows, 65536, groups=groups, rows_per_ms=rpm, int_keys=True)
    w = gpu_int_window(pa.int64(), L, expected_groups=groups)
    parts = []

    def take(r):
        if r.n_rows:
            a = w.fetch_device_result(r, max_keys=0)
            s = pc.binary_join_element_wise(pa.scalar(b"sensor_"), pa.array(a["key_values"]).cast(pa.string()).cast(pa.binary()), b"")
            a["key_off"] = np.frombuffer(s.buffers()[1], np.int32, r.n_rows + 1).copy()
            a["key_bytes"] = np.frombuffer(s.buffers()[2], np.uint8, int(a["key_off"][-1])).copy()
            assert s.offset == 0 and a["key_off"][0] == 0 and np.all(a["key_valid"] == 1)
            parts.append(a)
        return r.n_rows
    for g0 in range(0, dev.n_batches, 1024):
        k = min(1024, dev.n_batches - g0)
        w.push_device(array=C.cast(C.byref(dev.array, g0 * C.sizeof(capi.DeviceBatchC)), C.POINTER(capi.DeviceBatchC)), n=k)
        while take(w.poll_device_ready()):
            pass
    last = T0 + (n_rows - 1) // rpm
    close = (last // 1000 + 1) * 1000 + 2 * L
    w.flush(close)
    while take(w.poll_device()):
        pass
    st = w.stats()
    w.close(); dev.free()
    from tests.helpers import concat_arrays, rows_to_batch
    hb = host_stream(n_rows, groups=groups, rows_per_ms=rpm)
    hb.append(rows_to_batch([(close, 1.0, b"sentinel")]))
    want = result_table(oracle_mt_arrays(hb, L), "w")
    del hb
    got = result_table(concat_arrays(parts), "g")
    assert got.num_rows == want.num_rows == 20 * groups
    assert st["groups"] == pc.count_distinct(want["key"]).as_py() == groups and st["deferred_rows"] == 0
    assert assert_tables_equal(got, want) == want.num_rows


# ---------------------------------------------------------------------------------------------------------------- schema
@pytest.mark.parametrize("nullable", [True, False])
def test_emitted_key_field_keeps_the_input_nullability(nullable):
    typ = pa.uint32()
    rng = np.random.default_rng(8)
    batches, t = int_stream(rng, typ, 6, 1000, 100)
    batches.append(sentinel(t + 3000, typ))
    from denormalized_b200 import GpuStreamingWindow
    w = GpuStreamingWindow(int_schema(typ, nullable), "id", DEFAULT_AGGS, 1000)
    got = []
    for b in batches:
        rb = b.record_batch()
        w.push(pa.RecordBatch.from_arrays(rb.columns, schema=int_schema(typ, nullable)))
        got += int_rows(w.poll(), typ, nullable=nullable)
    w.close()
    assert_rows_equal(got, oracle_rows(batches, 1000))


# ---------------------------------------------------------------------------------------------------------------- 11. rejected
@pytest.mark.parametrize("typ", [pa.int16(), pa.uint8(), pa.float64(), pa.int8(), pa.dictionary(pa.int32(), pa.utf8())])
def test_other_key_types_are_unsupported(typ):
    from denormalized_b200 import DnzError, GpuStreamingWindow, canonical_schema
    meta = canonical_schema().field(3)
    schema = pa.schema([pa.field("id", typ), pa.field("reading", pa.float64()), meta])
    with pytest.raises(DnzError) as e:
        GpuStreamingWindow(schema, "id", DEFAULT_AGGS, 1000)
    assert e.value.code == -2
