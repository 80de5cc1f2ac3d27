"""Parity tests at the edges the fast path, the tile scan and the input code treat specially (run on an H100 with -m gpu).
Every test goes through the C ABI and is compared with the oracle (count / min / max bit-exact, avg within 1e-9), and asserts
the counters (fast / generic tiles, deferred rows, late batches, groups) that prove it reached the path it is named after.

  A  the kernel configuration matrix (tests/helpers.py: KERNEL_PATHS, run_paths), including a stream whose dictionary grows
     through 8192 groups, so that consecutive launches switch from per-CTA private pane copies to min/max hints
  B  sliced Arrow input: batch offsets, child offsets, a metadata struct with its own offset, bitmaps at non-byte offsets,
     key bytes that start at offsets that are not 16 B aligned; the raw-timestamp producer inputs sliced
  C  key layout: every length 0..40 at every misalignment 0..15, NUL-byte keys, tiles of exactly BCAP and BCAP + 1 key bytes
  D  tile geometry and timestamps: odd / even tile tails, > 1100 batches per launch, tiles spread over 2^31 ms, rows on pane
     boundaries, timestamps around 2^53 ms, the window / slide ratio limit
  E  dictionary collisions (keys chosen with the NumPy port of the hash) and an insert storm
  F  the post-aggregate filter at the totalOrder edges"""
import ctypes as C
import datetime as dt
import math

import numpy as np
import pyarrow as pa
import pytest

from tests.helpers import (DEFAULT_AGGS, assert_rows_equal, assert_tables_equal, batch_to_rows, columns_to_batch,
                           gpu_window, hash_keys, hash_words, oracle_mt_arrays, record_batch_rows, record_batch_table, result_table,
                           rows_to_batch, run_gpu, run_oracle_batches, run_paths, to_record_batch)

pytestmark = pytest.mark.gpu
T0 = 1_700_000_000_000
TILE, BCAP = 416, 6656           # denormalized_b200/csrc/dnz_kernels.h


def sentinel(ts):
    return rows_to_batch([(ts, 1.0, b"sentinel")])


def _distinct_keys(batches):
    return {r[2] for b in batches for r in batch_to_rows(b) if r[0] is not None} - {b"sentinel"}


def _adversarial_values(rng, keys, mode):
    """min / max streams that defeat a lossy reduction filter (as in test_minmax_hints_never_lose_an_extreme): values creeping up
    or down inside one top-16-bit bucket, magnitudes over the whole double range, values a hair apart.  The sign is fixed per key
    (negative for every third key id): an average of values that cancel depends on the summation order beyond 1e-9."""
    n = len(keys)
    mode %= 5
    if mode == 0:
        v = 100.0 + np.arange(n) * 1e-9 + rng.random(n) * 1e-7
    elif mode == 1:
        v = 50.0 - np.arange(n) * 1e-9 - rng.random(n) * 1e-7
    elif mode == 2:
        v = (rng.random(n) + 1e-3) * 10.0 ** rng.integers(-300, 300, n).astype(np.float64)
    elif mode == 3:
        v = np.where(rng.random(n) < 0.5, 113.99999, 114.00001)
    else:
        v = rng.random(n) * 115.0 + 1e-3
    return v * np.where(np.asarray(keys) % 3 == 0, -1.0, 1.0)


# =============================================================================================================================
# A. the kernel configuration matrix
def test_paths_agree_while_the_dictionary_grows_through_8192_groups():
    """20 K distinct keys introduced batch by batch, three batches per launch: the 16-group start grows the dictionary (deferred
    rows) from 1024 through 8192 to 32768 groups, so consecutive launches of `private` switch from private copies to hints."""
    rng = np.random.default_rng(2020)
    batches, t = [], T0
    n_keys, nb, rows = 20_000, 30, 4000
    for b in range(nb):
        hi = min(n_keys, (b + 1) * (n_keys // (nb - 2)))
        k = np.concatenate([np.arange(max(0, hi - n_keys // (nb - 2)), hi), rng.integers(0, hi, rows)])[:rows]
        v = _adversarial_values(rng, k, b)
        ts = t + rng.integers(0, 300, rows)
        batches.append(columns_to_batch(ts, v, [b"grow-%05d" % x for x in k]))
        t += 300
    batches.append(sentinel(t + 4000))
    assert len(_distinct_keys(batches)) == n_keys
    for L, S in [(1000, 0), (2000, 1000)]:
        st = run_paths(batches, L, S, max_rows_per_launch=3 * rows)
        for name, s in st.items():
            assert s["groups"] == n_keys + 1, name                     # + the sentinel
            assert s["agg_launches"] >= 10, name
        assert st["private"]["deferred_rows"] > 0 and st["noprivate_small"]["deferred_rows"] > 0
        assert st["hinted"]["deferred_rows"] == 0
        assert st["generic"]["fast_tiles"] == 0 and st["hinted"]["fast_tiles"] > 0.9 * nb * rows / TILE


# =============================================================================================================================
# B. sliced Arrow input
SLICE_OFFSETS = [1, 3, 7, 8, 13, 416, 417]


def _rows_with_nulls(rng, n, t, nulls):
    out = []
    for i in range(n):
        k = int(rng.integers(0, 29))
        key = b"s%d" % k + b"x" * (k % 7)
        val = float(rng.random() * 100.0) if k % 5 else [0.0, -0.0, float("nan"), float("inf"), 3.0][i % 5]
        r = [t + int(rng.integers(0, 900)), val, key]
        if nulls:
            for j in range(3):
                if rng.random() < 0.12:
                    r[j] = None
        out.append(tuple(r))
    return out


def _junk(n):
    return [(5, 1e300, b"junk-row-%d" % (i % 3)) for i in range(n)]        # wrong rows: ts before every window, a huge value


@pytest.mark.parametrize("nulls", [True, False])
@pytest.mark.parametrize("off", SLICE_OFFSETS)
def test_sliced_record_batches(off, nulls):
    """RecordBatch.slice(off, n): every child array carries the offset, validity bitmaps start at bit off & 7, the key bytes of the
    slice start at a non-zero offset that is not 16 B aligned."""
    rng = np.random.default_rng(off * 2 + nulls)
    rbs, logical, t = [], [], T0
    for b in range(6):
        n = 300 + 41 * b
        body = _rows_with_nulls(rng, n, t, nulls)
        if nulls and all(r[0] is None for r in body):
            body[0] = (t, 1.0, b"s1")
        full = _junk(off) + body + _junk(9)
        if sum(len(r[2]) for r in full[:off]) % 16 == 0:
            full[0] = (5, 1e300, full[0][2] + b"!")
        kb = rows_to_batch(full, force_validity=nulls)
        assert kb.key_off[off] % 16 != 0
        rbs.append(to_record_batch(kb).slice(off, n))
        logical.append(rows_to_batch(body))
        t += 500
    rbs.append(to_record_batch(sentinel(t + 4000)))
    logical.append(sentinel(t + 4000))
    for L, S in [(1000, 0), (2000, 1000)]:
        want = run_oracle_batches(logical, L, S)
        w = gpu_window(L, S)
        got = []
        for i, rb in enumerate(rbs):
            w.push(rb)
            got += record_batch_rows(w.poll(), i)
        st = w.stats()
        w.close()
        assert len(want) > 50
        assert_rows_equal(got, want, check_seq=True)
        assert st["groups"] == len(_distinct_keys(logical)) + 1          # + the sentinel; a NULL key is a group of its own
        if nulls:
            assert st["generic_tiles"] > 0
        else:
            assert st["fast_tiles"] > 0 and st["generic_tiles"] == 0


def _push_struct(w, sa):
    """dnz_window_push of a StructArray (the C-Data form of a RecordBatch) with a non-zero top-level offset."""
    from denormalized_b200 import capi
    ca = capi.ArrowArrayC()
    sa._export_to_c(C.addressof(ca))
    rc = w._L.dnz_window_push(w._h, C.byref(ca))
    if ca.release:
        C.CFUNCTYPE(None, C.POINTER(capi.ArrowArrayC))(ca.release)(C.byref(ca))
    w._check(rc)


def _prefixed(values, n_junk, junk, typ, mask=None):
    """Array of `values` behind n_junk junk entries, sliced so that its offset is n_junk."""
    m = None if mask is None else np.concatenate([np.zeros(n_junk, bool), mask])
    return pa.array([junk] * n_junk + list(values), typ, mask=m).slice(n_junk)


@pytest.mark.parametrize("nulls", [True, False])
def test_child_arrays_with_their_own_offsets(nulls):
    """Each child sliced by a different offset, the `_streaming_internal_metadata` struct with its own offset over a timestamp
    child that has another, and the top-level struct array sliced as well: the canonical timestamp sits at batch offset +
    struct offset + child offset."""
    from denormalized_b200 import canonical_schema
    schema = canonical_schema()
    meta_fields = list(schema.field(3).type)
    rng = np.random.default_rng(77 + nulls)
    w = gpu_window(2000, 1000)
    logical, got, t = [], [], T0
    for b in range(8):
        N = 700 + 13 * b
        rows = _rows_with_nulls(rng, N, t, nulls)
        ts = [r[0] if r[0] is not None else 0 for r in rows]
        tmask = np.array([r[0] is None for r in rows]) if nulls else None
        vmask = np.array([r[1] is None for r in rows]) if nulls else None
        kmask = np.array([r[2] is None for r in rows]) if nulls else None
        p_val, p_key, p_occ, p_meta, p_ts = 3 + b, 13 + 2 * b, 1 + b % 4, 5 + 3 * b, 7 + b
        val = _prefixed([r[1] if r[1] is not None else 0.0 for r in rows], p_val, 1e300, pa.float64(), vmask)
        key = _prefixed([(r[2] or b"").decode() for r in rows], p_key, "junk-prefix-key", pa.utf8(), kmask)
        occ = _prefixed(ts, p_occ, 5, pa.int64())
        tmask_full = None if tmask is None else np.concatenate([np.zeros(p_meta, bool), tmask])
        ts_child = _prefixed([5] * p_meta + ts, p_ts, 5, pa.timestamp("ms"), tmask_full)       # offset p_ts, length p_meta + N
        barrier = pa.array(["no_barrier"] * (p_meta + N), pa.utf8())
        meta = pa.StructArray.from_arrays([barrier, ts_child], fields=meta_fields).slice(p_meta)
        q = 1 + (b * 5) % 11
        m = N - q - 2
        top = pa.StructArray.from_arrays([occ, val, key, meta], fields=list(schema)).slice(q, m)
        assert top.offset == q and meta.offset == p_meta and ts_child.offset == p_ts
        body = rows[q:q + m]
        if all(r[0] is None for r in body):
            continue
        _push_struct(w, top)
        got += record_batch_rows(w.poll(), len(logical))
        logical.append(rows_to_batch(body))
        t += 500
    w.push(to_record_batch(sentinel(t + 4000)))
    got += record_batch_rows(w.poll(), len(logical))
    logical.append(sentinel(t + 4000))
    st = w.stats()
    w.close()
    want = run_oracle_batches(logical, 2000, 1000)
    assert len(want) > 100 and st["batches_in"] == len(logical)
    assert_rows_equal(got, want, check_seq=True)
    assert (st["generic_tiles"] > 0) if nulls else (st["fast_tiles"] > 0 and st["generic_tiles"] == 0)


def _iso(ms):
    return dt.datetime.fromtimestamp(ms // 1000, dt.timezone.utc).strftime("%Y-%m-%dT%H:%M:%S") + ".%03d" % (ms % 1000)


@pytest.mark.parametrize("unit", [1, 2, 3])        # DNZ_TS_INT64_MILLIS, DNZ_TS_INT64_SECONDS, DNZ_TS_STRING_ISO8601
def test_raw_timestamp_inputs_sliced(unit):
    """Raw producer batches (no metadata struct) sliced at odd offsets: the Int64 column is read from the slice, the Utf8 column's
    offsets are rebased by its first offset."""
    from denormalized_b200 import GpuStreamingWindow
    ts_type = pa.utf8() if unit == 3 else pa.int64()
    schema = pa.schema([pa.field("occurred_at", ts_type), pa.field("reading", pa.float64()), pa.field("sensor_name", pa.utf8())])
    fmt = "%Y-%m-%dT%H:%M:%S%.3f" if unit == 3 else None
    w = GpuStreamingWindow(schema, "sensor_name", DEFAULT_AGGS, 2000, 1000, None, timestamp=(unit, "occurred_at", fmt))
    rng = np.random.default_rng(unit)
    logical, got, t = [], [], T0
    for b, off in enumerate(SLICE_OFFSETS + [0]):
        n = 500 + 37 * b
        ms = t + rng.integers(0, 1500, n)
        if unit == 2:
            ms = ms // 1000 * 1000
        val = rng.random(n) * 115.0
        keys = ["s%d" % k + "y" * (k % 5) for k in rng.integers(0, 40, n)]
        jt = [T0 - 10**9] * off
        if unit == 1:
            tcol = pa.array(jt + ms.tolist(), pa.int64())
        elif unit == 2:
            tcol = pa.array([x // 1000 for x in jt] + (ms // 1000).tolist(), pa.int64())
        else:
            tcol = pa.array(["junk"] * off + [_iso(int(x)) for x in ms], pa.utf8())
        rb = pa.RecordBatch.from_arrays([tcol, pa.array([1e300] * off + val.tolist()), pa.array(["junk-key-%d" % i for i in range(off)] + keys)],
                                        schema=schema).slice(off, n)
        w.push(rb)
        got += record_batch_rows(w.poll(), b)
        logical.append(columns_to_batch(ms, val, [k.encode() for k in keys]))
        t += 1000
    last = t + 5000
    sent = pa.array([_iso(last)] if unit == 3 else [last // 1000 if unit == 2 else last], ts_type)
    w.push(pa.RecordBatch.from_arrays([sent, pa.array([1.0]), pa.array(["sentinel"])], schema=schema))
    got += record_batch_rows(w.poll(), len(logical))
    logical.append(sentinel(last - last % 1000 if unit == 2 else last))
    w.close()
    want = run_oracle_batches(logical, 2000, 1000)
    assert len(want) > 200
    assert_rows_equal(got, want, check_seq=True)


# =============================================================================================================================
# C. key layout
def _layout_key(length):
    return bytes(((i * 37 + length * 11) % 250) + 1 for i in range(length))      # no NUL byte: both key words non-zero


def test_every_key_length_at_every_misalignment():
    """Keys of 0..40 bytes, each one starting at every byte misalignment 0..15 of the staged buffer (a pad key in front steers the
    start); the same key at 16 misalignments must land in ONE group.  Empty-key rows keep every tile below BCAP."""
    rng = np.random.default_rng(40)
    batches = []
    for b in range(4):                                     # one pane per batch; the batch's key bytes start 16 B aligned
        keys, pos = [], 0
        for length in (range(41) if b % 2 == 0 else reversed(range(41))):
            for mis in range(16):
                pad = (mis - pos) % 16
                keys += [b"p" * pad, _layout_key(length), b""]
                pos += pad + length
        batches.append(columns_to_batch(T0 + b * 1000 + rng.integers(0, 1000, len(keys)), rng.random(len(keys)) * 100.0 - 50.0, keys))
        off = batches[-1].key_off
        starts = {(int(off[i + 1]) % 16, int(off[i + 2] - off[i + 1])) for i in range(0, len(keys), 3)}
        assert len(starts) == 41 * 16
        assert max(int(off[min(i + TILE, len(keys))] - off[i]) for i in range(0, len(keys), TILE)) <= BCAP
    batches.append(sentinel(T0 + 10_000))
    distinct = _distinct_keys(batches)
    assert len(distinct) == 41 + 15                      # 41 lengths (the empty key included) + pads of 1..15 bytes
    st = run_paths(batches, 1000)
    for name, s in st.items():
        assert s["groups"] == len(distinct) + 1, name
        if name != "generic":
            assert s["generic_tiles"] == 0 and s["fast_tiles"] > 0, name


def test_nul_byte_keys_are_distinct_groups():
    """"\\0" * n for n = 1..16 have all-zero key words and differ only in their length (the probe takes the ordered re-read of
    slot_keys_unsettled for them); "a" / "a\\0" / "a\\0\\0" share their words too; 16 B keys that differ only in their last byte."""
    special = [b"\0" * n for n in range(1, 17)] + [b"", b"a", b"a\0", b"a\0\0", b"\0a", b"a" * 15 + b"\0", b"a" * 15 + b"b",
                                                    b"\0" * 15 + b"\x01", b"sensor_1", b"sensor_1\0"]
    rng = np.random.default_rng(16)
    batches = []
    for b in range(12):
        k = rng.integers(0, len(special), 2000)
        v = _adversarial_values(rng, k, b)
        batches.append(columns_to_batch(T0 + b * 300 + rng.integers(0, 300, 2000), v, [special[i] for i in k]))
    batches.append(sentinel(T0 + 9000))
    for L, S in [(1000, 0), (2000, 1000)]:
        want = run_oracle_batches(batches, L, S)
        assert {r[2] for r in want} == set(special)
        st = run_paths(batches, L, S, want=want)
        for name, s in st.items():
            assert s["groups"] == len(special) + 1, name
            assert (s["fast_tiles"] == 0) if name == "generic" else (s["fast_tiles"] > 0 and s["generic_tiles"] == 0), name


@pytest.mark.parametrize("shift", [0, 15])
@pytest.mark.parametrize("extra", [0, 1])
def test_tile_of_exactly_bcap_key_bytes(shift, extra):
    """One 416-row tile whose keys total BCAP bytes (staged: the largest stage, BCAP + 15 bytes when the first key sits at
    byte0 % 16 == 15) and one with BCAP + 1 (key bytes read from global).  A first tile of empty keys and one `shift`-byte key
    places the edge tile."""
    rng = np.random.default_rng(shift * 2 + extra)
    batches = []
    for b in range(4):
        lead = [b""] * (TILE - 1) + [b"L" * shift] if shift else []
        edge = [b"edge-key-%07d" % ((b * 131 + i) % 600) for i in range(TILE)]           # 16 B each: 416 * 16 = BCAP
        if extra:
            edge[-1] = edge[-1] + b"+"                                                    # 17 B: BCAP + 1, and an arena key
        ks = lead + edge
        b_ = columns_to_batch(T0 + b * 500 + rng.integers(0, 400, len(ks)), rng.random(len(ks)) * 1e3 - 500.0, ks)
        t0 = len(lead)
        assert int(b_.key_off[t0]) % 16 == shift and int(b_.key_off[t0 + TILE]) - int(b_.key_off[t0]) == BCAP + extra
        batches.append(b_)
    batches.append(sentinel(T0 + 9000))
    st = run_paths(batches, 1000, names=("hinted", "private", "generic"))
    n_tiles = 4 * (1 + (shift > 0)) + 1                   # + the sentinel's
    assert st["hinted"]["fast_tiles"] == n_tiles and st["hinted"]["generic_tiles"] == 0
    assert st["generic"]["fast_tiles"] == 0 and st["generic"]["generic_tiles"] == n_tiles


# =============================================================================================================================
# D. tile geometry and timestamps
SIZES = [1, 2, 3, 415, 416, 417, 831, 832, 833, 4161]


def _boundary_batch(rng, n, base, pane_ms, key_base):
    """n rows in the pane starting at `base`, the LAST row exactly on the next pane's first millisecond: a tile whose odd tail row
    is its maximum and lies in another pane."""
    ts = base + (np.arange(n) * 7) % pane_ms
    if n > 1:
        ts[-1] = base + pane_ms
        ts[-2] = base + pane_ms - 1
    keys = [b"geo-%d" % (key_base + i % 9) for i in range(n)]
    return columns_to_batch(ts, rng.random(n) * 100.0 + 1.0, keys)


@pytest.mark.parametrize("L,S", [(1000, 0), (2000, 1000)])
def test_tile_tails_in_one_launch(L, S):
    """Batches of 1, 2, 3, 415 ... 4161 rows queued into one launch (odd and even tails, one-row tiles)."""
    pane = S or L
    rng = np.random.default_rng(L + S)
    batches = [_boundary_batch(rng, n, T0 + i * 2 * pane, pane, i) for i, n in enumerate(SIZES)]
    batches.append(sentinel(T0 + 30 * pane + 3 * L))
    st = run_paths(batches, L, S, names=("hinted", "private", "generic"))
    n_tiles = sum((n + TILE - 1) // TILE for n in SIZES) + 1
    assert st["hinted"]["agg_launches"] == 1 and st["hinted"]["fast_tiles"] == n_tiles
    assert st["generic"]["generic_tiles"] == n_tiles


def test_more_than_1100_batches_in_one_launch():
    """1500 batches of 1-3 rows: the tile scan's 32-ary batch search takes three rounds and every warp's four tiles belong to
    four batches."""
    rng = np.random.default_rng(1100)
    batches, t = [], T0
    for b in range(1500):
        n = 1 + b % 3
        ts = t + rng.integers(0, 40, n)
        ts = np.sort(ts)
        if b % 7 == 0 and n > 1:
            ts[-1] = (t // 1000 + 1) * 1000                 # on a pane boundary
        batches.append(columns_to_batch(ts, rng.random(n) * 10.0 - 5.0, [b"tiny-%d" % (x % 23) for x in rng.integers(0, 1000, n)]))
        t += 37
    batches.append(sentinel(t + 5000))
    st = run_paths(batches, 2000, 1000, names=("hinted", "generic"))
    assert st["hinted"]["agg_launches"] == 1 and st["hinted"]["batches_in"] == 1501


def test_tiles_spread_over_two_to_the_31_ms():
    """Tumbling 1 h windows.  One-tile batches whose timestamps reach exactly 2^31 - 1 and 2^31 ms past the tile's first row, and
    exactly 2^31 and 2^31 + 1 ms below it: the 32-bit reduction at its limit and the 64-bit fallback."""
    L = 3_600_000
    rng = np.random.default_rng(31)
    batches, base = [], T0
    for kind in range(4):
        n = 300
        span = (1 << 31) - 1 + (kind & 1) if kind < 2 else (1 << 31) + (kind & 1)
        if kind < 2:                                       # first row = minimum, one row `span` above it
            ts = base + rng.integers(0, span, n)
            ts[0], ts[1] = base, base + span
            lo = base
        else:                                              # first row = maximum, one row `span` below it
            first = base + span
            ts = first - rng.integers(0, span, n)
            ts[0], ts[1] = first, first - span
            lo = first - span
        assert ts.min() == lo and ts.max() - ts.min() == span
        batches.append(columns_to_batch(ts, rng.random(n) * 50.0, [b"wide-%d" % (i % 5) for i in range(n)]))
        base = int(ts.max()) + 10_000_000
    batches.append(sentinel(base + 3 * L))
    st = run_paths(batches, L, 0, names=("hinted", "private", "generic"), per_batch_poll=True)
    assert st["hinted"]["fast_tiles"] == 5


def test_rows_on_pane_boundaries():
    """Rows exactly on k * pane_ms - 1 and k * pane_ms inside one tile, with and without the tile's minimum on a boundary."""
    rng = np.random.default_rng(9)
    batches = []
    for b in range(6):
        k = T0 // 1000 + 1 + 3 * b
        ts = k * 1000 - 1 - rng.integers(0, 999, TILE)
        ts[5], ts[7] = k * 1000 - 1, k * 1000
        if b % 2:
            ts[0] = (k - 1) * 1000                               # minimum on a boundary too
        batches.append(columns_to_batch(ts, rng.random(TILE) * 20.0, [b"edge-%d" % (i % 4) for i in range(TILE)]))
    batches.append(sentinel(T0 + 40_000))
    for L, S in [(1000, 0), (3000, 1000)]:
        st = run_paths(batches, L, S, names=("hinted", "private", "generic"), per_batch_poll=True)
        assert st["hinted"]["fast_tiles"] == 7


def test_timestamps_around_two_to_the_53_ms():
    """Tiles whose minimum lies just below 2^53 ms (the pane comes from a double multiplication plus a fix-up) and just above it
    (integer division)."""
    T53 = 1 << 53
    rng = np.random.default_rng(53)
    batches = []
    for lo in (T53 - 1, T53 - 1000, T53 + 1, T53 + 2001):
        ts = lo + rng.integers(0, 2500, 500)
        ts[0] = lo
        batches.append(columns_to_batch(ts, rng.random(500) * 9.0, [b"big-%d" % (i % 6) for i in range(500)]))
    batches = sorted(batches, key=lambda b: int(b.ts.min()))
    batches.append(sentinel(T53 + 100_000))
    for L, S in [(1000, 0), (3000, 1000)]:
        st = run_paths(batches, L, S, names=("hinted", "generic"))
        assert st["hinted"]["fast_tiles"] == 9


def test_window_slide_ratio_limit():
    """L / S = 64 panes per window is accepted and matches the oracle; 65 is refused at creation."""
    from denormalized_b200 import DnzError
    rng = np.random.default_rng(64)
    batches = [columns_to_batch(T0 + b * 900 + rng.integers(0, 900, 200), rng.random(200),
                                [b"r%d" % x for x in rng.integers(0, 5, 200)]) for b in range(100)]
    batches.append(sentinel(T0 + 100 * 900 + 3 * 64_000))
    want = run_oracle_batches(batches, 64_000, 1000)
    got, _ = run_gpu(batches, 64_000, 1000, per_batch_poll=False)
    assert len(want) > 500
    assert_rows_equal(got, want)
    with pytest.raises(DnzError) as e:
        gpu_window(65_000, 1000)
    assert e.value.code == -2                              # DNZ_ERR_UNSUPPORTED


# =============================================================================================================================
# E. dictionary collisions and insert races
def _cluster_candidates(n=4_000_000):
    """sensor_1%07d: 15 B keys that share their first key word, so keys of one cluster differ only in the second."""
    i = np.arange(n, dtype=np.int64)
    a = np.zeros((n, 16), np.uint8)
    a[:, :8] = np.frombuffer(b"sensor_1", np.uint8)
    for p in range(7):
        a[:, 8 + p] = 48 + (i // 10 ** (6 - p)) % 10
    w = a.view("<u4").reshape(n, 4)
    return i, hash_words(w[:, 0], w[:, 1], w[:, 2], w[:, 3], np.full(n, 15, np.uint32))


def _collision_keys():
    # equal full 32-bit hashes: 16 B sensor_%9d keys (the cluster family above has none: only its last two words vary)
    ids = np.unique(np.random.default_rng(5).integers(10 ** 8, 10 ** 9, 4_000_000))
    cand = [b"sensor_%d" % x for x in ids.tolist()]
    h = hash_keys(cand)
    order = np.argsort(h, kind="stable")
    eq = np.nonzero(h[order][1:] == h[order][:-1])[0]
    pairs = [(cand[order[e]], cand[order[e + 1]]) for e in eq[:40]]
    i, h = _cluster_candidates()
    clusters = []
    for bits, size, count in ((16, 32, 6), (21, 32, 6)):       # one home slot while the table has <= 2^bits slots
        low = (h & np.uint32((1 << bits) - 1)).astype(np.int64)
        cnt = np.bincount(low, minlength=1 << bits)
        for b in np.argsort(-cnt, kind="stable")[:count]:
            clusters.append([b"sensor_1%07d" % int(j) for j in np.nonzero(low == b)[0][:size]])
    return pairs, clusters


def test_colliding_keys_on_every_probe_path():
    """Pairs of 16 B keys with the same full 32-bit hash (the same chain at every table size) and clusters of 15 B keys that share
    their home slot at 2^14..2^16 slots (the `private` table) and at 2^21 slots (the `hinted` table).  The keys of a cluster share
    their first key word and their length, so only the second word tells them apart."""
    pairs, clusters = _collision_keys()
    assert len(pairs) >= 20 and min(len(c) for c in clusters) >= 4
    for a, b in pairs:
        assert hash_keys([a])[0] == hash_keys([b])[0] and len(a) == len(b) == 16 and a != b
    keys = sorted({k for p in pairs for k in p} | {k for c in clusters for k in c})
    assert len(keys) < 900                                  # no growth at 1024 groups: the collisions stay on one table
    rng = np.random.default_rng(32)
    batches = []
    for b in range(24):
        n = 8 * TILE
        k = rng.integers(0, len(keys), n)
        v = _adversarial_values(rng, k, b)
        batches.append(columns_to_batch(T0 + b * 250 + rng.integers(0, 250, n), v, [keys[j] for j in k]))
    batches.append(sentinel(T0 + 10_000))
    st = run_paths(batches, 1000, 0, names=("private", "hinted", "hinted_noqueue"))
    for name, s in st.items():
        assert s["groups"] == len(keys) + 1 and s["deferred_rows"] == 0 and s["fast_tiles"] > 0, name


def _storm_batches(n_rows, batch_rows):
    """Every key new; each key occurs once in four tiles that belong to four different producer claims (4 tiles each), so four
    CTAs probe its slot while one of them inserts it.  Inline keys of 9-16 B (both key words non-zero) and 24 B arena keys, few
    enough that they fit the long-key arena's initial 1 MiB (a full arena defers rows, which would take them out of the race)."""
    n_tiles = n_rows // TILE
    t = np.arange(n_rows, dtype=np.int64) // TILE
    r = np.arange(n_rows, dtype=np.int64) % TILE
    u = t % 16
    kid = (t // 16) * (4 * TILE) + (u % 4) * TILE + (r + 97 * (u // 4)) % TILE
    n_keys = int(kid.max()) + 1
    ids = np.arange(n_keys)
    inline = ids % 128 != 0
    names = [b"s%0*d" % (8 + j % 8, j) if inline[j] else b"storm-long-key-%09d" % j for j in range(n_keys)]
    lens = np.fromiter((len(x) for x in names), np.int64, n_keys)
    starts = np.zeros(n_keys + 1, np.int64)
    np.cumsum(lens, out=starts[1:])
    blob = np.frombuffer(b"".join(names), np.uint8)
    rng = np.random.default_rng(8)
    val = (rng.random(n_rows) - 0.5) * 200.0
    ts = T0 + np.arange(n_rows, dtype=np.int64) // 20_000
    out = []
    for r0 in range(0, n_rows, batch_rows):
        k = kid[r0:r0 + batch_rows]
        kl = lens[k]
        off = np.zeros(len(k) + 1, np.int64)
        np.cumsum(kl, out=off[1:])
        src = np.repeat(starts[k] - off[:-1], kl) + np.arange(int(off[-1]))
        kb = np.concatenate([blob[src], np.zeros(16, np.uint8)])
        from oracle import Batch
        out.append(Batch(ts=ts[r0:r0 + batch_rows].copy(), val=val[r0:r0 + batch_rows].copy(), key_off=off.astype(np.int32), key_bytes=kb))
    assert n_tiles % 16 == 0 and all(len(x) >= 9 for x in names[:8])
    return out, n_keys


def test_insert_storm_interns_every_key_once():
    """8 Mi rows in one launch, every key new and probed by several CTAs while it is inserted: groups == distinct keys (a key
    interned twice would split its rows between two groups) and row-by-row parity with the oracle."""
    n_rows = 8 * 1024 * 1024 - (8 * 1024 * 1024) % (16 * TILE)
    batches, n_keys = _storm_batches(n_rows, 1 << 20)
    w = gpu_window(60_000, 0, None, expected_groups=n_keys)
    for b in batches:
        w.push(to_record_batch(b))
    got = [w.poll()]
    st0 = w.stats()
    end = sentinel(T0 + 10_000_000)
    w.push(to_record_batch(end))
    got.append(w.poll())
    w.close()
    assert st0["groups"] == n_keys
    assert st0["agg_launches"] == 1 and st0["deferred_rows"] == 0 and st0["fast_tiles"] > 0.9 * n_rows / TILE
    want = oracle_mt_arrays(batches + [end], 60_000)
    gt = pa.concat_tables([record_batch_table(rb, "g") for rb in got])
    wt = result_table(want, "w")
    assert wt.num_rows >= n_keys
    assert assert_tables_equal(gt, wt) == wt.num_rows


# =============================================================================================================================
# F. the filter at the totalOrder edges
def _special_stream():
    nan, inf = float("nan"), float("inf")
    per_key = {b"zn": [-0.0, 0.0], b"zp": [0.0, -0.0], b"z0": [0.0], b"z-": [-0.0], b"nan": [nan], b"nanmix": [7.25, nan],
               b"pinf": [inf], b"ninf": [-inf], b"infs": [inf, -inf], b"neg": [-3.5, -1.0], b"pos": [2.0, 7.25],
               b"zpos": [0.0, 3.0], b"zneg": [-2.0, -0.0], b"null": [None], b"exact": [7.25, 7.25], b"negz": [-7.25, 0.0]}
    batches = []
    for w in range(3):
        rows = []
        for j, (k, vals) in enumerate(per_key.items()):
            order = vals if w != 1 else vals[::-1]
            rows += [(T0 + w * 1000 + 10 * j + i, v, k) for i, v in enumerate(order)]
        batches.append(rows_to_batch(rows))
    batches.append(sentinel(T0 + 6000))
    return batches


@pytest.mark.parametrize("agg", ["count", "min", "max", "average"])
def test_filter_grid_at_total_order_edges(agg):
    """Every operator against -0.0, +0.0, NaN, +-inf and a value present in the data, on windows whose min / max / avg are
    +-0.0, NaN and +-inf."""
    batches = _special_stream()
    lits = [-0.0, 0.0, float("nan"), float("inf"), float("-inf"), 7.25, 2.0]
    kept = 0
    for op in [">", ">=", "<", "<=", "==", "!="]:
        for lit in lits:
            filt = (agg, op, lit)
            want = run_oracle_batches(batches, 1000, 0, filt)
            got, _ = run_gpu(batches, 1000, 0, filt)
            try:
                assert_rows_equal(got, want, check_seq=True)
            except AssertionError as e:
                raise AssertionError(f"filter {filt}: {e}") from None
            kept += len(want)
    assert kept > 0
    full = run_oracle_batches(batches, 1000)
    assert any(r[4] is not None and math.isnan(r[6]) for r in full) and any(r[4] == 0.0 and math.copysign(1, r[4]) < 0 for r in full)
