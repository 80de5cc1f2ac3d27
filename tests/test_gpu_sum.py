"""sum(reading) of grouped windows against the oracle on streams whose every sum is exact (run on an H100 with -m gpu).

Values are k / 1024 with integer |k| <= 2^20, both signs, some -0.0, and NULL values and keys in every third batch (the
others carry no validity bitmaps, so their tiles take the fast path).  Any partial sum of fewer than 2^32 of them is a multiple
of 2^-10 below 2^42 in magnitude, so it is exact in f64: every summation order -- lane-pair reductions,
private pane copies, pane combination, exchange merge, checkpoint -- gives the same bits, the sign of a zero sum included (+0.0:
every state starts at +0.0).  So sum is compared bit for bit, and avg too (a correctly rounded division of two exact numbers).
An accumulator narrower than f64 fails: 2^30 of dynamic range does not fit 24 bits.  In-order streams are also checked against
an independent NumPy int64 reduction per (window, key).  Streams that are not exact are checked against math.fsum with the
bound |got - fsum| <= gamma_(n-1) * sum|v| that holds for every summation tree."""
import math

import numpy as np
import pyarrow as pa
import pytest

from oracle import OracleWindow
from tests.helpers import (KERNEL_PATHS, SUM_AGGS, agg_rows, assert_rows_exact, columns_to_batch, rows_to_batch, same_f64,
                           to_record_batch)
from tests.test_gpu_int_keys import IntBatch, int_schema

pytestmark = pytest.mark.gpu
T0 = 1_700_000_000_000
FLAG_SCALAR_PROBE, FLAG_STAGE_TS = 64, 128          # include/dnz_gpu.h
PATHS = {**KERNEL_PATHS, "scalar_probe": (FLAG_SCALAR_PROBE, 0), "stage_ts": (FLAG_STAGE_TS, 0)}
U = 2.0 ** -53


def _bitmap(valid):
    return None if valid.all() else np.packbits(np.concatenate([valid, np.zeros(8, bool)]), bitorder="little")


def key_name(j):
    """Key id -> Utf8 key: empty, long (> 16 B: the long-key arena) and short inline keys."""
    return b"" if j == 0 else b"long-sensor-key-%06d" % j if j % 11 == 0 else b"s%d" % j


class Utf8Batch:
    def __init__(self, b):
        self.b = b

    def record_batch(self):
        return to_record_batch(self.b)

    def oracle(self):
        return self.b


def exact_stream(rng, n_batches, rows, n_keys, *, typ=None, span_ms=300, late_every=0, late_shift_ms=0, null_frac=0.02, t0=T0,
                 values=None):
    """-> (batches, raw): batches with record_batch() / oracle(); raw = (ts, k, value valid, key id or -1 for NULL) per batch.
    Every third batch has NULL values (null_frac) and NULL keys (1 %): the others have no validity bitmaps.
    `values(rng, n)` replaces the exact values k / 1024 (raw k is then meaningless)."""
    batches, raw, t = [], [], t0
    for bi in range(n_batches):
        back = late_shift_ms if (late_every and bi % late_every == late_every - 1) else 0
        ts = t - back + rng.integers(0, span_ms, rows)
        k = rng.integers(-2 ** 20, 2 ** 20 + 1, rows)
        val = k / 1024.0 if values is None else values(rng, rows)
        negz = rng.random(rows) < 0.01
        k[negz] = 0
        if values is None:
            val[negz] = -0.0
        nulls = bi % 3 == 1                            # batches without validity bitmaps take the fast tiles (TILE_FAST)
        vvalid = rng.random(rows) >= (null_frac if nulls else 0.0)
        kid = rng.integers(0, n_keys, rows)
        kvalid = rng.random(rows) >= (0.01 if nulls else 0.0)
        if typ is None:
            b = columns_to_batch(ts, val, [key_name(j) for j in kid])
            b.val_valid, b.key_valid = _bitmap(vvalid), _bitmap(kvalid)
            batches.append(Utf8Batch(b))
        else:
            batches.append(IntBatch(ts, val, kid * 7919 - 50_000, typ, None, None if vvalid.all() else vvalid, None if kvalid.all() else kvalid))
        raw.append((ts, k, vvalid, np.where(kvalid, kid, -1)))
        t += span_ms
    return batches, raw


def sentinel(ts, typ=None):
    if typ is None:
        return Utf8Batch(rows_to_batch([(ts, 1.0, b"sentinel")]))
    return IntBatch([ts], [1.0], [424242], typ)


def oracle_key(j, typ):
    return None if j < 0 else key_name(j) if typ is None else str(j * 7919 - 50_000).encode()


def exact_reduction(raw, L, S, typ=None):
    """Independent NumPy int64 reduction of an in-order stream: {(window_start, key): (count, sum of k)} for every window a row
    falls in (also groups whose values are all NULL: count 0)."""
    ts = np.concatenate([r[0] for r in raw]); k = np.concatenate([r[1] for r in raw])
    valid = np.concatenate([r[2] for r in raw]); kid = np.concatenate([r[3] for r in raw])
    P = S or L
    out = {}
    for j in range(L // P):
        ws = (ts // P - j) * P
        uniq, inv = np.unique(np.stack([ws, kid], 1), axis=0, return_inverse=True)
        inv = inv.reshape(-1)
        cnt = np.bincount(inv, weights=valid, minlength=len(uniq)).astype(np.int64)
        s = np.zeros(len(uniq), np.int64)
        np.add.at(s, inv, np.where(valid, k, 0))
        for (w, kd), c, sm in zip(uniq.tolist(), cnt.tolist(), s.tolist()):          # pane j of the windows starting at w
            c0, s0 = out.get((w, oracle_key(kd, typ)), (0, 0))
            out[(w, oracle_key(kd, typ))] = (c0 + c, s0 + sm)
    return out


def assert_matches_reduction(rows, exact):
    rows = [r for r in rows if r[2] not in (b"sentinel", b"424242")]
    assert len(rows) == len(exact), f"{len(rows)} rows, the reduction has {len(exact)} (window, key) pairs"
    for r in rows:
        c, s = exact[(r[0], r[2])]
        assert r[3] == c, f"count {r}: {c}"
        want_sum = s / 1024.0 if c else None
        assert same_f64(r[8], want_sum), f"sum {r}: {want_sum}"
        assert same_f64(r[6], None if not c else want_sum / c), f"avg {r}"


def gpu_sum_window(L, S=0, filt=None, typ=None, aggs=SUM_AGGS, **kw):
    from denormalized_b200 import GpuStreamingWindow, canonical_schema
    if typ is None:
        return GpuStreamingWindow(canonical_schema(), "sensor_name", aggs, L, S, filt, **kw)
    return GpuStreamingWindow(int_schema(typ), "id", aggs, L, S, filt, **kw)


def run_sum(batches, L, S=0, filt=None, typ=None, aggs=SUM_AGGS, aliases=None, per_batch_poll=False, **kw):
    w = gpu_sum_window(L, S, filt, typ, aggs, **kw)
    aliases = aliases or [a[2] for a in aggs]
    got = []
    for i, b in enumerate(batches):
        w.push(b.record_batch())
        if per_batch_poll:
            got += agg_rows(w.poll(), aliases, i)
    if not per_batch_poll:
        got += agg_rows(w.poll(), aliases)
    st = w.stats()
    w.close()
    return got, st


def oracle_sum_rows(batches, L, S=0, filt=None):
    o = OracleWindow(L, S, filt)
    for b in batches:
        o.push(b.oracle())
    return o.results(with_sum=True)


def run_exact_paths(batches, L, S=0, typ=None, names=tuple(PATHS), want=None, exact=None, **kw):
    """Every named configuration bit-exact against the oracle (and the NumPy reduction), and bit-identical to each other."""
    want = oracle_sum_rows(batches, L, S) if want is None else want
    stats, ref = {}, None
    for name in names:
        flags, eg = PATHS[name]
        got, st = run_sum(batches, L, S, typ=typ, flags=flags, expected_groups=eg, **kw)
        try:
            assert_rows_exact(got, want)
            if exact is not None:
                assert_matches_reduction(got, exact)
        except AssertionError as e:
            raise AssertionError(f"kernel path {name!r}: {e}") from None
        keyed = sorted(got, key=lambda r: (r[0], r[2] is None, r[2] or b"", r[3], str(r[8])))
        if ref is None:
            ref = (name, keyed)
        else:
            assert all(a[:4] == b[:4] and all(same_f64(a[i], b[i]) for i in (4, 5, 6, 8)) for a, b in zip(keyed, ref[1])), \
                f"kernel paths {ref[0]!r} and {name!r} emit different bits"
        stats[name] = st
    return stats, want


# ================================================================================================ every path, Utf8 and integer keys
@pytest.mark.parametrize("late", [False, True])
@pytest.mark.parametrize("L,S", [(1000, 0), (3000, 1000)])
def test_exact_sum_on_every_path(L, S, late):
    rng = np.random.default_rng(L + S + late)
    kw = dict(late_every=5, late_shift_ms=2500) if late else {}
    batches, raw = exact_stream(rng, 20, 1500, 300, **kw)
    batches.append(sentinel(T0 + 20 * 300 + 3 * L))
    exact = None if late else exact_reduction(raw, L, S)
    stats, want = run_exact_paths(batches, L, S, exact=exact, max_rows_per_launch=4500)
    assert len(want) > 1000
    assert all(s["agg_launches"] >= 5 for s in stats.values())
    if late:
        assert all(s["late_batches"] > 0 for s in stats.values())
    assert stats["hinted"]["fast_tiles"] >= 40 and stats["generic"]["fast_tiles"] == 0       # of 81 tiles


@pytest.mark.parametrize("tname", ["int64", "int32"])
@pytest.mark.parametrize("L,S", [(1000, 0), (3000, 1000)])
def test_exact_sum_integer_keys(tname, L, S):
    typ = {"int64": pa.int64(), "int32": pa.int32()}[tname]
    rng = np.random.default_rng(L + S + len(tname))
    batches, raw = exact_stream(rng, 16, 1500, 400, typ=typ)
    batches.append(sentinel(T0 + 16 * 300 + 3 * L, typ))
    stats, want = run_exact_paths(batches, L, S, typ=typ, exact=exact_reduction(raw, L, S, typ), max_rows_per_launch=4500,
                                  names=("private", "hinted", "generic", "scalar_probe", "stage_ts"))
    assert len(want) > 1000 and stats["hinted"]["fast_tiles"] > 0


# ================================================================================================ paths that only some inputs take
def test_exact_sum_while_the_dictionary_grows():
    """20 K keys introduced batch by batch from a 16-group start: rows replayed by k_deferred after each growth."""
    rng = np.random.default_rng(20)
    batches, t = [], T0
    for b in range(24):
        n = 4000
        hi = min(20_000, (b + 1) * 1000)
        kid = np.concatenate([np.arange(hi - 1000, hi), rng.integers(0, hi, n - 1000)])
        k = rng.integers(-2 ** 20, 2 ** 20 + 1, n)
        batches.append(Utf8Batch(columns_to_batch(t + rng.integers(0, 300, n), k / 1024.0, [b"grow-%05d" % j for j in kid])))
        t += 300
    batches.append(sentinel(t + 4000))
    stats, want = run_exact_paths(batches, 2000, 1000, names=("private", "noprivate_small", "hinted"), max_rows_per_launch=8000)
    assert stats["private"]["deferred_rows"] > 0 and stats["noprivate_small"]["deferred_rows"] > 0
    assert stats["private"]["groups"] == 20_001 and len(want) > 20_000


def test_exact_sum_with_colliding_keys():
    """Keys with equal 32-bit hashes and clusters sharing a home slot: the per-warp retry queue and the in-place probe loop."""
    from tests.test_gpu_kernel_edges import _collision_keys
    pairs, clusters = _collision_keys()
    keys = sorted({k for p in pairs for k in p} | {k for c in clusters for k in c})
    rng = np.random.default_rng(33)
    batches = []
    for b in range(16):
        n = 8 * 416
        k = rng.integers(-2 ** 20, 2 ** 20 + 1, n)
        batches.append(Utf8Batch(columns_to_batch(T0 + b * 250 + rng.integers(0, 250, n), k / 1024.0,
                                                  [keys[j] for j in rng.integers(0, len(keys), n)])))
    batches.append(sentinel(T0 + 10_000))
    stats, _ = run_exact_paths(batches, 1000, 0, names=("private", "hinted", "hinted_noqueue"))
    assert all(s["groups"] == len(keys) + 1 for s in stats.values())


# ================================================================================================ streams that are not exact
def gamma(n):
    return n * U / (1 - n * U)


@pytest.mark.parametrize("L,S", [(1000, 0), (2000, 1000)])
def test_cancellation_within_the_summation_bound(L, S):
    """Values of +-1e6 mixed with small ones: the sum of every (window, key) within gamma_(n-1) * sum|v| of math.fsum on every
    path, avg within that / n + u * |avg|."""
    def values(rng, n):
        big = rng.random(n) < 0.5
        return np.where(big, np.where(rng.random(n) < 0.5, 1e6, -1e6) * (1 + rng.random(n) * 1e-3), rng.random(n) * 3.0 - 1.5)
    rng = np.random.default_rng(7 + S)
    batches, raw = exact_stream(rng, 12, 2000, 40, values=values)
    batches.append(sentinel(T0 + 12 * 300 + 3 * L))
    P = S or L
    vals = np.concatenate([b.oracle().val for b in batches[:-1]])
    ts = np.concatenate([r[0] for r in raw]); valid = np.concatenate([r[2] for r in raw]); kid = np.concatenate([r[3] for r in raw])
    groups = {}
    for j in range(L // P):
        ws = (ts // P - j) * P
        for i in np.nonzero(valid)[0].tolist():
            groups.setdefault((int(ws[i]), key_name(int(kid[i])) if kid[i] >= 0 else None), []).append(float(vals[i]))
    for name in PATHS:
        flags, eg = PATHS[name]
        got, _ = run_sum(batches, L, S, flags=flags, expected_groups=eg, max_rows_per_launch=6000)
        checked = 0
        for r in got:
            if r[2] == b"sentinel" or r[3] == 0:
                continue
            v = groups[(r[0], r[2])]
            n, exact, mag = len(v), math.fsum(v), math.fsum(abs(x) for x in v)
            bound = gamma(n - 1) * mag
            assert r[3] == n and abs(r[8] - exact) <= bound, f"{name}: sum {r} vs fsum {exact} (bound {bound})"
            assert abs(r[6] - exact / n) <= bound / n + U * abs(r[6]) + U * abs(exact / n), f"{name}: avg {r}"
            checked += 1
        assert checked > 100


# ================================================================================================ aggregate lists and the schema
AGG_LISTS = {
    "sum_only": [("sum", "reading", "total")],
    "reordered": [("sum", "reading", "s"), ("avg", "reading", "a"), ("count", "reading", "c"), ("max", "reading", "hi"), ("min", "reading", "lo")],
    "twice": [("sum", "reading", "s1"), ("count", "reading", "n"), ("sum", "reading", "s2"), ("min", "reading", "m"), ("count", "reading", "n2")],
}


@pytest.mark.parametrize("name", list(AGG_LISTS))
@pytest.mark.parametrize("grouped", [True, False])
def test_aggregate_lists(name, grouped):
    """The exported schema (names, order, formats l / g, count non-null and the rest nullable) and every column's values."""
    from denormalized_b200 import GpuStreamingWindow, canonical_schema
    from oracle import OracleUngrouped
    aggs = AGG_LISTS[name]
    rng = np.random.default_rng(len(name) + grouped)
    batches, _ = exact_stream(rng, 10, 800, 50 if grouped else 1, span_ms=1000)
    batches.append(sentinel(T0 + 10 * 1000 + 4000))
    batches[3].oracle().val_valid = _bitmap(np.zeros(800, bool))              # a batch of NULL values only
    w = GpuStreamingWindow(canonical_schema(), "sensor_name" if grouped else None, aggs, 1000, 0, None)
    o = OracleWindow(1000) if grouped else OracleUngrouped(1000)
    col_of = {"count": 3, "min": 4, "max": 5, "avg": 6, "sum": 8}
    n_rows = 0
    for i, b in enumerate(batches):
        w.push(b.record_batch())
        rb = w.poll()
        o.push(b.oracle())
        want = sorted(o.results(with_sum=True), key=lambda r: (r[0], r[2] is None, r[2] or b""))
        head = ["sensor_name"] if grouped else []
        assert rb.schema.names == head + [a[2] for a in aggs] + ["window_start_time", "window_end_time"]
        for f, (kind, _, _) in zip([rb.schema.field(j) for j in range(len(head), len(head) + len(aggs))], aggs):
            assert f.type == (pa.int64() if kind == "count" else pa.float64()) and f.nullable == (kind != "count"), f
        assert rb.schema.field("window_start_time").type == pa.timestamp("ms")
        cols = {n: rb.column(j).to_pylist() for j, n in enumerate(rb.schema.names)}
        ws = rb.column(rb.schema.names.index("window_start_time")).cast(pa.int64()).to_pylist()
        keys = cols["sensor_name"] if grouped else [None] * rb.num_rows
        order = sorted(range(rb.num_rows), key=lambda j: (ws[j], keys[j] is None, (keys[j] or "").encode()))
        assert len(order) == len(want), (i, len(order), len(want))
        for j, r in zip(order, want):
            assert ws[j] == r[0] and (keys[j].encode() if keys[j] is not None else None) == r[2]
            for kind, _, alias in aggs:
                assert same_f64(cols[alias][j], r[col_of[kind]]) if kind != "count" else cols[alias][j] == r[3], (alias, cols[alias][j], r)
        n_rows += len(want)
    w.close()
    assert n_rows > (200 if grouped else 5)


# ================================================================================================ the fused filter
FILTER_AGGS = [("sum", "reading", "total"), ("count", "reading", "n"), ("avg", "reading", "mean"), ("min", "reading", "lo"),
               ("max", "reading", "hi")]


def _filter_stream():
    rng = np.random.default_rng(44)
    batches, _ = exact_stream(rng, 6, 600, 30, span_ms=500)
    nan, inf = float("nan"), float("inf")
    special = {b"zero": [2.5, -2.5], b"negz": [-0.0], b"nan": [1.0, nan], b"pinf": [inf], b"ninf": [-inf, 3.0], b"infs": [inf, -inf],
               b"null": [None], b"one": [0.125]}
    for w in range(3):
        rows = [(T0 + w * 1000 + 10 * j + i, v, k) for j, (k, vals) in enumerate(special.items()) for i, v in enumerate(vals)]
        batches.append(Utf8Batch(rows_to_batch(rows)))
    batches.append(sentinel(T0 + 9000))
    return batches


@pytest.mark.parametrize("alias,kind", [("total", "sum"), ("mean", "avg"), ("n", "count")])
def test_filter_on_aggregates_at_other_list_positions(alias, kind):
    """sum sits at list position 0, count at 1 and avg at 2: the filter must follow the aggregate's kind, not its position.  Every
    operator against a window's exact sum, +-0.0, NaN and +-inf."""
    batches = _filter_stream()
    full = oracle_sum_rows(batches, 1000)
    exact = next(r[8] for r in full if r[2] and r[2].startswith(b"s") and r[8] not in (None, 0.0))
    lits = [exact, 0.0, -0.0, float("nan"), float("inf"), float("-inf"), 2.0]
    kept = 0
    for op in [">", ">=", "<", "<=", "==", "!="]:
        for lit in lits:
            want = oracle_sum_rows(batches, 1000, 0, (kind, op, lit))
            got, _ = run_sum(batches, 1000, 0, (alias, op, lit), aggs=FILTER_AGGS, aliases=["n", "lo", "hi", "mean", "total"])
            try:
                assert_rows_exact(got, want)
            except AssertionError as e:
                raise AssertionError(f"filter {(alias, op, lit)}: {e}") from None
            kept += len(want)
            if op == "==" and lit == exact and kind == "sum":
                assert len(want) >= 1
    assert kept > 0


# ================================================================================================ other ways out
def test_poll_ready_and_device_polls():
    rng = np.random.default_rng(5)
    batches, raw = exact_stream(rng, 16, 2000, 500)
    batches.append(sentinel(T0 + 16 * 300 + 3000))
    exact = exact_reduction(raw, 1000, 0)
    want = oracle_sum_rows(batches, 1000)
    # poll_ready between pushes, one blocking poll at the end
    w = gpu_sum_window(1000)
    got = []
    for b in batches:
        w.push(b.record_batch())
        got += agg_rows(w.poll_ready())
    got += agg_rows(w.poll())
    w.close()
    assert_rows_exact(got, want)
    assert_matches_reduction(got, exact)
    # device-resident results
    w = gpu_sum_window(1000)
    got = []

    def rows_of(r):
        if not r.n_rows:
            return []
        a = w.fetch_device_result(r)
        ok = a["agg_valid"]
        return [(int(a["window_start"][i]), int(a["window_end"][i]), a["key"][i], int(a["count"][i]),
                 float(a["min"][i]) if ok[i] else None, float(a["max"][i]) if ok[i] else None, float(a["avg"][i]) if ok[i] else None, 0,
                 float(a["sum"][i]) if ok[i] else None) for i in range(r.n_rows)]
    for b in batches:
        w.push(b.record_batch())
        got += rows_of(w.poll_device_ready())
    while True:
        r = w.poll_device()
        if not r.n_rows:
            break
        got += rows_of(r)
    w.close()
    assert_rows_exact(got, want)
    assert_matches_reduction(got, exact)


# ================================================================================================ exchange and checkpoint
def _exchange_stream():
    rng = np.random.default_rng(77)
    batches, raw = exact_stream(rng, 32, 1500, 600, span_ms=200)
    close = (T0 + 32 * 200) // 1000 * 1000 + 3000
    return batches, raw, close


@pytest.mark.parametrize("world", [2, 4])
def test_fused_exchange_sum_is_exact(world):
    from denormalized_b200 import ExchangeGroup
    batches, raw, close = _exchange_stream()
    want = oracle_sum_rows(batches + [sentinel(close)], 1000)
    one, _ = run_sum(batches + [sentinel(close)], 1000)
    assert_rows_exact(one, want)
    groups = ExchangeGroup.create_local([0] * world, ring_entries=1 << 16, ring_key_bytes=4 << 20)
    wins = [gpu_sum_window(1000, expected_groups=4096) for _ in range(world)]
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
            got.extend(agg_rows(w.poll()))
    for i, b in enumerate(batches):
        wins[i % world].push(b.record_batch())
        if i % (2 * world) == 2 * world - 1:
            step()
    for w in wins:
        w.push(sentinel(close).record_batch())
    for _ in range(3):                                 # publish | pack | merge + emit
        step(force=True)
    step()
    st = [w.stats() for w in wins]
    for w in wins:
        w.close()
    for g in groups:
        g.close()
    assert sum(s["exchanged_in"] for s in st) > 500
    assert_rows_exact(got, want)
    assert_matches_reduction(got, exact_reduction(raw, 1000, 0))


def test_host_driven_exchange_sum_is_exact():
    from denormalized_b200.exchange import LocalTransport
    world = 2
    batches, raw, close = _exchange_stream()
    want = oracle_sum_rows(batches + [sentinel(close)], 1000)
    wins = [gpu_sum_window(1000, expected_groups=64) for _ in range(world)]
    for r, w in enumerate(wins):
        w.set_exchange(r, world)
    lt = LocalTransport(wins)
    got = []
    for i, b in enumerate(batches):
        wins[i % world].push(b.record_batch())
        if i % 6 == 5:
            got += [r for rb in lt.exchange_all() for r in agg_rows(rb)]
    for w in wins:
        w.push(sentinel(close).record_batch())
    got += [r for rb in lt.exchange_all() for r in agg_rows(rb)]
    st = [w.stats() for w in wins]
    for w in wins:
        w.close()
    assert sum(s["exchanged_out"] for s in st) == sum(s["exchanged_in"] for s in st) > 500
    assert_rows_exact(got, want)
    assert_matches_reduction(got, exact_reduction(raw, 1000, 0))


@pytest.mark.parametrize("L,S", [(1000, 0), (3000, 1000)])
def test_checkpoint_restore_mid_stream(L, S):
    rng = np.random.default_rng(L + S + 1)
    batches, raw = exact_stream(rng, 16, 1500, 400)
    batches.append(sentinel(T0 + 16 * 300 + 3 * L))
    want = oracle_sum_rows(batches, L, S)
    w = gpu_sum_window(L, S)
    got = []
    for b in batches[:7]:
        w.push(b.record_batch())
        got += agg_rows(w.poll())
    blob = w.checkpoint()
    w.close()
    w2 = gpu_sum_window(L, S)
    w2.restore(blob)
    for b in batches[7:]:
        w2.push(b.record_batch())
        got += agg_rows(w2.poll())
    w2.close()
    assert_rows_exact(got, want)
    assert_matches_reduction(got, exact_reduction(raw, L, S))
