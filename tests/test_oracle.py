"""CPU-only: pins the C oracle against (a) an independent pure-Python model of the reference semantics,
(b) pyarrow/Acero group_by arithmetic, (c) the reference's one adjacent known-answer
(crates/core/src/utils/serialization.rs:535-557), and (d) hand-computed window enumerations."""
import math

import numpy as np
import pyarrow as pa
import pytest

from oracle import OracleMT, OracleWindow, synth_batch, sort_rows
from tests.helpers import assert_rows_equal, random_stream, rows_to_batch, batch_to_rows
from tests.pymodel import PyModel, windows_for

T0 = 1_700_000_000_000


def run_oracle(batches, L, S=0, filt=None):
    o = OracleWindow(L, S, filt)
    for rows in batches:
        o.push(rows_to_batch(rows))
    return o.results()


def run_model(batches, L, S=0, filt=None):
    m = PyModel(L, S, filt)
    for rows in batches:
        m.push(rows)
    return m.out


def test_known_answer_avg_56():
    # test_avg_accumulator_serialization: 56 copies of 56.0 -> avg 56.0 (state = [count, sum])
    rows = [(T0 + 5, 56.0, b"a")] * 56
    out = run_oracle([rows, [(T0 + 5000, 1.0, b"a")]], 1000)
    assert out == [(T0, T0 + 1000, b"a", 56, 56.0, 56.0, 56.0, 1)]


def test_window_enumeration_tumbling_and_sliding():
    # tumbling 1 s: batch covering [t0+100, t0+2100] -> 3 windows
    assert windows_for(T0 + 100, T0 + 2100, 1000, 0) == [(T0, T0 + 1000), (T0 + 1000, T0 + 2000), (T0 + 2000, T0 + 3000)]
    # sliding 10 s / 1 s, single-ms batch -> windows with start in [t-10s, t], INCLUSIVE end test keeps end == min
    w = windows_for(T0, T0, 10_000, 1000)
    assert w[0] == (T0 - 10_000, T0) and w[-1] == (T0, T0 + 10_000) and len(w) == 11
    # the C oracle opens exactly these frames (the first one gets 0 rows and emits nothing)
    o = OracleWindow(10_000, 1000)
    o.push(rows_to_batch([(T0, 1.0, b"a")]))
    assert o.open_frames == 10           # the [T0-10s, T0) frame closed immediately (wm >= end), empty
    assert o.results() == []


@pytest.mark.parametrize("L,S", [(1000, 0), (2000, 0), (5000, 1000), (10_000, 1000), (4000, 2000), (3000, 2000), (1500, 0), (2500, 1000)])
@pytest.mark.parametrize("jitter", [0, 1500])
def test_oracle_matches_python_model(L, S, jitter):
    rng = np.random.default_rng(L * 7 + S + jitter)
    batches = random_stream(rng, 30, 40, 9, span_ms=350, jitter_ms=jitter, ragged=True, late_every=6 if jitter else 0,
                            late_shift_ms=3 * jitter)
    batches.append([(T0 + 30 * 350 + 3 * L, 1.0, b"sentinel")])
    assert_rows_equal(run_oracle(batches, L, S), run_model(batches, L, S), rel=0.0, check_seq=True)


def test_oracle_nulls_and_special_values_match_model():
    rng = np.random.default_rng(5)
    batches = random_stream(rng, 25, 50, 6, span_ms=300, null_frac=0.15, special_vals=True)
    batches[0] = batches[0] + [(T0 + 5, None, b"onlynull"), (T0 + 6, None, b"onlynull")]
    batches.append([(T0 + 25 * 300 + 5000, 1.0, b"s")])
    for L, S in [(1000, 0), (3000, 1000)]:
        got, want = run_oracle(batches, L, S), run_model(batches, L, S)
        assert any(r[2] is None for r in got) and any(r[4] is None for r in got)
        assert_rows_equal(got, want, rel=0.0, check_seq=True)


def test_min_max_quirks():
    # NaN never replaces; +-0.0 keeps the first seen; +inf never lowers f64::MAX start; all-NaN group -> MAX/MIN
    F = 1.7976931348623157e308
    rows = [(T0, float("nan"), b"nan"), (T0, -0.0, b"z1"), (T0 + 1, 0.0, b"z1"), (T0, 0.0, b"z2"), (T0 + 1, -0.0, b"z2"),
            (T0, float("inf"), b"pinf"), (T0, float("-inf"), b"ninf"), (T0, 5.0, b"mix"), (T0, float("nan"), b"mix")]
    out = {r[2]: r for r in run_oracle([rows, [(T0 + 3000, 1.0, b"s")]], 1000)}
    assert out[b"nan"][4] == F and out[b"nan"][5] == -F and math.isnan(out[b"nan"][6]) and out[b"nan"][3] == 1
    assert math.copysign(1, out[b"z1"][4]) == -1 and math.copysign(1, out[b"z1"][5]) == -1
    assert math.copysign(1, out[b"z2"][4]) == 1 and math.copysign(1, out[b"z2"][5]) == 1
    assert out[b"pinf"][4] == F and out[b"pinf"][5] == float("inf")
    assert out[b"ninf"][4] == float("-inf") and out[b"ninf"][5] == -F
    assert out[b"mix"][4] == 5.0 and out[b"mix"][5] == 5.0 and math.isnan(out[b"mix"][6])


def test_filter_total_order():
    rows = [(T0, 114.0, b"hi"), (T0, 112.0, b"lo"), (T0, float("nan"), b"nan"), (T0, None, b"null"), (T0, 113.0, b"eq")]
    close = [(T0 + 3000, 1.0, b"s")]
    got = {r[2] for r in run_oracle([rows, close], 1000, filt=("max", ">", 113))}
    # arrow-rs cmp::gt is totalOrder: the all-NaN group's max is f64::MIN (NaN never replaces) -> dropped;
    assert got == {b"hi"}
    got = {r[2] for r in run_oracle([rows, close], 1000, filt=("average", ">", 113))}
    assert got == {b"hi", b"nan"}          # avg of NaN is NaN; NaN > 113.0 under totalOrder
    got = {r[2] for r in run_oracle([rows, close], 1000, filt=("count", ">=", 1))}
    assert got == {b"hi", b"lo", b"nan", b"eq"}
    assert_rows_equal(run_oracle([rows, close], 1000, filt=("max", ">=", 113)), run_model([rows, close], 1000, filt=("max", ">=", 113)), check_seq=True)


def test_late_rows_reopen_window_and_unclosed_windows_never_emit():
    b1 = [(T0 + 100, 1.0, b"a"), (T0 + 900, 3.0, b"a")]
    b2 = [(T0 + 1500, 5.0, b"a")]                       # wm -> T0+1500: closes [T0, T0+1000)
    b3 = [(T0 + 200, 7.0, b"a"), (T0 + 1600, 9.0, b"a")]  # late row re-opens [T0,T0+1000) -> second partial row
    o = OracleWindow(1000)
    outs = []
    for rows in (b1, b2, b3):
        o.push(rows_to_batch(rows))
        outs.append(o.results())
    assert outs[0] == []
    assert outs[1] == [(T0, T0 + 1000, b"a", 2, 1.0, 3.0, 2.0, 1)]
    assert outs[2] == [(T0, T0 + 1000, b"a", 1, 7.0, 7.0, 7.0, 2)]
    assert o.open_frames == 1 and o.watermark == T0 + 1500   # [T0+1000, T0+2000) stays open forever


def test_empty_batch_does_not_trigger():
    o = OracleWindow(1000)
    o.push(rows_to_batch([(T0 + 10, 1.0, b"a")]))
    assert o.push(rows_to_batch([])) == 0
    assert o.results() == []


def test_error_cases():
    o = OracleWindow(1000)
    with pytest.raises(RuntimeError):
        o.push(rows_to_batch([(None, 1.0, b"a")]))
    o = OracleWindow(500)
    with pytest.raises(RuntimeError):
        o.push(rows_to_batch([(T0, 1.0, b"a")]))


def test_arithmetic_against_pyarrow_group_by():
    """Acero as a second opinion for count/min/max (exact) and mean (1e-9) per window."""
    nb, n = 12, 4096
    batches = [synth_batch(i * n, n, groups=50, rows_per_ms=8) for i in range(nb)]
    o = OracleWindow(1000)
    for b in batches:
        o.push(b)
    o.push(rows_to_batch([(T0 + 60_000, 0.0, b"s")]))
    got = o.results()
    ts = np.concatenate([b.ts for b in batches])
    val = np.concatenate([b.val for b in batches])
    keys = sum(([r[2] for r in batch_to_rows(b)] for b in batches), [])
    tbl = pa.table({"w": (ts // 1000) * 1000, "k": pa.array(keys, pa.binary()), "v": val})
    agg = tbl.group_by(["w", "k"], use_threads=False).aggregate([("v", "count"), ("v", "min"), ("v", "max"), ("v", "mean")])
    want = [(w, w + 1000, k, c, mn, mx, av, 0) for w, k, c, mn, mx, av in zip(*[agg[c].to_pylist() for c in ["w", "k", "v_count", "v_min", "v_max", "v_mean"]])]
    assert len(got) == len(want) > 100
    assert_rows_equal(got, want, rel=1e-9)


def test_synth_generator_properties():
    b = synth_batch(0, 10_000, groups=1000, rows_per_ms=1000)
    assert b.ts[0] == T0 and b.ts[-1] == T0 + 9 and np.all(np.diff(b.ts) >= 0)
    assert 0.0 <= b.val.min() and b.val.max() < 115.0
    rows = batch_to_rows(b)
    assert all(r[2].startswith(b"sensor_") and 0 <= int(r[2][7:]) < 1000 for r in rows)
    # counter based: any slice reproduces
    c = synth_batch(5000, 100, groups=1000, rows_per_ms=1000)
    assert batch_to_rows(c) == rows[5000:5100]
    u = synth_batch(0, 64, groups=10, uuid_keys=True)
    ku = batch_to_rows(u)[0][2]
    assert len(ku) == 36 and ku[8:9] == b"-" and ku[13:14] == b"-" and ku[18:19] == b"-" and ku[23:24] == b"-"


def test_mt_partitioned_equals_single_partition():
    nb, n = 40, 2048
    batches = [synth_batch(i * n, n, groups=300, rows_per_ms=10, extra_columns=True) for i in range(nb)]
    sentinel = rows_to_batch([(T0 + 100_000, 0.0, b"s")])
    for L, S in [(1000, 0), (4000, 1000)]:
        o = OracleWindow(L, S, ("max", ">", 100))
        for b in batches + [sentinel]:
            o.push(b)
        want = o.results()
        m = OracleMT(L, S, ("max", ">", 100), partitions=4)
        m.push_many(batches + [sentinel])
        got = m.results()
        assert len(want) > 50
        assert_rows_equal(got, want, rel=0.0)


@pytest.mark.parametrize("L,S", [(3000, 2000), (1500, 0)])
def test_non_lattice_geometries_depend_on_batch_boundaries(L, S):
    """Why the GPU operator rejects L % S != 0 and L that is not a whole number of seconds (DNZ_ERR_UNSUPPORTED): the reference
    enumerates a batch's windows from snap_to_window_start(batch minimum) in steps of the slide (streaming_window.rs:1053-1094),
    so on these geometries the SET of windows -- not just their content -- depends on where the stream is cut into batches.  The
    same 40 rows in one batch, in four batches and in four ragged batches give three different window sets; both the C oracle and
    the independent Python model say so.  On the lattice geometries (L a whole number of seconds, L % S == 0) the cut does not
    matter, which is what a pane organisation needs."""
    rows = [(T0 + 250 * i, float(i), b"a") for i in range(40)]        # 10 s of rows, 4 per second
    close = [(T0 + 60_000, 1.0, b"z")]

    def window_set(run, cuts, l, s):
        batches, i = [], 0
        for c in cuts:
            batches.append(rows[i:i + c]); i += c
        return sorted({(r[0], r[1]) for r in run(batches + [close], l, s) if r[2] == b"a"})
    cuts = ([40], [10, 10, 10, 10], [3, 7, 11, 19])
    sets = [window_set(run_oracle, c, L, S) for c in cuts]
    assert sets[0] != sets[1] and sets[1] != sets[2] and sets[0] != sets[2]
    assert [window_set(run_model, c, L, S) for c in cuts] == sets       # the independent model agrees on every cut
    for l, s in [(2000, 0), (4000, 1000), (4000, 2000)]:                  # lattice geometries: the cut is irrelevant
        lattice = [window_set(run_oracle, c, l, s) for c in cuts]
        assert lattice[0] == lattice[1] == lattice[2]


@pytest.mark.parametrize("L,S", [(1000, 0), (2000, 0), (4000, 1000), (6000, 2000)])
@pytest.mark.parametrize("late", [False, True])
def test_ungrouped_oracle_matches_python_model(L, S, late):
    """`.window([], aggs, ..)` (SURVEY §8 f2): the C restatement of the Partial -> Final chain against the independent Python model,
    batch by batch (emission lag of the Final stage, batches that close several Partial windows at once merged into the frame of the
    largest start, late partial results dropped), NULL values and windows that only see NULLs included."""
    from oracle import OracleUngrouped
    from tests.pymodel import PyUngroupedModel
    rng = np.random.default_rng(7 * L + S + late)
    kw = dict(jitter_ms=500, late_every=5, late_shift_ms=2500) if late else dict(null_frac=0.15, ragged=True)
    raw = random_stream(rng, 60, 200, 3, span_ms=300, **kw)
    if not late:
        raw[7] = [(ts, None, k) for ts, _, k in raw[7]]             # a batch of NULL values only
    o, m = OracleUngrouped(L, S), PyUngroupedModel(L, S)
    got = []
    for rows in raw:
        o.push(rows_to_batch(rows)); got += o.results()
        m.push(rows)
    assert len(m.out) > 3
    assert_rows_equal(got, m.out, check_seq=True)


def test_ungrouped_oracle_special_values_match_model():
    """totalOrder min / max over NaN, +-0.0, +-inf; a window that sees zeros only; windows that only see NULL values."""
    from oracle import OracleUngrouped
    from tests.pymodel import PyUngroupedModel
    vals = [float("nan"), -0.0, 0.0, float("inf"), float("-inf"), 5.0, -3.0, None, -float("nan")]
    o, m, got = OracleUngrouped(1000, 0), PyUngroupedModel(1000, 0), []
    for b in range(24):
        rows = [(T0 + b * 500 + i, vals[(b + i) % len(vals)], b"x") for i in range(40)]
        if b in (4, 5):
            rows = [(T0 + b * 500 + i, -0.0 if (i + b) % 2 else 0.0, b"x") for i in range(40)]
        if b in (8, 9):
            rows = [(T0 + b * 500 + i, None, b"x") for i in range(10)]
        if b in (12, 13):
            rows = [(T0 + b * 500 + i, -0.0, b"x") for i in range(10)]          # only negative zeros: min = max = -0.0, but the
                                                                                # sum starts from +0.0 (get_or_insert(0.)): avg +0.0
        o.push(rows_to_batch(rows)); got += o.results()
        m.push(rows)
    assert any(r[4] is None and r[3] == 0 for r in m.out)
    zeros = [r for r in m.out if r[0] == T0 + 2000][0]
    assert math.copysign(1.0, zeros[4]) == -1.0 and math.copysign(1.0, zeros[5]) == 1.0 and zeros[4] == 0.0 == zeros[5]
    negz = [r for r in m.out if r[0] == T0 + 6000][0]
    assert negz[3] == 20 and math.copysign(1.0, negz[4]) == -1.0 and math.copysign(1.0, negz[6]) == 1.0
    assert_rows_equal(got, m.out, check_seq=True)
    assert all(math.copysign(1.0, a[6]) == math.copysign(1.0, b[6]) for a, b in zip(got, m.out) if a[6] == 0.0)     # zero signs too


# sum(reading): PrimitiveGroupsAccumulator (grouped) and SumAccumulator (ungrouped) -- +0.0, then += v; NULL when no value was seen
def exact_rows(rng, n_batches, rows, n_keys, span_ms=300, null_frac=0.02):
    """Rows whose values are k / 1024 with integer |k| <= 2^20: every partial sum is exact in f64, whatever the order."""
    out, t = [], T0
    for _ in range(n_batches):
        b = []
        for _ in range(rows):
            k = int(rng.integers(-2 ** 20, 2 ** 20 + 1))
            b.append((t + int(rng.integers(0, span_ms)), None if rng.random() < null_frac else k / 1024.0, b"k%d" % int(rng.integers(0, n_keys))))
        out.append(b)
        t += span_ms
    return out


def _window_sums(batches, L):
    """{(window_start, key): exact integer sum of 1024 * v} of in-order tumbling windows, NULL values left out."""
    acc = {}
    for rows in batches:
        for ts, v, k in rows:
            if v is not None:
                acc[(ts // L * L, k)] = acc.get((ts // L * L, k), 0) + int(v * 1024)
    return acc


@pytest.mark.parametrize("L,S", [(1000, 0), (4000, 1000)])
def test_oracle_sum_matches_model_and_exact_integers(L, S):
    from tests.helpers import assert_rows_exact
    rng = np.random.default_rng(L + S)
    batches = exact_rows(rng, 24, 60, 7)
    batches.append([(T0 + 24 * 300 + 3 * L, 1.0, b"sentinel")])
    o = OracleWindow(L, S)
    for rows in batches:
        o.push(rows_to_batch(rows))
    got = o.results(with_sum=True)
    assert len(got) > 20 and all(len(r) == 9 for r in got)
    assert_rows_exact(got, run_model(batches, L, S), check_seq=True)      # avg too: sum and count are exact, so is the division
    if S == 0:
        exact = _window_sums(batches[:-1], L)
        assert {(r[0], r[2]): r[8] for r in got} == {key: s / 1024.0 for key, s in exact.items()}


def test_oracle_sum_against_pyarrow_group_by():
    nb, n = 12, 4096
    batches = [synth_batch(i * n, n, groups=50, rows_per_ms=8) for i in range(nb)]
    for b in batches:                                   # exact values: k / 1024
        b.val = np.round(b.val * 1024.0) / 1024.0 - 57.0
    o = OracleWindow(1000)
    for b in batches:
        o.push(b)
    o.push(rows_to_batch([(T0 + 60_000, 0.0, b"s")]))
    got = {(r[0], r[2]): r[8] for r in o.results(with_sum=True)}
    ts = np.concatenate([b.ts for b in batches])
    keys = sum(([r[2] for r in batch_to_rows(b)] for b in batches), [])
    tbl = pa.table({"w": (ts // 1000) * 1000, "k": pa.array(keys, pa.binary()), "v": np.concatenate([b.val for b in batches])})
    agg = tbl.group_by(["w", "k"], use_threads=False).aggregate([("v", "sum")])
    want = dict(zip(zip(agg["w"].to_pylist(), agg["k"].to_pylist()), agg["v_sum"].to_pylist()))
    assert len(want) > 100 and got == want


def test_oracle_sum_edges():
    """NULL-only -> NULL; -0.0 only -> +0.0 (the state starts at +0.0); NaN; +inf with -inf -> NaN; +inf alone."""
    import struct
    nan, inf = float("nan"), float("inf")
    per_key = {b"null": [None, None], b"negz": [-0.0, -0.0], b"z": [0.0, -0.0], b"nan": [1.5, nan], b"infs": [inf, -inf],
               b"pinf": [inf, 2.0], b"ex": [0.5, 0.25, -0.125]}
    rows = [(T0 + i, v, k) for k, vals in per_key.items() for i, v in enumerate(vals)]
    close = [(T0 + 5000, 1.0, b"s")]
    for run in (run_model, None):
        if run is None:
            o = OracleWindow(1000)
            o.push(rows_to_batch(rows)); o.push(rows_to_batch(close))
            out = {r[2]: r[8] for r in o.results(with_sum=True)}
        else:
            out = {r[2]: r[8] for r in run([rows, close], 1000)}
        assert out[b"null"] is None
        assert struct.pack("<d", out[b"negz"]) == struct.pack("<d", 0.0) and struct.pack("<d", out[b"z"]) == struct.pack("<d", 0.0)
        assert math.isnan(out[b"nan"]) and math.isnan(out[b"infs"]) and out[b"pinf"] == inf and out[b"ex"] == 0.625
    tbl = pa.table({"k": [k for k, vals in per_key.items() for _ in vals], "v": pa.array([v for vals in per_key.values() for v in vals], pa.float64())})
    pa_sum = dict(zip(*[tbl.group_by("k", use_threads=False).aggregate([("v", "sum")])[c].to_pylist() for c in ("k", "v_sum")]))
    assert pa_sum[b"null"] is None and pa_sum[b"ex"] == 0.625 and math.isnan(pa_sum[b"infs"]) and pa_sum[b"pinf"] == inf


@pytest.mark.parametrize("op", [">", ">=", "<", "<=", "==", "!="])
def test_oracle_sum_filter_matches_model(op):
    rng = np.random.default_rng(11)
    batches = exact_rows(rng, 12, 40, 5)
    special = [(T0 + 1, 2.5, b"a"), (T0 + 2, -2.5, b"a"), (T0 + 3, -0.0, b"nz"), (T0 + 4, float("nan"), b"nan"),
               (T0 + 5, float("inf"), b"inf"), (T0 + 6, None, b"null")]
    batches[0] = batches[0] + special
    batches.append([(T0 + 12 * 300 + 3000, 1.0, b"sentinel")])
    o = OracleWindow(1000)
    for rows in batches:
        o.push(rows_to_batch(rows))
    exact = next(r[8] for r in o.results(with_sum=True) if r[2] != b"a")
    for lit in (exact, 0.0, -0.0, float("nan"), float("inf"), float("-inf")):
        got, want = run_oracle(batches, 1000, filt=("sum", op, lit)), run_model(batches, 1000, filt=("sum", op, lit))
        assert_rows_equal(got, want, rel=0.0, check_seq=True)
        if lit == exact and op == "==":
            assert got


@pytest.mark.parametrize("L,S", [(1000, 0), (4000, 1000)])
def test_ungrouped_oracle_sum_matches_model(L, S):
    from oracle import OracleUngrouped
    from tests.helpers import assert_rows_exact
    from tests.pymodel import PyUngroupedModel
    rng = np.random.default_rng(3 * L + S)
    raw = exact_rows(rng, 40, 50, 1)
    raw[5] = [(ts, None, k) for ts, _, k in raw[5]]
    raw[9] = [(ts, -0.0, k) for ts, _, k in raw[9]]
    o, m, got = OracleUngrouped(L, S), PyUngroupedModel(L, S), []
    for rows in raw:
        o.push(rows_to_batch(rows)); got += o.results(with_sum=True)
        m.push(rows)
    assert len(m.out) > 3
    assert_rows_exact(got, m.out, check_seq=True)
