"""The experiment switches of k_aggregate's memory traffic must not change a single emitted bit (run on an H100 with -m gpu).

  DNZ_FLAG_SCALAR_PROBE   every row loads both halves of its dictionary slot instead of the lane-paired probe
  DNZ_FLAG_STAGE_TS       the timestamps of tiles inside one pane are staged although no consumer reads them

Each stream runs under every switch alone and under all of them together; count / min / max and the null flags must be
bit-identical across the runs and every run must match the oracle (avg within 1e-9)."""
import math

import numpy as np
import pytest

import pyarrow as pa

from tests.helpers import (assert_rows_equal, assert_tables_equal, bits, columns_to_batch, gpu_window, host_stream, oracle_mt_arrays,
                           random_stream, record_batch_table, result_table, rows_to_batch, run_gpu, run_oracle_batches, to_record_batch)
from tests.test_gpu_kernel_edges import T0, TILE, _adversarial_values, _collision_keys, _storm_batches, sentinel

pytestmark = pytest.mark.gpu
FLAG_SCALAR_PROBE, FLAG_STAGE_TS = 64, 128       # include/dnz_gpu.h
VARIANTS = {"default": 0, "scalar_probe": FLAG_SCALAR_PROBE, "stage_ts": FLAG_STAGE_TS, "both_off": FLAG_SCALAR_PROBE | FLAG_STAGE_TS}


def _row_bits(r):
    return (r[0], r[1], r[2], r[3], bits(r[4]), bits(r[5]), r[6] is None)


def run_variants(batches, L, S=0, want=None, per_batch_poll=False, **kw):
    """Runs `batches` under every entry of VARIANTS; returns {name: stats}."""
    if want is None:
        want = run_oracle_batches(batches, L, S)
    stats, ref = {}, None
    for name, flags in VARIANTS.items():
        got, st = run_gpu(batches, L, S, per_batch_poll=per_batch_poll, flags=flags, **kw)
        try:
            assert_rows_equal(got, want, check_seq=per_batch_poll)
        except AssertionError as e:
            raise AssertionError(f"variant {name!r}: {e}") from None
        got_bits = sorted(_row_bits(r) for r in got)
        if ref is None:
            ref = got_bits
        else:
            assert got_bits == ref, f"variant {name!r} emits different bits than 'default'"
        stats[name] = st
    return stats


def run_variants_large(batches, L, **kw):
    """The same for streams with hundreds of thousands of result rows: compared as tables (count / min / max bit-exact with the
    oracle, hence with each other).  Returns {name: stats}."""
    want = result_table(oracle_mt_arrays(batches, L), "w")
    stats = {}
    for name, flags in VARIANTS.items():
        w = gpu_window(L, 0, None, flags=flags, **kw)
        for b in batches:
            w.push(to_record_batch(b))
        got = pa.concat_tables([record_batch_table(w.poll(), "g")])
        stats[name] = w.stats()
        w.close()
        try:
            assert assert_tables_equal(got, want) == want.num_rows
        except AssertionError as e:
            raise AssertionError(f"variant {name!r}: {e}") from None
    return stats


def test_cfg2_shaped_stream_under_every_switch():
    """The synthetic sensor stream at cfg 2's key count (100 K groups, 16 B keys), 4 Mi rows over eight 1 s panes: almost every
    tile lies inside one pane (no timestamps staged), the few around each boundary take the per-row pane path."""
    batches = host_stream(4 << 20, groups=100_000, rows_per_ms=512, seed=7)
    batches.append(sentinel(int(batches[-1].ts[-1]) + 5000))
    st = run_variants_large(batches, 1000, max_rows_per_launch=1 << 20)
    for name, s in st.items():
        assert s["groups"] == 100_001 and s["deferred_rows"] == 0 and s["agg_launches"] >= 4, name
        assert s["fast_tiles"] > 0.99 * (4 << 20) / TILE, name


def test_colliding_keys_under_every_switch():
    """Keys with equal 32-bit hashes and clusters that share their home slot (tests/test_gpu_kernel_edges.py), on the hinted
    table and on the small table with private pane copies: parked rows, retry rounds and in-place chains next to paired probes."""
    pairs, clusters = _collision_keys()
    keys = sorted({k for p in pairs for k in p} | {k for c in clusters for k in c})
    rng = np.random.default_rng(64)
    batches = []
    for b in range(24):
        n = 8 * TILE
        k = rng.integers(0, len(keys), n)
        batches.append(columns_to_batch(T0 + b * 250 + rng.integers(0, 250, n), _adversarial_values(rng, k, b), [keys[j] for j in k]))
    batches.append(sentinel(T0 + 10_000))
    want = run_oracle_batches(batches, 1000)
    for eg in (0, 16):
        st = run_variants(batches, 1000, want=want, expected_groups=eg)
        for name, s in st.items():
            assert s["groups"] == len(keys) + 1 and s["deferred_rows"] == 0 and s["fast_tiles"] > 0, (eg, name)


def test_insert_storm_under_every_switch():
    """8 Mi rows in one launch, every key new and probed by several CTAs while it is inserted (the torn-read case of the paired
    probe: a slot published between its two halves): every key is interned exactly once under every switch."""
    n_rows = 8 * 1024 * 1024 - (8 * 1024 * 1024) % (16 * TILE)
    batches, n_keys = _storm_batches(n_rows, 1 << 20)
    batches.append(sentinel(T0 + 10_000_000))
    st = run_variants_large(batches, 60_000, expected_groups=n_keys)
    for name, s in st.items():
        assert s["groups"] == n_keys + 1 and s["fast_tiles"] > 0.9 * n_rows / TILE, name


def test_late_batches_and_special_values_under_every_switch():
    """Batches that re-open emitted windows (tiles of a late pane: every row on the per-row path with the tile's pane), tiles that
    span panes (the only ones whose timestamps are staged), +-0.0 / NaN / +-inf and keys longer than 16 B."""
    rng = np.random.default_rng(128)
    rows = random_stream(rng, 40, 3000, 500, span_ms=300, special_vals=True, late_every=7, late_shift_ms=2500)
    # +-1e308 would make the average depend on the order of the additions (1e308 + 1e308 overflows, 1e308 - 1e308 does not)
    rows = [[(t, math.copysign(113.0, v) if abs(v) == 1e308 else v, k) for t, v, k in b] for b in rows]
    batches = [rows_to_batch(r) for r in rows]
    batches.append(sentinel(T0 + 40 * 300 + 10_000))
    st = run_variants(batches, 1000, per_batch_poll=True)
    for name, s in st.items():
        assert s["late_batches"] > 0 and s["fast_tiles"] > 0, name
