"""Oracle comparison at BASELINE-config shapes on LARGE samples (VERDICT r1, "next round" item 1a): 100-200 M rows of the
cfg 2 / cfg 3 / cfg 4 / cfg 5 streams through the C ABI (device-resident input, the same generator on both sides) against the
multi-threaded CPU oracle, row by row: a sort-free hash join on (window_start, key), count/min/max bit-exact, avg within 1e-9
relative.  These reach what the small tests cannot: 100 K - 2 M live groups, dictionary sectors that miss L2, long-key arena growth
at scale, dozens of 64 Mi-row launches through the three-slot pipeline."""
import ctypes as C
import os

import numpy as np
import pytest

from tests.helpers import (assert_tables_equal, concat_arrays, gpu_window, host_stream, oracle_mt_arrays, result_table, rows_to_batch)

pytestmark = pytest.mark.gpu
T0 = 1_700_000_000_000
BATCH = 65536


def _gpu_arrays(n_rows, L, S, filt, groups, rpm, uuid, close_step_ms, max_rows_per_launch=0):
    from denormalized_b200 import DeviceBatches, capi
    dev = DeviceBatches(n_rows, BATCH, groups=groups, rows_per_ms=rpm, uuid_keys=uuid)
    w = gpu_window(L, S, filt, expected_groups=groups, max_rows_per_launch=max_rows_per_launch)
    parts = []

    def take(r):
        if r.n_rows:
            parts.append(w.fetch_device_result(r, max_keys=0))
        return r.n_rows
    group = 1024
    for g0 in range(0, dev.n_batches, group):
        k = min(group, dev.n_batches - g0)
        w.push_device(array=C.cast(C.byref(dev.array, g0 * C.sizeof(capi.DeviceBatchC)), C.POINTER(capi.DeviceBatchC)), n=k)
        while take(w.poll_device_ready()):
            pass
    last = T0 + (n_rows - 1) // rpm
    wm, close = (last // 1000) * 1000, (last // 1000 + 1) * 1000 + 2 * L
    while wm < close:                      # close the remaining windows a few at a time (one poll stays below 2 GiB of key bytes)
        wm = min(wm + close_step_ms, close)
        w.flush(wm)
        while take(w.poll_device()):
            pass
    st = w.stats()
    w.close(); dev.free()
    return parts, st, close


def _check(n_rows, L, S, filt, groups, rpm, uuid=False, close_step_ms=64_000):
    parts, st, close = _gpu_arrays(n_rows, L, S, filt, groups, rpm, uuid, close_step_ms)
    hb = host_stream(n_rows, groups=groups, rows_per_ms=rpm, uuid_keys=uuid)
    hb.append(rows_to_batch([(close, 1.0, b"sentinel")]))
    want = oracle_mt_arrays(hb, L, S, filt)
    del hb
    # compare window by window range so that no concatenation exceeds the 2 GiB Utf8 limit
    got_n = sum(len(p["count"]) for p in parts)
    assert got_n == len(want["count"]), f"row count {got_n} != {len(want['count'])}"
    wt = result_table(want, "w")
    import pyarrow.compute as pc
    # every key of the stream ends up in a closed window: a key interned twice by racing inserts would show up as extra groups
    assert st["groups"] == pc.count_distinct(wt["key"]).as_py(), "groups != distinct keys"
    matched = 0
    # pieces of ~8 M GPU rows
    piece, acc = [], 0
    for p in parts + [None]:
        if p is not None:
            piece.append(p); acc += len(p["count"])
        if piece and (p is None or acc >= 8_000_000):
            g = concat_arrays(piece)
            lo, hi = int(g["window_start"].min()), int(g["window_start"].max())
            sub = wt.filter(pc.and_(pc.greater_equal(wt["ws"], lo), pc.less_equal(wt["ws"], hi)))
            gt = result_table(g, "g")
            # a window range may be split across pieces: restrict the oracle side to the (window, key) pairs of this piece by joining
            j = gt.join(sub, keys=["ws", "key"], join_type="inner")
            assert j.num_rows == gt.num_rows, f"{gt.num_rows - j.num_rows} emitted rows have no oracle counterpart"
            sub2 = sub.join(gt.select(["ws", "key"]), keys=["ws", "key"], join_type="inner")
            matched += assert_tables_equal(gt, sub2)
            piece, acc = [], 0
    assert matched == got_n
    return st, got_n


def test_cfg2_200m_rows_100k_groups_tumbling():
    st, n = _check(200_000_000, 1000, 0, None, 100_000, 10_000)
    assert n == 20 * 100_000 and st["agg_launches"] >= 3 and st["deferred_rows"] == 0


def test_cfg4_200m_rows_filter_max_gt_113():
    st, n = _check(200_000_000, 1000, 0, ("max", ">", 113.0), 100_000, 10_000)
    assert 0.80 * 2_000_000 < n < 0.85 * 2_000_000          # P(pass) = 1 - (113/115)^100 = 0.826


def test_cfg3_100m_rows_1m_groups_sliding_10s_1s():
    st, n = _check(100_000_000, 10_000, 1000, None, 1_000_000, 10_000)
    assert n > 15_000_000


def test_cfg5_50m_rows_2m_uuid_keys_sliding_60s_5s():
    st, n = _check(50_000_000, 60_000, 5000, None, 2_000_000, 8_000, uuid=True, close_step_ms=5_000)
    assert n > 10_000_000
