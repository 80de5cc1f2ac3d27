"""Ungrouped windows `.window([], aggs, ..)` at launch scale (run on an H100 with -m gpu): streams of 70-140 M rows, so that
launches fill to the default 64 Mi rows, k_aggregate_ungrouped runs 1056-CTA grids over contiguous tile chunks, chunk boundaries
fall inside panes, CTAs see pane changes inside their chunk (the block-wide uacc_flush) and, at 4 rows/ms, many tiles span panes
(the per-row path) and one run closes more than 4096 windows.

Values are k / 1024 with integer |k| <= 2^20 and about 2 % NULL, so every sum is exact in f64 whatever the summation order:
count, min, max, sum and avg are compared bit for bit with the oracle's Partial -> Final chain, and every emitted window with an
independent NumPy recomputation from per-pane integer sums, counts and plain min / max.  Every batch is shorter than a pane, so
a batch closes at most one window and each emitted row is exactly one window."""
import numpy as np
import pyarrow as pa
import pytest

from oracle import Batch, OracleUngrouped
from tests.helpers import SUM_AGGS, agg_rows, assert_rows_exact, rows_to_batch, same_f64, to_record_batch

pytestmark = pytest.mark.gpu
T0 = 1_700_000_000_000
LAUNCH_ROWS = 64 << 20                              # default max_rows_per_launch
CHUNK = 1 << 22                                     # rows generated at a time


def _schema():
    from denormalized_b200 import canonical_schema
    return pa.schema([pa.field("reading", pa.float64()), canonical_schema().field(3)])


def _bitmap(valid):
    return None if valid is None else np.packbits(np.concatenate([valid, np.zeros(8, bool)]), bitorder="little")


class Piece:
    """One pushed batch: the Arrow record batch (built from the numpy buffers, no copies) and the oracle's view of it."""
    _zero_off = np.zeros(CHUNK + 1, np.int32)
    _no_bytes = np.zeros(16, np.uint8)

    def __init__(self, ts, val, val_valid, ts_valid=None):
        self.ts, self.val, self.vbm, self.tbm = ts, val, _bitmap(val_valid), _bitmap(ts_valid)

    def record_batch(self, schema):
        n = len(self.ts)
        meta_type = schema.field(1).type
        buf = (lambda bm: None if bm is None else pa.py_buffer(bm))
        barrier = pa.Array.from_buffers(pa.utf8(), n, [None, pa.py_buffer(self._zero_off[:n + 1]), pa.py_buffer(self._no_bytes)])
        ts = pa.Array.from_buffers(pa.timestamp("ms"), n, [buf(self.tbm), pa.py_buffer(self.ts)])
        val = pa.Array.from_buffers(pa.float64(), n, [buf(self.vbm), pa.py_buffer(self.val)])
        meta = pa.StructArray.from_arrays([barrier, ts], fields=list(meta_type))
        return pa.RecordBatch.from_arrays([val, meta], schema=schema)

    def oracle(self):
        n = len(self.ts)
        return Batch(ts=self.ts, val=self.val, key_off=self._zero_off[:n + 1], key_bytes=self._no_bytes, ts_valid=self.tbm,
                     val_valid=self.vbm)


class PaneStats:
    """Per-pane count, integer sum of k, min and max of the valid rows (1 s panes), accumulated chunk by chunk."""

    def __init__(self, p0, n):
        self.p0 = p0
        self.cnt = np.zeros(n, np.int64); self.sum = np.zeros(n, np.int64)
        self.mn = np.full(n, np.inf); self.mx = np.full(n, -np.inf)

    def add(self, ts, k, valid):
        ts, k = ts[valid], k[valid]
        if not len(ts):
            return
        p = ts // 1000 - self.p0
        assert np.all(np.diff(p) >= 0)
        starts = np.concatenate([[0], np.nonzero(np.diff(p))[0] + 1])
        idx = p[starts]
        self.cnt[idx] += np.diff(np.concatenate([starts, [len(p)]]))
        self.sum[idx] += np.add.reduceat(k, starts)
        v = k / 1024.0
        self.mn[idx] = np.minimum(self.mn[idx], np.minimum.reduceat(v, starts))
        self.mx[idx] = np.maximum(self.mx[idx], np.maximum.reduceat(v, starts))

    def check(self, row):
        ws, we = row[0], row[1]
        a, b = max(ws // 1000 - self.p0, 0), we // 1000 - self.p0          # panes before the stream's first are empty
        c = int(self.cnt[a:b].sum())
        assert row[3] == c, f"count {row}: {c}"
        if c == 0:
            assert row[4] is None and row[8] is None, row
            return
        s = int(self.sum[a:b].sum()) / 1024.0
        assert same_f64(row[8], s) and same_f64(row[6], s / c), f"sum / avg {row}: {s}"
        assert row[4] == float(self.mn[a:b].min()) and row[5] == float(self.mx[a:b].max()), f"min / max {row}"


VARIANTS = {
    # rows per ms, window, slide, rows, rows per batch (never a multiple of the 416-row tile)
    "cfg2_rate_tumbling_1s": (10_000, 1000, 0, 2 * LAUNCH_ROWS + 5_000_000, 99_999),
    "100_per_ms_sliding_10s": (100, 10_000, 1000, 2 * LAUNCH_ROWS + 5_000_000, 77_777),
    "4_per_ms_sliding_64s": (4, 64_000, 1000, LAUNCH_ROWS + 3_000_000, 3_001),
}


@pytest.mark.parametrize("name", list(VARIANTS))
def test_ungrouped_launch_scale(name):
    from denormalized_b200 import GpuStreamingWindow
    rate, L, S, n_rows, batch = VARIANTS[name]
    schema = _schema()
    w = GpuStreamingWindow(schema, None, SUM_AGGS, L, S, None)
    o = OracleUngrouped(L, S)
    rng = np.random.default_rng(rate + L + S)
    panes = PaneStats(T0 // 1000, n_rows // rate // 1000 + 2)
    got, want, pushes = [], [], 0
    null_ts_at = n_rows // 2 // CHUNK * CHUNK if rate == 10_000 else -1      # one batch with NULL timestamps inside a launch

    def push(piece):
        nonlocal pushes
        w.push(piece.record_batch(schema))
        o.push(piece.oracle()); want.extend(o.results(with_sum=True))
        pushes += 1
        if pushes % 64 == 0:
            got.extend(agg_rows(w.poll_ready()))
    for c0 in range(0, n_rows, CHUNK):
        n = min(CHUNK, n_rows - c0)
        ts = T0 + (np.arange(c0, c0 + n, dtype=np.int64) // rate)
        k = rng.integers(-2 ** 20, 2 ** 20 + 1, n)
        val = k / 1024.0
        valid = rng.random(n) >= 0.02
        tvalid = np.ones(n, bool)
        if c0 == null_ts_at:
            tvalid[:batch] = rng.random(batch) >= 0.1
        panes.add(ts[tvalid], k[tvalid], valid[tvalid])
        for i in range(0, n, batch):                   # the last batch of a chunk is shorter
            j = min(n, i + batch)
            tv = tvalid[i:j]
            push(Piece(ts[i:j], val[i:j], valid[i:j], None if tv.all() else tv))
        del ts, k, val, valid, tvalid
    if rate == 10_000:                                  # a late batch: 5 s behind, its windows were finalized long ago
        lt = T0 + n_rows // rate - 5000 + np.arange(5000, dtype=np.int64) // 1000
        lk = rng.integers(-2 ** 20, 2 ** 20 + 1, 5000)
        push(Piece(lt, lk / 1024.0, np.ones(5000, bool)))
    got.extend(agg_rows(w.poll()))
    st = w.stats()
    w.close()
    o.close()
    assert st["rows_in"] >= n_rows > LAUNCH_ROWS and st["agg_launches"] >= n_rows // LAUNCH_ROWS + 1 >= 2
    n_panes = n_rows // rate // 1000
    assert len(want) >= n_panes - L // 1000 - 3, (len(want), n_panes)
    assert_rows_exact(got, want)
    for r in got:
        panes.check(r)


def test_one_run_closing_more_than_4096_windows():
    """A sparse stream: 8192 rows one second apart, then one row after them.  The second poll's run closes 8192 windows at once,
    more than the operator stages at creation; it grows the staging instead of failing.  Two more rows let the Final stage emit
    the frame those windows were merged into.  The grouped path on the same stream."""
    from denormalized_b200 import GpuStreamingWindow, canonical_schema
    from oracle import OracleWindow
    n = 8192
    a = rows_to_batch([(T0 + 1000 * i + 7, float(i % 97) - 48.0, b"k%d" % (i % 3)) for i in range(n)])
    later = [rows_to_batch([(T0 + 1000 * (n + d) + 7, 1.0, b"k0")]) for d in (0, 5, 10)]
    for key in (None, "sensor_name"):
        w = GpuStreamingWindow(canonical_schema(), key, SUM_AGGS, 1000, 0, None)
        o = OracleUngrouped(1000) if key is None else OracleWindow(1000)
        got, want = [], []
        for i, x in enumerate([a] + later):
            w.push(to_record_batch(x))
            got += agg_rows(w.poll(), seq=i)
            o.push(x); want += o.results(with_sum=True)
        w.close()
        assert len(want) >= (2 if key is None else n)
        assert_rows_exact(got, want, check_seq=True)
