"""Utf8 against Int64 group keys on cfg 2's stream (1e9 rows, 100 K groups, tumbling 1 s), device resident.

Both streams come from dnz_synth_generate with the same key ids: "sensor_<id>" (Utf8) and the id itself (Int64).  Runs of the two
alternate in one process.  Per run: k_aggregate time from DNZ_FLAG_KERNEL_TIMING (ms per launch and per 64 Mi rows), rows per
second over the whole step (CUDA events around it), and the roofline fraction of k_aggregate from the key type's algorithmic bytes
(Utf8: 20 B per row + key bytes; Int64: 24 B per row).  The outputs of the two key types are compared under the key map
sensor_<id> <-> id (count / min / max bit-exact, avg within 1e-9); those outputs come from one more, untimed run per type.

    python profiles/int_keys_bench.py [--rows N] [--runs R] [--warmup W]
"""
import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

T0 = 1_700_000_000_000
BATCH_ROWS = 65536
GROUPS, ROWS_PER_MS, WINDOW_MS = 100_000, 10_000, 1000
AGGS = [("count", "reading", "count"), ("min", "reading", "min"), ("max", "reading", "max"), ("avg", "reading", "average")]


def card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=20).stdout.strip()
    except Exception as e:          # noqa: BLE001 -- reported, not fatal
        q = f"nvidia-smi unavailable ({e})"
    return name, q


def peak_gbs():
    try:
        with open(os.path.join(ROOT, "MEASURED_PEAKS.json")) as f:
            return float(json.load(f)["hbm_gbs"]), "measured (MEASURED_PEAKS.json)"
    except Exception:
        return 3350.0, "data sheet (H100 SXM HBM3 3.35 TB/s)"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1_000_000_000)
    ap.add_argument("--runs", type=int, default=3, help="timed runs per key type (alternated)")
    ap.add_argument("--warmup", type=int, default=1)
    args = ap.parse_args()

    import numpy as np
    import pyarrow as pa
    import pyarrow.compute as pc
    import torch
    import denormalized_b200 as d
    from tests.helpers import assert_tables_equal, concat_arrays, result_table

    torch.cuda.set_device(0)
    stream = torch.cuda.Stream()
    rows = args.rows
    last_ts = T0 + (rows - 1) // ROWS_PER_MS
    close = (last_ts // 1000 + 1) * 1000 + 2 * WINDOW_MS
    dev = {"utf8": d.DeviceBatches(rows, BATCH_ROWS, groups=GROUPS, rows_per_ms=ROWS_PER_MS),
           "int64": d.DeviceBatches(rows, BATCH_ROWS, groups=GROUPS, rows_per_ms=ROWS_PER_MS, int_keys=True)}
    meta = d.canonical_schema().field(3)
    schemas = {"utf8": d.canonical_schema(), "int64": pa.schema([pa.field("id", pa.int64()), pa.field("reading", pa.float64()), meta])}
    keycol = {"utf8": "sensor_name", "int64": "id"}

    def step(kind, capture=None):
        w = d.GpuStreamingWindow(schemas[kind], keycol[kind], AGGS, WINDOW_MS, 0, None, flags=d.capi.FLAG_KERNEL_TIMING,
                                 expected_groups=GROUPS, cuda_stream=stream.cuda_stream)
        b = dev[kind]

        def take(r):
            if r.n_rows and capture is not None:
                capture.append(w.fetch_device_result(r, max_keys=0))
            return r.n_rows
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        for g0 in range(0, b.n_batches, 1024):
            n = min(1024, b.n_batches - g0)
            w.push_device(array=C.cast(C.byref(b.array, g0 * C.sizeof(d.capi.DeviceBatchC)), C.POINTER(d.capi.DeviceBatchC)), n=n)
            while take(w.poll_device_ready()):
                pass
        w.flush(close)
        while take(w.poll_device()):
            pass
        e1.record(stream)
        e1.synchronize()
        st = w.stats()
        w.close()
        return e0.elapsed_time(e1), st

    for _ in range(args.warmup):
        for kind in dev:
            step(kind)
    res = {k: [] for k in dev}
    outs = {}
    for i in range(args.runs):
        for kind in (("utf8", "int64") if i % 2 == 0 else ("int64", "utf8")):
            ms, st = step(kind)
            res[kind].append((ms, st))
            print(f"run {i} {kind}: step {ms:.1f} ms, k_aggregate {st['agg_kernel_ms']:.2f} ms over {st['agg_launches']} launches",
                  file=sys.stderr, flush=True)
    for kind in dev:                 # one more, untimed run per type whose output is copied to the host
        outs[kind] = []
        step(kind, outs[kind])

    # the two runs' outputs under the key map sensor_<id> <-> id
    parts = []
    for p in outs["int64"]:
        s = pc.binary_join_element_wise(pa.scalar(b"sensor_"), pa.array(p["key_values"]).cast(pa.string()).cast(pa.binary()), b"")
        q = dict(p)
        q["key_off"] = np.frombuffer(s.buffers()[1], np.int32, len(p["count"]) + 1).copy()
        q["key_bytes"] = np.frombuffer(s.buffers()[2], np.uint8, int(q["key_off"][-1])).copy()
        parts.append(q)
    got, want = result_table(concat_arrays(parts), "g"), result_table(concat_arrays(outs["utf8"]), "w")
    matched = assert_tables_equal(got, want)

    peak, peak_src = peak_gbs()
    name, power = card()
    summary = {"card": name, "power_limit_and_max_sm_clock": power, "rows": rows, "groups": GROUPS, "runs": args.runs,
               "outputs_agree": matched == want.num_rows, "rows_compared": int(matched), "peak_gbs": peak, "peak_source": peak_src}
    for kind, rs in res.items():
        launch_ms = [st["agg_kernel_ms"] / max(st["agg_launches"], 1) for _, st in rs]
        per64 = [st["agg_kernel_ms"] * (64 << 20) / rows for _, st in rs]
        grs = [rows / (ms * 1e-3) / 1e9 for ms, _ in rs]
        frac = [st["agg_algorithmic_bytes"] / (st["agg_kernel_ms"] * 1e-3) / 1e9 / peak for _, st in rs]
        summary[kind] = {"k_aggregate_avg_launch_ms": [round(x, 4) for x in launch_ms],
                         "k_aggregate_ms_per_64Mi_rows": [round(x, 4) for x in per64],
                         "median_ms_per_64Mi_rows": round(statistics.median(per64), 4),
                         "grows_per_s_per_step": [round(x, 2) for x in grs], "median_grows_per_s": round(statistics.median(grs), 2),
                         "roofline_frac": [round(x, 4) for x in frac],
                         "algorithmic_bytes_per_row": rs[0][1]["agg_algorithmic_bytes"] / rows,
                         "groups": rs[0][1]["groups"], "deferred_rows": rs[0][1]["deferred_rows"]}
    for b in dev.values():
        b.free()
    print(json.dumps(summary))


if __name__ == "__main__":
    main()
