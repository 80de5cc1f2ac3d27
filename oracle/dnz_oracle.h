/*
 * dnz_oracle.h -- CPU oracle for the windowed grouped aggregate + post-aggregate filter.
 *
 * TEST INFRASTRUCTURE ONLY.  Nothing under oracle/ is part of the product: only tests/,
 * __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may load it,
 * and there only as the checker (or the timed CPU baseline), never as the thing shipped.
 *
 * PARITY UNPINNED: the reference (Rust, DataFusion-42 fork) cannot be built in this image
 * (no cargo/rustc, no vendored crates) and holds no test, fixture or golden vector for this
 * path (SURVEY.md §4, §8c).  This file is a restatement of the reference algorithm, function by
 * function, cross-checked against pyarrow/Acero group_by on small inputs and against the one
 * adjacent known-answer in the reference (crates/core/src/utils/serialization.rs:535-557:
 * avg of 56 x 56.0 == 56.0, avg state = [count, sum]).
 *
 * Reference files restated (paths relative to /root/reference/crates/core/src/physical_plan):
 *   continuous/grouped_window_agg_stream.rs:326-349  per-batch order of operations
 *   continuous/grouped_window_agg_stream.rs:276-313  ensure_window_frames_for_ranges
 *   continuous/grouped_window_agg_stream.rs:548-605  GroupedAggWindowFrame::push (two filter copies)
 *   continuous/grouped_window_agg_stream.rs:501-537  group_aggregate_batch (intern + 4 update_batch passes)
 *   continuous/grouped_window_agg_stream.rs:255-266  process_watermark
 *   continuous/grouped_window_agg_stream.rs:220-253  trigger_windows
 *   continuous/grouped_window_agg_stream.rs:609-629  evaluate
 *   continuous/streaming_window.rs:1053-1094         get_windows_for_watermark / snap_to_window_start
 *   utils/time.rs:31-57                              RecordBatchWatermark::try_from
 *   continuous/mod.rs:64-89                          add_window_columns_to_record_batch
 * Third-party arithmetic restated from its published algorithm (NOT under /root/reference):
 *   datafusion 42.0.0 (git probably-nothing-labs/arrow-datafusion @ d812edc, Cargo.toml:31):
 *     GroupValuesByes<i32>::intern (first-seen dense group ids, NULL key is its own group),
 *     CountGroupsAccumulator, PrimitiveGroupsAccumulator<Float64> min/max
 *     (start f64::MAX / f64::MIN, `if *cur > new` / `if *cur < new`) and sum (start +0.0, += v in row order), AvgGroupsAccumulator
 *     (sum += v in row order; u64 count; sum / count), NullState, FilterExec.
 *   arrow-ord 53.3.0 cmp::{gt_eq,lt,gt,...}: floats compare with IEEE-754 totalOrder.
 */
#ifndef DNZ_ORACLE_H
#define DNZ_ORACLE_H
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

enum { ORC_OP_GT = 0, ORC_OP_GTE = 1, ORC_OP_LT = 2, ORC_OP_LTE = 3, ORC_OP_EQ = 4, ORC_OP_NEQ = 5 };
enum { ORC_COL_COUNT = 0, ORC_COL_MIN = 1, ORC_COL_MAX = 2, ORC_COL_AVG = 3, ORC_COL_SUM = 4 };

typedef struct {
  int64_t window_ms;     /* window length (Duration, ms resolution)                       */
  int64_t slide_ms;      /* 0 = tumbling (slide: None)                                    */
  int32_t has_filter;    /* post-aggregate FilterExec: <col> <op> <literal>                */
  int32_t filter_col;    /* ORC_COL_*                                                      */
  int32_t filter_op;     /* ORC_OP_*                                                       */
  int32_t reserved;
  double  filter_lit;    /* literal, already coerced to Float64 (lit(113) -> 113.0)        */
} orc_config;

/* One input RecordBatch, canonical sensor schema (kafka_config.rs:186-214).  Validity bitmaps are
 * Arrow LSB-first, NULL pointer = no nulls.  occurred_at / barrier_* are unused by the aggregation
 * but ARE copied by the reference's two filter_record_batch calls per window; they may be NULL, in
 * which case the copies of those columns are skipped. */
typedef struct {
  int64_t n;
  const int64_t* ts;        const uint8_t* ts_valid;    /* _streaming_internal_metadata.canonical_timestamp */
  const double*  val;       const uint8_t* val_valid;   /* reading     */
  const int32_t* key_off;   const uint8_t* key_bytes;   const uint8_t* key_valid; /* sensor_name */
  const int64_t* occurred_at;
  const int32_t* barrier_off; const uint8_t* barrier_bytes;
} orc_batch;

typedef struct orc_window orc_window;

/* Emitted rows accumulate in an internal result set until orc_clear_results. */
typedef struct {
  int64_t n;
  const int32_t* key_off;  const uint8_t* key_bytes; const uint8_t* key_isnull;  /* byte per row */
  const int64_t* count;
  const double* min; const double* max; const double* avg;
  const uint8_t* agg_isnull;          /* byte per row: min/max/avg are null (group saw no non-null reading) */
  const int64_t* window_start_ms; const int64_t* window_end_ms;
  const int64_t* emit_seq;            /* index of the push() call that emitted the row */
  const double* sum;                  /* sum(reading): +0.0 plus every non-null value in row order (null when agg_isnull) */
} orc_result;

orc_window* orc_create(const orc_config* cfg);
void orc_destroy(orc_window* w);
/* Returns number of rows emitted by this call (after the filter), or <0 on error
 * (-1: all-null timestamp column -- the reference panics; -2: unsupported geometry, e.g. window < 1 s
 * divides by zero in snap_to_window_start; -3: timestamp before epoch+window). */
int64_t orc_push(orc_window* w, const orc_batch* b);
void orc_get_results(orc_window* w, orc_result* out);
void orc_clear_results(orc_window* w);
int64_t orc_open_frames(const orc_window* w);
int64_t orc_watermark(const orc_window* w);   /* INT64_MIN when unset */
const char* orc_last_error(const orc_window* w);

/* Multi-threaded hash-partition mode = the timed CPU baseline ("CPU restatement of the reference"):
 * mirrors RepartitionExec(Hash(group keys), P) -> P independent GroupedWindowAggStreams
 * (physical_optimizer/coalesce_before_streaming_window_aggregate.rs:63-73, streaming_window.rs:470-481).
 * Processes `nb` batches with `threads` threads; results of all partitions are concatenated into
 * partition 0's result set view via orc_mt_get_results.  Watermark: the shared-Mutex watermark of the
 * reference (streaming_window.rs:210) is made deterministic: every partition observes the watermark of
 * the full batch and triggers after each batch. */
typedef struct orc_mt orc_mt;
orc_mt* orc_mt_create(const orc_config* cfg, int partitions);
void orc_mt_destroy(orc_mt* m);
int64_t orc_mt_push_many(orc_mt* m, const orc_batch* batches, int64_t nb);
int64_t orc_mt_num_results(const orc_mt* m);
void orc_mt_get_results(orc_mt* m, int partition, orc_result* out);
void orc_mt_clear_results(orc_mt* m);

/* Synthetic sensor generator (SURVEY.md §8d): counter-based, identical to the device generator.
 * Fills rows [row0, row0+n) of the global stream.  key_off must hold n+1 entries, key_bytes must hold
 * at least n*max_key_len bytes; returns bytes written.  uuid_keys != 0 -> 36-char UUID-shaped keys.
 * key id = (r>>11) % groups * key_mul + key_add (key_mul=world, key_add=rank shards the key space by rank). */
int64_t orc_synth_fill(int64_t row0, int64_t n, uint64_t seed, int64_t groups, int64_t rows_per_ms,
                       int64_t t0_ms, int32_t uuid_keys, int64_t key_mul, int64_t key_add,
                       int64_t* ts, double* val, int32_t* key_off, uint8_t* key_bytes);

/* Ungrouped windows `.window([], aggs, ..)`: one partition of the Partial -> Final chain the planner builds
 * (planner/streaming_window.rs:133-153; streaming_window.rs:640-828, :882-1051).  Results use orc_result with every key NULL. */
typedef struct orc_uwindow orc_uwindow;
orc_uwindow* orc_u_create(const orc_config* cfg);
void orc_u_destroy(orc_uwindow* w);
int64_t orc_u_push(orc_uwindow* w, const orc_batch* b);
void orc_u_get_results(orc_uwindow* w, orc_result* out);
void orc_u_clear_results(orc_uwindow* w);
const char* orc_u_last_error(const orc_uwindow* w);

/* Canonical event time from a raw column: array_to_timestamp_array (physical_plan/utils/time.rs:59-94).
 * unit: 1 Int64Millis, 2 Int64Seconds, 3 StringIso8601(fmt).  Returns 0, or 1 + the index of the first unparsable row. */
int64_t orc_ts_convert(int32_t unit, int64_t n, const int64_t* ints, const int32_t* off, const uint8_t* bytes, const char* fmt, int64_t* out);

#ifdef __cplusplus
}
#endif
#endif
