/*
 * dnz_gpu.h -- C ABI of the H100 windowed grouped aggregate (+ post-aggregate filter).
 *
 * This is the drop-in boundary for Denormalized's streaming-window hot path (SURVEY.md §8b).  Every entry
 * point names the reference interface it replaces (paths relative to /root/reference/crates/core/src).
 * Plain C: opaque handles, plain pointers and sizes, Arrow C Data Interface structs for RecordBatches.
 * No C++ exception crosses the boundary; every call returns a status (0 = ok, <0 = error) and the
 * message is available from dnz_window_last_error().  There is NO CPU fallback: if no CUDA device or an
 * unsupported plan shape is given the call fails.
 *
 * Threading (mirrors `Stream::poll_next(&mut self)`): a handle is externally synchronised (one caller at
 * a time) but not thread-affine; distinct handles may be used concurrently.
 */
#ifndef DNZ_GPU_H
#define DNZ_GPU_H
#include <stdint.h>
#include "arrow_c_data.h"

#ifdef __cplusplus
extern "C" {
#endif

#define DNZ_ABI_VERSION 2
#define DNZ_NO_KEY (-1)           /* key_column: no group key -- `.window([], aggs, ..)`, the ungrouped window (SURVEY.md §8 f2) */

/* status codes */
#define DNZ_OK 0
#define DNZ_ERR_INVALID (-1)      /* bad argument / schema mismatch                                      */
#define DNZ_ERR_UNSUPPORTED (-2)  /* plan shape the GPU operator does not implement (no CPU fallback)     */
#define DNZ_ERR_CUDA (-3)         /* CUDA runtime error (sticky per handle)                               */
#define DNZ_ERR_DATA (-4)         /* input the reference would panic on (all-null timestamps, ts<epoch)   */
#define DNZ_ERR_NOMEM (-5)

/* AggregateFunctionExpr kinds accepted in DataStream::window(.., aggr_expr, ..) (datastream.rs:178-196) */
enum { DNZ_AGG_COUNT = 0, DNZ_AGG_MIN = 1, DNZ_AGG_MAX = 2, DNZ_AGG_AVG = 3, DNZ_AGG_SUM = 4 };
/* BinaryExpr operators of the post-aggregate DataStream::filter(predicate) (datastream.rs:94-105) */
enum { DNZ_OP_GT = 0, DNZ_OP_GTE = 1, DNZ_OP_LT = 2, DNZ_OP_LTE = 3, DNZ_OP_EQ = 4, DNZ_OP_NEQ = 5 };

enum { DNZ_TS_CANONICAL = 0, DNZ_TS_INT64_MILLIS = 1, DNZ_TS_INT64_SECONDS = 2, DNZ_TS_STRING_ISO8601 = 3 };   /* TimestampUnit (kafka_config.rs) */

#define DNZ_FLAG_KERNEL_TIMING 1u  /* record CUDA events around every aggregate-kernel launch (dnz_stats) */
#define DNZ_FLAG_FORCE_GENERIC 2u  /* testing: disable the TMA-staged fast path                           */
#define DNZ_FLAG_NO_HINTS 4u        /* experiments: disable the per-group min/max reduction filter                 */
#define DNZ_FLAG_NO_PRIVATE 16u     /* experiments: no per-CTA private pane copies for low-cardinality streams        */
#define DNZ_FLAG_NO_QUEUE 8u        /* experiments: colliding probes loop in place instead of using the retry queue */
#define DNZ_FLAG_SYNCHRONOUS 32u    /* testing / A-B: wait for every aggregate launch before emitting (no speculative pipeline) */
#define DNZ_FLAG_SCALAR_PROBE 64u   /* experiments: every row loads both halves of its dictionary slot (no lane-paired probe) */
#define DNZ_FLAG_STAGE_TS 128u      /* experiments: stage the timestamps of tiles that lie inside one pane too              */

typedef struct {
  int32_t kind;          /* DNZ_AGG_*                                            */
  int32_t arg_column;    /* top-level input column index of the Float64 argument */
  const char* alias;     /* output column name (count/min/max/average ...)       */
} dnz_agg;

/* Arguments of StreamingWindowExec::try_new (physical_plan/continuous/streaming_window.rs:221-251):
 * group_by -> key_column, aggr_expr -> aggs, window_type -> window_ms/slide_ms; plus the FilterExec that
 * the planner stacks directly above the window (SURVEY.md §3.2) as an optional fused predicate. */
typedef struct {
  uint32_t abi_version;      /* DNZ_ABI_VERSION                                                     */
  int32_t device;            /* CUDA device ordinal                                                 */
  int32_t key_column;        /* top-level index of the group-key column (one plain column,
                                planner/streaming_window.rs:36-66) of Arrow format "u" (Utf8), "l" (Int64),
                                "i" (Int32), "L" (UInt64) or "I" (UInt32) -- integer keys group as DataFusion's
                                GroupValuesPrimitive does: one group per distinct value, NULL a group of its own; the
                                emitted key column has the input's type and nullability (a Utf8 key column
                                is emitted nullable) -- or DNZ_NO_KEY: the ungrouped window --
                                one partition of the Partial -> Final chain the planner builds for an empty
                                group_by (planner/streaming_window.rs:133-153; WindowAggStream
                                streaming_window.rs:640-828 on the device, FullWindowAggStream :882-1051 on
                                the host over one 40 B state per window).  Output: aggregates, window_start_time,
                                window_end_time; a window is emitted once a window that starts after its end has
                                closed (the reference's Final stage), late partial results are dropped.  */
  int32_t n_aggs;
  const dnz_agg* aggs;
  int64_t window_ms;         /* PhysicalStreamingWindowType::{Tumbling(len) | Sliding(len, slide)}  */
  int64_t slide_ms;          /* 0 = tumbling                                                        */
  int32_t has_filter;        /* FilterExec: aggs[filter_agg] <filter_op> filter_literal             */
  int32_t filter_agg;
  int32_t filter_op;
  uint32_t flags;
  double filter_literal;     /* literal already coerced to Float64 (lit(113) -> 113.0)              */
  int64_t expected_groups;   /* capacity hint (0 = default); tables grow on demand                  */
  int64_t max_rows_per_launch; /* rows aggregated per kernel launch (0 = default 64 Mi)             */
  void* cuda_stream;         /* optional caller-owned cudaStream_t for all work (NULL = own stream) */
  /* Input-contract producer (SURVEY.md §8 f1): where the event time comes from.  DNZ_TS_CANONICAL (0, default): the batch carries
   * `_streaming_internal_metadata.canonical_timestamp` as the reference's Kafka reader attaches it
   * (datasource/kafka/kafka_stream_read.rs:222-271).  Otherwise the batch is the RAW decoded batch and the library derives the
   * canonical timestamp itself, on the device, from top-level column `ts_column` as `array_to_timestamp_array` does
   * (physical_plan/utils/time.rs:59-94): Int64 milliseconds, Int64 seconds (x 1000) or a Utf8 ISO-8601 string parsed with the
   * chrono format `ts_format` (NaiveDateTime::parse_from_str(..).and_utc().timestamp_millis()); the constant `barrier_batch`
   * column is never materialised.  A NULL or unparsable timestamp is DNZ_ERR_DATA (the reference unwraps and panics). */
  int32_t ts_source;         /* DNZ_TS_* */
  int32_t ts_column;
  const char* ts_format;     /* DNZ_TS_STRING_ISO8601 only, e.g. "%Y-%m-%dT%H:%M:%S%.f" */
} dnz_window_config;

typedef struct dnz_window dnz_window;

/* One RecordBatch whose needed column buffers are already resident in device memory (the
 * Arrow<->device buffer manager's output format; also what dnz_synth_generate produces).
 * Validity bitmaps: Arrow LSB-first, NULL = no nulls, bit 0 = row 0.
 * Utf8 keys: key_off holds n_rows+1 offsets into key_bytes.  Integer keys: key_off must be NULL and key_bytes points at the
 * n_rows values (4 or 8 bytes each, aligned to their width); a non-NULL key_off is DNZ_ERR_INVALID. */
typedef struct {
  int64_t n_rows;
  const int64_t* ts;        const uint8_t* ts_valid;    /* _streaming_internal_metadata.canonical_timestamp (ms) */
  const double* val;        const uint8_t* val_valid;   /* aggregate argument                                     */
  const int32_t* key_off;   const uint8_t* key_bytes;   const uint8_t* key_valid;  /* Utf8 key: n_rows+1 offsets; integer: NULL */
} dnz_device_batch;

/* Emitted rows, device resident (valid until the next call on the handle).  Integer keys: key_off = NULL, key_bytes = the
 * n_rows values (the input's width; a NULL key's value is zero), key_bytes_len = n_rows * width. */
typedef struct {
  int64_t n_rows;
  int64_t key_bytes_len;
  const int32_t* key_off;  const uint8_t* key_bytes;  const uint8_t* key_valid;   /* one byte per row, 1 = valid */
  const int64_t* count;
  const double* min; const double* max; const double* avg; const double* sum;
  const uint8_t* agg_valid;         /* one byte per row, shared by min/max/avg/sum (0 = null: no non-null value seen) */
  const int64_t* window_start_ms; const int64_t* window_end_ms;
} dnz_device_result;

typedef struct {
  int64_t rows_in;              /* input rows consumed                                   */
  int64_t batches_in;
  int64_t rows_out;             /* rows emitted (after the filter)                       */
  int64_t windows_emitted;
  int64_t groups;               /* distinct keys interned so far                         */
  int64_t agg_launches;         /* aggregate-kernel launches                             */
  int64_t total_launches;       /* all kernel launches issued by the handle              */
  double agg_kernel_ms;         /* sum of aggregate-kernel durations (DNZ_FLAG_KERNEL_TIMING) */
  double agg_algorithmic_bytes; /* 8 ts + 8 val + 4 offset + key bytes (integer keys: 8 ts + 8 val + key width), summed over
                                   rows of timed launches */
  int64_t h2d_bytes; int64_t d2h_bytes;
  int64_t deferred_rows;        /* rows replayed after a table grew                      */
  int64_t generic_tiles; int64_t fast_tiles;
  int64_t late_batches;         /* batches that contained late rows (exact re-open path) */
  int64_t exchanged_out; int64_t exchanged_in;   /* pane-exchange packets sent / merged   */
  int64_t h2d_pageable_bytes;   /* part of h2d_bytes that came from pageable host memory (cudaMemcpyAsync, driver-staged) */
} dnz_stats;

/* replaces: StreamingWindowExec::try_new + ExecutionPlan::execute(partition, ctx)
 * (streaming_window.rs:221-251, :421-482) -- one handle per output partition.
 * input_schema: the upstream schema; must contain struct column `_streaming_internal_metadata` with child
 * `canonical_timestamp: Timestamp(ms)` (grouped_window_agg_stream.rs:549-560, common/src/lib.rs:5). */
int32_t dnz_window_create(const dnz_window_config* cfg, const struct ArrowSchema* input_schema, dnz_window** out);

/* replaces: the `Some(Ok(batch))` arm of GroupedWindowAggStream::poll_next_inner
 * (grouped_window_agg_stream.rs:326-342).  `batch` is a struct array (the C-Data form of a RecordBatch) in HOST
 * memory; it is MOVED (released by the callee once its buffers have been copied to the device).  Batches are
 * queued and aggregated max_rows_per_launch rows at a time; results appear at the next poll. */
int32_t dnz_window_push(dnz_window* w, struct ArrowArray* batch);

/* Same for batches already resident on the device (zero copy).  Buffers must stay valid until the next
 * dnz_window_poll or dnz_window_poll_device call returns. */
int32_t dnz_window_push_device(dnz_window* w, const dnz_device_batch* batches, int64_t n_batches);

/* replaces: the RecordBatch returned by poll_next (trigger_windows + concat_batches,
 * grouped_window_agg_stream.rs:220-253) with FilterExec applied.  Aggregates everything queued, then returns ALL
 * rows emitted since the previous poll as one RecordBatch (struct array) with schema
 * key | aggs... | window_start_time | window_end_time (continuous/mod.rs:42-62).  *has_output = 0 and an
 * empty batch when nothing closed (the reference returns an empty batch, :343-348). */
int32_t dnz_window_poll(dnz_window* w, struct ArrowArray* out, struct ArrowSchema* out_schema, int32_t* has_output);

/* Non-forcing variant: returns the rows emitted so far WITHOUT aggregating batches that are still queued or in flight
 * (what a poll_next would hand downstream while upstream keeps producing).  Keeps host->device transfers, kernels and
 * result hand-off overlapped; rows of queued batches appear at a later poll. */
int32_t dnz_window_poll_ready(dnz_window* w, struct ArrowArray* out, struct ArrowSchema* out_schema, int32_t* has_output);

/* As dnz_window_poll but leaves the emitted rows on the device. */
int32_t dnz_window_poll_device(dnz_window* w, dnz_device_result* out);
/* As dnz_window_poll_ready, device resident: the oldest range of emitted rows that is complete on the device and has not been
 * handed out (n_rows = 0 when there is none); never waits for queued input.  key_off entries are offsets into key_bytes,
 * key_bytes_len is where the last returned key ends.  Valid until the next call on the handle. */
int32_t dnz_window_poll_device_ready(dnz_window* w, dnz_device_result* out);

/* Test/bench only (the reference has no flush: open windows are never emitted, :348): advance the watermark
 * to watermark_ms as process_watermark would and trigger. */
int32_t dnz_window_flush(dnz_window* w, int64_t watermark_ms);

/* replaces: ExecutionPlan::metrics() / BaselineMetrics (streaming_window.rs:491-493) */
int32_t dnz_window_stats(const dnz_window* w, dnz_stats* out);
int32_t dnz_window_reset_stats(dnz_window* w);
/* current watermark (ms) or INT64_MIN: GroupedWindowAggStream::latest_watermark */
int64_t dnz_window_watermark(const dnz_window* w);
/* replaces: DataFusionError message; valid until the next call on the handle (w may be NULL: global error) */
const char* dnz_window_last_error(const dnz_window* w);
/* replaces: Drop for GroupedWindowAggStream */
void dnz_window_destroy(dnz_window* w);

/* ---- checkpoint / restore of the device state (SURVEY.md §8 f4) ----------------------------------------------------------
 * replaces: the barrier hook of GroupedWindowAggStream, which serialises its open frames into the state backend and reloads them
 * at start-up (grouped_window_agg_stream.rs:84-102, :357-417, :631-649; utils/serialization.rs:130-241).  The reference stores
 * the accumulator states per frame WITHOUT the group keys (SURVEY §5); this blob is self-contained: stream clock (watermark,
 * emission horizon, batch sequence), the key dictionary in group-id order (inline keys + long-key arena) and every open pane
 * (count/sum/min/max states, null-row counts, first-zero marks).  Layout: dnz_window.cu, `CkptHeader`.  Everything that was pushed is
 * aggregated first; emitted rows must have been polled.  The blob is allocated with malloc and freed with dnz_blob_free.
 * dnz_window_restore loads it into a FRESH operator created with the same window / aggregate configuration. */
int32_t dnz_window_checkpoint(dnz_window* w, void** blob, int64_t* bytes);
int32_t dnz_window_restore(dnz_window* w, const void* blob, int64_t bytes);
void dnz_blob_free(void* blob);

/* ---- multi-GPU pane exchange (SURVEY.md §8e): replaces RepartitionExec(Hash(group keys))
 * (physical_optimizer/coalesce_before_streaming_window_aggregate.rs:63-73) when the input is NOT key-partitioned.
 * Every rank aggregates the batches it was dealt into its own panes.  One exchange step, driven by the caller
 * (denormalized_b200/exchange.py does it with torch.distributed; the Rust shim would use NCCL directly):
 *   1. dnz_window_process          aggregate what is queued, learn the local watermark
 *   2. all-reduce(min) of the local watermarks -> global watermark
 *   3. dnz_window_export_partials  pack, per owner rank, the partial states of the keys this rank does NOT own for every
 *                                  pane that ended at or before the global watermark (owner = key hash % world)
 *   4. one all-to-all (NCCL over NVLink) of the packets and their key bytes
 *   5. dnz_window_import_partials  the owner merges them into its panes (count +, sum +, min/max, ...)
 *   6. dnz_window_flush(global watermark) + dnz_window_poll: every rank emits the closed windows of ITS keys.
 * In exchange mode windows are emitted only by step 6 (the watermark is global: no rank emits early, which also removes the
 * reference's cross-partition watermark race, SURVEY.md §5.2); batches that arrive late for an exchanged pane are rejected
 * with DNZ_ERR_UNSUPPORTED. ------------------------------------------------------------------------------------ */
typedef struct {
  int64_t n_entries;              /* packed entries, grouped by owner rank                        */
  const uint8_t* entries;         /* device: n_entries * DNZ_PARTIAL_BYTES                         */
  const int64_t* owner_counts;    /* host: entries per owner rank (world entries)                  */
  int64_t key_bytes_len;          /* device key byte arena accompanying the entries                */
  const uint8_t* key_bytes;
  const int64_t* owner_key_bytes; /* host: key bytes per owner rank (world entries)                */
  int64_t pane_lo, pane_hi;       /* pane ids covered by this export (pane_hi < pane_lo: none)     */
} dnz_partials;
#define DNZ_PARTIAL_BYTES 64
int32_t dnz_window_set_exchange(dnz_window* w, int32_t rank, int32_t world);
/* Aggregates everything queued (no emission in exchange mode).  *local_watermark_ms = INT64_MIN if none yet. */
int32_t dnz_window_process(dnz_window* w, int64_t* local_watermark_ms);
/* Packs the partial states of all panes that ended at or before `watermark_ms` and were not exported before.  The
 * buffers stay valid until the next export. */
int32_t dnz_window_export_partials(dnz_window* w, int64_t watermark_ms, dnz_partials* out);
/* Merges packets received from the other ranks (device pointers; src_counts / src_key_bytes: per sending rank, in rank
 * order) into panes pane_lo..pane_hi (the union of the ranks' exported ranges). */
int32_t dnz_window_import_partials(dnz_window* w, const uint8_t* entries, const int64_t* src_counts,
                                   const uint8_t* key_bytes, const int64_t* src_key_bytes, int64_t pane_lo, int64_t pane_hi);

/* ---- fused pane exchange: the library owns the communicator (SURVEY.md §8b/§8e).  One rank per GPU.  The six host-driven calls
 * above collapse into ONE collective call per step; the data path has no host synchronisation and no library collective:
 * every rank packs the partial states of the keys it does not own and writes them straight into the owner's receive ring in
 * the owner's HBM with P2P stores over NVLink (CUDA IPC mappings), ring space is reserved with remote atomics, the streams of
 * different ranks are ordered by interprocess CUDA events, the owner merges and emits (dnz_exchange.cu).  Scalars that the HOSTS need per step
 * (local watermark -> global watermark) travel through a POSIX shared-memory block.  The only thing asked of the caller is a
 * rendezvous all-gather at creation (the role the ncclUniqueId broadcast plays for NCCL). */
typedef struct dnz_group dnz_group;
/* all-gather `bytes` bytes from every rank into recv[rank * bytes]; returns 0 on success */
typedef int32_t (*dnz_allgather_fn)(void* ctx, const void* send, void* recv, int64_t bytes);
typedef struct {
  uint32_t abi_version;     /* DNZ_ABI_VERSION */
  int32_t rank, world;      /* world <= 32, all ranks on one node */
  int32_t device;           /* CUDA device of this rank */
  int64_t ring_entries;     /* packets one rank can RECEIVE per step (0 = 8 Mi); one packet per (pane, group) partial state */
  int64_t ring_key_bytes;   /* key bytes one rank can receive per step (0 = 256 MiB) */
} dnz_group_config;
int32_t dnz_group_create(const dnz_group_config* cfg, dnz_allgather_fn allgather, void* ctx, dnz_group** out);
/* all `world` ranks inside this process (out[world]); devices[r] may repeat (tests on one GPU) */
int32_t dnz_group_create_local(int32_t world, const int32_t* devices, int64_t ring_entries, int64_t ring_key_bytes, dnz_group** out);
void dnz_group_destroy(dnz_group* g);
/* puts the operator into exchange mode as rank `g.rank` of `g.world` (before its first batch).  expected_groups of the operator
 * must cover the GLOBAL key set: an owner interns keys it has never seen in a batch of its own.  A group serves one stream at a time: the first
 * dnz_group_step of a fresh operator begins a new stream (COLLECTIVE: on every rank in the same step, after dnz_group_flush of the
 * previous stream's operators); operators may be attached any time before. */
int32_t dnz_group_attach(dnz_group* g, dnz_window* w);
/* One exchange step = dnz_group_step_begin + dnz_group_step_pack + dnz_group_step_finish, everything enqueued on the operator's
 * stream; streams of different ranks are ordered by interprocess CUDA events.  COLLECTIVE: every rank calls it the same number
 * of times.  Multi-process callers use dnz_group_step; a process that drives several ranks calls each phase for all of its ranks
 * before the next phase.  Emitted rows are fetched with dnz_window_poll / poll_device(_ready) as usual.
 * The protocol is pipelined over three steps so that no step waits for what a peer does at the same moment:
 *   step s   begin   publishes this rank's local watermark (that of the batches LAUNCHED so far; the most recently sealed
 *                    superbatch, whose tile scan is still queued on the device, joins the next step)
 *   step s+1 pack    global watermark = min over the ranks' step-s watermarks; the panes it closes are packed and written
 *                    straight into the owners' rings
 *   step s+2 finish  the owners merge those packets and emit the windows closed under that watermark (returned in
 *                    *global_watermark_ms; INT64_MIN while there is none)
 * Numerical note: which of +0.0 / -0.0 a min / max reports when both occur in a window is decided by arrival order ("first seen
 * wins", DataFusion's `if cur > v`); across ranks the order is each rank's LOCAL batch sequence, so the sign of such a zero can
 * differ from what a single stream would report.  Everything else is bit-identical (count, min, max) or within 1e-9 (avg).
 * dnz_group_flush = dnz_window_process + three steps: everything pushed so far is exchanged and its closed windows are emitted
 * (end of stream, tests). */
int32_t dnz_group_step_begin(dnz_group* g, dnz_window* w);
int32_t dnz_group_step_pack(dnz_group* g, dnz_window* w);
int32_t dnz_group_step_finish(dnz_group* g, dnz_window* w, int64_t* global_watermark_ms);
int32_t dnz_group_step(dnz_group* g, dnz_window* w, int64_t* global_watermark_ms);
int32_t dnz_group_flush(dnz_group* g, dnz_window* w, int64_t* global_watermark_ms);

/* ---- Arrow<->device buffer manager helpers ---------------------------------------------------------- */
/* Reserves the device staging area for host batches up front (both halves of the double buffer, `bytes_per_launch`
 * each; ~40 B per row of max_rows_per_launch for the sensor schema) so that a fresh operator does not pay for
 * device allocations while its first batches stream in.  Optional; without it the arena grows on demand.
 * (≙ the buffer-capacity knobs of a DataFusion operator, e.g. batch_size; no direct counterpart.) */
int32_t dnz_window_reserve_input(dnz_window* w, int64_t bytes_per_launch);
/* Page-locked host allocation: Arrow buffers placed here are copied host->device at full PCIe speed without a
 * staging copy (arrow-rs: Buffer::from_custom_allocation). */
void* dnz_host_alloc(int64_t bytes);
void dnz_host_free(void* p);
void* dnz_device_alloc(int32_t device, int64_t bytes);
void dnz_device_free(int32_t device, void* p);
int32_t dnz_device_count(void);
/* plain cudaMemcpy for callers that hold device pointers from this library (kind: 1 = host->device, 2 = device->host) */
int32_t dnz_memcpy(void* dst, const void* src, int64_t bytes, int32_t kind);

/* ---- synthetic sensor stream (SURVEY.md §8d; examples/examples/emit_measurements.rs:30-33,45) -------- */
/* Generates rows [row0, row0+n_rows) of the counter-based stream directly into device buffers laid out as
 * consecutive batches of batch_rows rows; fills `out` (n_batches = ceil(n_rows/batch_rows) entries).  The
 * buffers belong to the returned arena handle and are freed by dnz_synth_free. */
typedef struct dnz_synth dnz_synth;
int32_t dnz_synth_generate(int32_t device, int64_t row0, int64_t n_rows, int64_t batch_rows, uint64_t seed,
                           int64_t groups, int64_t rows_per_ms, int64_t t0_ms,
                           int32_t key_kind,  /* 0 "sensor_<id>" (Utf8), 1 a UUID string per id (Utf8), 2 Int64 keys = id */
                           int64_t key_mul, int64_t key_add, /* key id = id * key_mul + key_add (rank sharding) */
                           dnz_synth** arena, dnz_device_batch* out, int64_t n_batches);
int64_t dnz_synth_bytes(const dnz_synth* arena);   /* algorithmic bytes held: 20*rows + key bytes (Int64 keys: 24*rows) */
void dnz_synth_free(dnz_synth* arena);

#ifdef __cplusplus
}
#endif
#endif
