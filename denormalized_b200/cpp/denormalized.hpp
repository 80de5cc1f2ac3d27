// denormalized.hpp -- C++ host-side mirror of the reference's operator interface for the streaming-window hot path,
// written above the C ABI (include/dnz_gpu.h).  The reference is Rust; no Rust toolchain exists in this image, so the
// host side that a Rust maintainer would write (rust/gpu_streaming_window.rs, INTEGRATION.md) is mirrored here in C++
// with the same names, argument meaning and error behaviour, so that tests read like the reference's own examples:
//
//   reference (examples/examples/udf_example.rs:51-62)                 this header
//   ctx.from_topic(t).await?                                           DataStream::from_schema(schema)
//      .window(vec![col("sensor_name")],                                  .window({col("sensor_name")},
//              vec![count(col("reading")).alias("count"), ...],                    {count(col("reading")).alias("count"), ...},
//              Duration::from_millis(1000), None)?                                 Duration::from_millis(1000), std::nullopt)
//      .filter(col("max").gt(lit(113)))?                                  .filter(col("max").gt(lit(113)))
//
//   StreamingWindowExec::try_new(mode, group_by, aggr_expr, filter_expr, input, input_schema, window_type,
//                                upstream_partitioning)   crates/core/src/physical_plan/continuous/streaming_window.rs:221-251
//   ExecutionPlan::execute(partition, ctx) -> stream      streaming_window.rs:421-482
//   Stream::poll_next                                      grouped_window_agg_stream.rs:326-349, :432-436
//
// Errors: the reference returns datafusion::common::Result<T>; here every fallible call throws DataFusionError
// (message = dnz_window_last_error).  There is no CPU fallback: unsupported plan shapes throw.
#pragma once
#include <cstdint>
#include <memory>
#include <optional>
#include <stdexcept>
#include <string>
#include <utility>
#include <vector>

#include "../../include/dnz_gpu.h"

namespace denormalized {

struct DataFusionError : std::runtime_error {
  int32_t code;
  DataFusionError(int32_t c, const std::string& m) : std::runtime_error(m), code(c) {}
};

struct Duration {
  int64_t ms;
  static Duration from_millis(int64_t v) { return Duration{v}; }
  static Duration from_secs(int64_t v) { return Duration{v * 1000}; }
};

// ---- logical expressions (the subset the planner accepts on this path, planner/streaming_window.rs:36-66) ------------
struct Expr {
  enum Kind { Column, Literal, Aggregate, Binary } kind = Column;
  std::string name;            // column name / alias
  double literal = 0.0;
  int agg_kind = -1;           // DNZ_AGG_*
  int op = -1;                 // DNZ_OP_*
  std::shared_ptr<Expr> lhs, rhs;
  Expr alias(const std::string& a) const { Expr e = *this; e.name = a; return e; }
  Expr cmp(int o, const Expr& r) const {
    Expr e; e.kind = Binary; e.op = o; e.lhs = std::make_shared<Expr>(*this); e.rhs = std::make_shared<Expr>(r); return e;
  }
  Expr gt(const Expr& r) const { return cmp(DNZ_OP_GT, r); }
  Expr gt_eq(const Expr& r) const { return cmp(DNZ_OP_GTE, r); }
  Expr lt(const Expr& r) const { return cmp(DNZ_OP_LT, r); }
  Expr lt_eq(const Expr& r) const { return cmp(DNZ_OP_LTE, r); }
  Expr eq(const Expr& r) const { return cmp(DNZ_OP_EQ, r); }
  Expr not_eq_(const Expr& r) const { return cmp(DNZ_OP_NEQ, r); }
};
inline Expr col(const std::string& n) { Expr e; e.kind = Expr::Column; e.name = n; return e; }
inline Expr lit(double v) { Expr e; e.kind = Expr::Literal; e.literal = v; return e; }   // lit(113) coerces to Float64 as the analyzer does
inline Expr agg(int kind, const Expr& arg, const char* dflt) {
  Expr e; e.kind = Expr::Aggregate; e.agg_kind = kind; e.lhs = std::make_shared<Expr>(arg); e.name = dflt; return e;
}
inline Expr count(const Expr& a) { return agg(DNZ_AGG_COUNT, a, "count"); }
inline Expr min(const Expr& a) { return agg(DNZ_AGG_MIN, a, "min"); }
inline Expr max(const Expr& a) { return agg(DNZ_AGG_MAX, a, "max"); }
inline Expr avg(const Expr& a) { return agg(DNZ_AGG_AVG, a, "avg"); }
inline Expr sum(const Expr& a) { return agg(DNZ_AGG_SUM, a, "sum"); }

// PhysicalStreamingWindowType (streaming_window.rs:193-198); Session is declared but `todo!()` in the reference.
struct PhysicalStreamingWindowType {
  enum Kind { Tumbling, Sliding } kind;
  Duration length, slide;
  static PhysicalStreamingWindowType tumbling(Duration l) { return {Tumbling, l, Duration{0}}; }
  static PhysicalStreamingWindowType sliding(Duration l, Duration s) { return {Sliding, l, s}; }
};
// grouped windows are planned as AggregateMode::Single; the ungrouped `.window([], ..)` as Partial -> Final
// (planner/streaming_window.rs:120-165) -- here ONE operator runs the Partial reduction on the device and the Final stage on
// the host (include/dnz_gpu.h, DNZ_NO_KEY), so the mirror accepts Single for both.
enum class AggregateMode { Single };

// TimestampUnit (physical_plan/utils/time.rs:15-19) + KafkaTopicBuilder::with_timestamp (datasource/kafka/kafka_config.rs:171-179):
// where the event time of a batch comes from.  Without it the batch already carries `_streaming_internal_metadata`.
struct TimestampUnit {
  int32_t source = DNZ_TS_CANONICAL; std::string format;
  static TimestampUnit Int64Millis() { return {DNZ_TS_INT64_MILLIS, {}}; }
  static TimestampUnit Int64Seconds() { return {DNZ_TS_INT64_SECONDS, {}}; }
  static TimestampUnit StringIso8601(std::string chrono_format) { return {DNZ_TS_STRING_ISO8601, std::move(chrono_format)}; }
};

struct AggregateFunctionExpr { int kind; std::string arg_column; std::string alias; };
struct PhysicalGroupBy { std::vector<std::string> columns; };
struct FilterPredicate { std::string column; int op; double literal; };     // FilterExec: BinaryExpr(Column op Literal)

// An owned Arrow C-Data RecordBatch (struct array + schema); released on destruction.
struct RecordBatch {
  ArrowArray array{}; ArrowSchema schema{};
  RecordBatch() = default;
  RecordBatch(const RecordBatch&) = delete; RecordBatch& operator=(const RecordBatch&) = delete;
  RecordBatch(RecordBatch&& o) noexcept : array(o.array), schema(o.schema) { o.array.release = nullptr; o.schema.release = nullptr; }
  ~RecordBatch() { if (array.release) array.release(&array); if (schema.release) schema.release(&schema); }
  int64_t num_rows() const { return array.length; }
};

// GroupedWindowAggStream (grouped_window_agg_stream.rs:63-82): one partition's stream.
class GroupedWindowAggStream {
 public:
  explicit GroupedWindowAggStream(dnz_window* h) : h_(h) {}
  GroupedWindowAggStream(const GroupedWindowAggStream&) = delete;
  GroupedWindowAggStream(GroupedWindowAggStream&& o) noexcept : h_(o.h_) { o.h_ = nullptr; }
  ~GroupedWindowAggStream() { if (h_) dnz_window_destroy(h_); }
  // poll_next with an upstream batch available: feeds it (moved) and returns what has closed.  The reference emits after
  // every batch; pass `drain=false` to let batches queue (rows appear at a later poll) -- same stream contents, less latency control.
  RecordBatch poll_next(ArrowArray* upstream_batch, bool drain = true) {
    if (upstream_batch) check(dnz_window_push(h_, upstream_batch));
    RecordBatch out; int32_t has = 0;
    check(drain ? dnz_window_poll(h_, &out.array, &out.schema, &has) : dnz_window_poll_ready(h_, &out.array, &out.schema, &has));
    return out;
  }
  int64_t watermark() const { return dnz_window_watermark(h_); }
  // The barrier hook (grouped_window_agg_stream.rs:357-417): serialise the open frames / reload them into a fresh stream of the
  // same plan (:84-102).  The reference writes into its SlateDB backend; here the caller owns the bytes.
  std::vector<uint8_t> checkpoint() {
    void* blob = nullptr; int64_t n = 0;
    check(dnz_window_checkpoint(h_, &blob, &n));
    std::vector<uint8_t> out(static_cast<uint8_t*>(blob), static_cast<uint8_t*>(blob) + n);
    dnz_blob_free(blob);
    return out;
  }
  void restore(const std::vector<uint8_t>& blob) { check(dnz_window_restore(h_, blob.data(), (int64_t)blob.size())); }
  dnz_stats metrics() const { dnz_stats s{}; dnz_window_stats(h_, &s); return s; }   // ExecutionPlan::metrics()
  dnz_window* handle() { return h_; }

 private:
  void check(int32_t rc) { if (rc != DNZ_OK) throw DataFusionError(rc, dnz_window_last_error(h_)); }
  dnz_window* h_;
};

// StreamingWindowExec (streaming_window.rs:200-251) -- the operator shell.  `input` is represented by its schema: the
// upstream operator's batches are handed to the per-partition stream by the caller (DataFusion's pull loop in the reference).
class StreamingWindowExec {
 public:
  static StreamingWindowExec try_new(AggregateMode mode, PhysicalGroupBy group_by, std::vector<AggregateFunctionExpr> aggr_expr,
                                     std::optional<FilterPredicate> filter_expr, const ArrowSchema* input_schema,
                                     PhysicalStreamingWindowType window_type, std::optional<size_t> upstream_partitioning,
                                     int32_t device = 0) {
    (void)mode;
    if (group_by.columns.size() > 1) throw DataFusionError(DNZ_ERR_UNSUPPORTED, "GPU streaming window: at most one plain group-by column is implemented");
    StreamingWindowExec e;
    e.group_by_ = std::move(group_by); e.aggr_ = std::move(aggr_expr); e.filter_ = std::move(filter_expr);
    e.input_schema_ = input_schema; e.window_type_ = window_type; e.upstream_partitioning_ = upstream_partitioning; e.device_ = device;
    return e;
  }
  // ExecutionPlan::execute(partition, ctx): one handle per output partition (streaming_window.rs:470-481)
  GroupedWindowAggStream execute(size_t partition, int64_t expected_groups = 0, int64_t max_rows_per_launch = 0) const {
    (void)partition;
    auto col_index = [&](const std::string& n) -> int32_t {
      for (int64_t i = 0; i < input_schema_->n_children; i++) if (input_schema_->children[i]->name && n == input_schema_->children[i]->name) return (int32_t)i;
      throw DataFusionError(DNZ_ERR_INVALID, "no such column: " + n);
    };
    std::vector<dnz_agg> aggs;
    for (auto& a : aggr_) aggs.push_back(dnz_agg{a.kind, col_index(a.arg_column), a.alias.c_str()});
    dnz_window_config c{};
    c.abi_version = DNZ_ABI_VERSION; c.device = device_;
    // the group key column: Utf8, Int64, Int32, UInt64 or UInt32 (the library returns DNZ_ERR_UNSUPPORTED for any other type)
    c.key_column = group_by_.columns.empty() ? DNZ_NO_KEY : col_index(group_by_.columns[0]);      // `.window([], ..)`: WindowAggStream
    if (timestamp_unit_.source != DNZ_TS_CANONICAL) {
      c.ts_source = timestamp_unit_.source; c.ts_column = col_index(timestamp_column_);
      c.ts_format = timestamp_unit_.source == DNZ_TS_STRING_ISO8601 ? timestamp_unit_.format.c_str() : nullptr;
    }
    c.n_aggs = (int32_t)aggs.size(); c.aggs = aggs.data();
    c.window_ms = window_type_.length.ms; c.slide_ms = window_type_.kind == PhysicalStreamingWindowType::Sliding ? window_type_.slide.ms : 0;
    if (filter_) {
      c.has_filter = 1; c.filter_op = filter_->op; c.filter_literal = filter_->literal; c.filter_agg = -1;
      for (size_t i = 0; i < aggr_.size(); i++) if (aggr_[i].alias == filter_->column) c.filter_agg = (int32_t)i;
      if (c.filter_agg < 0) throw DataFusionError(DNZ_ERR_UNSUPPORTED, "filter column must be one of the window's aggregates");
    }
    c.expected_groups = expected_groups; c.max_rows_per_launch = max_rows_per_launch;
    dnz_window* h = nullptr;
    int32_t rc = dnz_window_create(&c, input_schema_, &h);
    if (rc != DNZ_OK) throw DataFusionError(rc, dnz_window_last_error(nullptr));
    return GroupedWindowAggStream(h);
  }
  // schema(): group key | aggregates | window_start_time | window_end_time (create_schema :1096-1134 + continuous/mod.rs:42-62)
  std::vector<std::string> schema_names() const {
    std::vector<std::string> n;
    if (!group_by_.columns.empty()) n.push_back(group_by_.columns[0]);
    for (auto& a : aggr_) n.push_back(a.alias);
    n.push_back("window_start_time"); n.push_back("window_end_time");
    return n;
  }
  const char* name() const { return "StreamingWindowExec"; }
  // the source's with_timestamp(column, unit): the operator derives the canonical timestamp itself (utils/time.rs:59-94)
  StreamingWindowExec& with_timestamp(std::string timestamp_column, TimestampUnit unit) {
    timestamp_column_ = std::move(timestamp_column); timestamp_unit_ = std::move(unit); return *this;
  }

 private:
  std::string timestamp_column_; TimestampUnit timestamp_unit_;
  PhysicalGroupBy group_by_; std::vector<AggregateFunctionExpr> aggr_; std::optional<FilterPredicate> filter_;
  const ArrowSchema* input_schema_ = nullptr; PhysicalStreamingWindowType window_type_{PhysicalStreamingWindowType::Tumbling, {0}, {0}};
  std::optional<size_t> upstream_partitioning_; int32_t device_ = 0;
};

// DataStream (crates/core/src/datastream.rs:35-40): window() (:178-196) and filter() (:94-105) build the plan; the
// "physical planning" step (StreamingWindowPlanner::plan_extension, planner/streaming_window.rs:71-172) is `plan()`.
class DataStream {
 public:
  static DataStream from_schema(const ArrowSchema* schema) { DataStream d; d.schema_ = schema; return d; }
  DataStream window(std::vector<Expr> group_expr, std::vector<Expr> aggr_expr, Duration window_length, std::optional<Duration> slide) const {
    DataStream d = *this;
    for (auto& g : group_expr) {
      if (g.kind != Expr::Column) throw DataFusionError(DNZ_ERR_UNSUPPORTED, "only plain column group keys are accepted (planner/streaming_window.rs:36-66)");
      d.group_.columns.push_back(g.name);
    }
    for (auto& a : aggr_expr) {
      if (a.kind != Expr::Aggregate || !a.lhs || a.lhs->kind != Expr::Column) throw DataFusionError(DNZ_ERR_UNSUPPORTED, "aggregate must be f(col)");
      d.aggr_.push_back(AggregateFunctionExpr{a.agg_kind, a.lhs->name, a.name});
    }
    d.window_ = slide ? PhysicalStreamingWindowType::sliding(window_length, *slide) : PhysicalStreamingWindowType::tumbling(window_length);
    d.has_window_ = true;
    return d;
  }
  DataStream filter(const Expr& predicate) const {
    if (!has_window_) throw DataFusionError(DNZ_ERR_UNSUPPORTED, "only the post-aggregate filter is on the GPU path");
    if (predicate.kind != Expr::Binary || predicate.lhs->kind != Expr::Column || predicate.rhs->kind != Expr::Literal)
      throw DataFusionError(DNZ_ERR_UNSUPPORTED, "filter must be <aggregate column> <op> <literal>");
    DataStream d = *this;
    d.filter_ = FilterPredicate{predicate.lhs->name, predicate.op, predicate.rhs->literal};
    return d;
  }
  // KafkaTopicBuilder::with_timestamp (kafka_config.rs:171-179): the raw event-time column of the source and its unit
  DataStream with_timestamp(std::string timestamp_column, TimestampUnit unit) const {
    DataStream d = *this; d.ts_column_ = std::move(timestamp_column); d.ts_unit_ = std::move(unit); return d;
  }
  StreamingWindowExec plan(int32_t device = 0) const {
    if (!has_window_) throw DataFusionError(DNZ_ERR_INVALID, "no window() in the pipeline");
    StreamingWindowExec e = StreamingWindowExec::try_new(AggregateMode::Single, group_, aggr_, filter_, schema_, window_, std::nullopt, device);
    if (ts_unit_.source != DNZ_TS_CANONICAL) e.with_timestamp(ts_column_, ts_unit_);
    return e;
  }

 private:
  const ArrowSchema* schema_ = nullptr; PhysicalGroupBy group_; std::vector<AggregateFunctionExpr> aggr_;
  std::optional<FilterPredicate> filter_; PhysicalStreamingWindowType window_{PhysicalStreamingWindowType::Tumbling, {0}, {0}};
  bool has_window_ = false;
  std::string ts_column_; TimestampUnit ts_unit_;
};

// RepartitionExec(Hash(group keys), n) for input that is NOT key-partitioned
// (physical_optimizer/coalesce_before_streaming_window_aggregate.rs:63-73), with the communicator owned by the library: every rank
// aggregates the batches it is dealt, `step` moves the closed panes' partial states to their owners over NVLink and the owners emit.
// One group per process and GPU; `allgather` is whatever the deployment has (used twice, at creation).
class RepartitionGroup {
 public:
  RepartitionGroup(int32_t rank, int32_t world, int32_t device, dnz_allgather_fn allgather, void* ctx,
                   int64_t ring_entries = 0, int64_t ring_key_bytes = 0) {
    dnz_group_config c{}; c.abi_version = DNZ_ABI_VERSION; c.rank = rank; c.world = world; c.device = device;
    c.ring_entries = ring_entries; c.ring_key_bytes = ring_key_bytes;
    const int32_t rc = dnz_group_create(&c, allgather, ctx, &g_);
    if (rc != DNZ_OK) throw DataFusionError(rc, dnz_window_last_error(nullptr));
  }
  RepartitionGroup(const RepartitionGroup&) = delete;
  ~RepartitionGroup() { if (g_) dnz_group_destroy(g_); }
  void attach(GroupedWindowAggStream& s) { check(dnz_group_attach(g_, s.handle()), s); }
  // COLLECTIVE; returns the global watermark under which this step emitted (INT64_MIN: none yet)
  int64_t step(GroupedWindowAggStream& s) { int64_t wm = 0; check(dnz_group_step(g_, s.handle(), &wm), s); return wm; }
  int64_t flush(GroupedWindowAggStream& s) { int64_t wm = 0; check(dnz_group_flush(g_, s.handle(), &wm), s); return wm; }

 private:
  void check(int32_t rc, GroupedWindowAggStream& s) { if (rc != DNZ_OK) throw DataFusionError(rc, dnz_window_last_error(s.handle())); }
  dnz_group* g_ = nullptr;
};

}  // namespace denormalized
