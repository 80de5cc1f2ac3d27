// dnz_window.cu -- host side of the H100 streaming-window operator behind the C ABI of include/dnz_gpu.h.
//
// Mirrors GroupedWindowAggStream (crates/core/src/physical_plan/continuous/grouped_window_agg_stream.rs):
//   push/poll           <-> poll_next_inner (:326-349): watermark -> windows -> frames.push -> process_watermark -> trigger
//   pipeline (Slot)     <-> the stream's poll loop, three superbatches deep: scan k+1 | aggregate + emit k | verify k-1
//   PaneStore           <-> window_frames: BTreeMap<SystemTime, GroupedAggWindowFrame> (:63-82), re-organised as hop-sized
//                           panes shared by the L/S windows that overlap them (SURVEY.md §5.7)
//   Dictionary          <-> GroupValues (one per frame in the reference; one per stream here, ids are stable)
//   plan_runs           <-> the per-batch watermark rule (:255-266) + late rows re-opening emitted windows (§8a-3)
// and the Arrow<->device buffer manager (host Arrow C-Data in, device columns; the way out is dnz_results.cu).  Ungrouped windows
// finish in dnz_ungrouped.cu, the multi-GPU exchange lives in dnz_group.cu; dnz_window.h declares what they share.
#include "dnz_window.h"

namespace dnz {

// ------------------------------------------------------------------------------------------------
// device memory helpers.  All device buffers come from the CUDA stream-ordered allocator with an unbounded release
// threshold: blocks freed by one operator stay cached in the process and are handed to the next one without a driver
// call (plain cudaMalloc/cudaFree cost milliseconds to seconds once tens of GB are mapped, and cudaFree synchronises
// the whole device).
AllocCtx& alloc_ctx() {
  static thread_local int cached_dev = -1; static thread_local AllocCtx* cur = nullptr;
  static std::mutex m; static std::map<int, AllocCtx> ctxs;
  int dev = 0; cudaGetDevice(&dev);
  if (dev == cached_dev && cur) return *cur;
  std::lock_guard<std::mutex> g(m);
  AllocCtx& c = ctxs[dev];
  if (!c.s) {
    int supported = 0; cudaDeviceGetAttribute(&supported, cudaDevAttrMemoryPoolsSupported, dev);
    if (cudaStreamCreateWithFlags(&c.s, cudaStreamNonBlocking) != cudaSuccess) c.s = nullptr;
    cudaMemPool_t pool;
    if (supported && c.s && cudaDeviceGetDefaultMemPool(&pool, dev) == cudaSuccess) {
      uint64_t thr = UINT64_MAX;
      c.async_ok = cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &thr) == cudaSuccess;
    }
    cudaGetLastError();
  }
  cached_dev = dev; cur = &c;
  return c;
}
void* dev_alloc(size_t n) {
  AllocCtx& c = alloc_ctx();
  void* p = nullptr;
  if (g_trace && n >= (256ull << 20)) { size_t fr = 0, tot = 0; cudaMemGetInfo(&fr, &tot); fprintf(stderr, "[dnz] alloc %.2f GB (device free %.1f of %.1f GB)\n", n / 1e9, fr / 1e9, tot / 1e9); }
  if (c.async_ok) { CK(cudaMallocAsync(&p, n, c.s)); CK(cudaStreamSynchronize(c.s)); }
  else CK(cudaMalloc(&p, n));
  return p;
}
void dev_free(void* p) {          // callers free only after the work that used the block has completed
  if (!p) return;
  AllocCtx& c = alloc_ctx();
  if (c.async_ok) cudaFreeAsync(p, c.s); else cudaFree(p);
}

}  // namespace dnz

// =================================================================================================
dnz_window::~dnz_window() {
  cudaSetDevice(dev);
  if (copy_stream) cudaStreamSynchronize(copy_stream);
  if (stream) cudaStreamSynchronize(stream);
  for (Slot& s : slot) {
    for (auto& pb : s.batches) if (pb.has_moved && pb.moved.release) pb.moved.release(&pb.moved);
    for (cudaEvent_t e : {s.copy_done, s.scan_done, s.done, s.ev0, s.ev1}) if (e) cudaEventDestroy(e);
  }
  if (copy_stream) cudaStreamDestroy(copy_stream);
  if (d2h_stream) { cudaStreamSynchronize(d2h_stream); cudaStreamDestroy(d2h_stream); }
  for (auto& r : rs) if (r.snap_ev) cudaEventDestroy(r.snap_ev);
  if (own_stream && stream) cudaStreamDestroy(stream);
}

void dnz_window::init(const dnz_window_config* c, const ArrowSchema* schema) {
  if (!c || !schema) fail(DNZ_ERR_INVALID, "null config or schema");
  if (c->abi_version != DNZ_ABI_VERSION) fail(DNZ_ERR_INVALID, "abi_version %u != %u", c->abi_version, DNZ_ABI_VERSION);
  cfg = *c;
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) fail(DNZ_ERR_CUDA, "no CUDA device: the GPU operator has no CPU fallback");
  if (c->device < 0 || c->device >= ndev) fail(DNZ_ERR_INVALID, "device %d out of range (%d devices)", c->device, ndev);
  dev = c->device;
  CK(cudaSetDevice(dev));
  cudaDeviceProp prop; CK(cudaGetDeviceProperties(&prop, dev));
  if (prop.major != 9 || prop.minor != 0) fail(DNZ_ERR_UNSUPPORTED, "device %s is sm_%d%d; this library is built for sm_90a only", prop.name, prop.major, prop.minor);
  sm_count = prop.multiProcessorCount;

  // ---- plan shape (planner/streaming_window.rs:36-66: plain column group keys; count/min/max/avg aggregates)
  if (c->n_aggs <= 0 || !c->aggs) fail(DNZ_ERR_INVALID, "no aggregate expressions");
  if (!schema->format || strcmp(schema->format, "+s") != 0) fail(DNZ_ERR_INVALID, "input schema must be a struct (RecordBatch)");
  n_input_cols = (int)schema->n_children;
  if (c->key_column == DNZ_NO_KEY) {       // `.window([], aggs, ..)`: WindowAggStream (Partial) -> FullWindowAggStream (Final)
    ungrouped = true; key_col = -1; key_name = "";
    if (c->has_filter) fail(DNZ_ERR_UNSUPPORTED, "a fused filter on an ungrouped window is not implemented");
  } else {
    if (c->key_column < 0 || c->key_column >= n_input_cols) fail(DNZ_ERR_INVALID, "key_column out of range");
    key_col = c->key_column;
    const ArrowSchema* ks = schema->children[key_col];
    // DataFusion's GroupValuesPrimitive for the integer types: one group per distinct value, NULL is a group of its own
    const char* kf = ks->format ? ks->format : "";
    if (ks->dictionary) fail(DNZ_ERR_UNSUPPORTED, "group key column '%s' is dictionary-encoded; dictionary keys are not implemented", ks->name);
    key_type = -1;
    for (int t = 0; t < N_KEY_TYPES; t++) if (strcmp(kf, KEY_TYPES[t].format) == 0) key_type = t;
    if (key_type < 0) fail(DNZ_ERR_UNSUPPORTED, "group key column '%s' has format '%s'; only Utf8, Int64, Int32, UInt64 and UInt32 keys are implemented", ks->name, kf);
    key_width = KEY_TYPES[key_type].width;
    key_nullable = (ks->flags & ARROW_FLAG_NULLABLE) != 0;
    key_name = ks->name ? ks->name : "key";
  }
  val_col = -1;
  for (int i = 0; i < c->n_aggs; i++) {
    const dnz_agg& a = c->aggs[i];
    if (a.kind < DNZ_AGG_COUNT || a.kind > DNZ_AGG_SUM) fail(DNZ_ERR_UNSUPPORTED, "aggregate kind %d not implemented", a.kind);
    if (a.arg_column < 0 || a.arg_column >= n_input_cols) fail(DNZ_ERR_INVALID, "aggregate %d: arg_column out of range", i);
    if (strcmp(schema->children[a.arg_column]->format, "g") != 0) fail(DNZ_ERR_UNSUPPORTED, "aggregate %d: argument must be Float64", i);
    if (val_col >= 0 && val_col != a.arg_column) fail(DNZ_ERR_UNSUPPORTED, "all aggregates must share one argument column (got %d and %d)", val_col, a.arg_column);
    val_col = a.arg_column;
    aggs.push_back(a);
    aliases.push_back(a.alias ? a.alias : (a.kind == DNZ_AGG_COUNT ? "count" : a.kind == DNZ_AGG_MIN ? "min" : a.kind == DNZ_AGG_MAX ? "max" : a.kind == DNZ_AGG_AVG ? "average" : "sum"));
  }
  for (size_t i = 0; i < aggs.size(); i++) aggs[i].alias = aliases[i].c_str();
  ts_source = c->ts_source; ts_col = -1;
  if (ts_source == DNZ_TS_CANONICAL) {
    meta_col = -1;
    for (int i = 0; i < n_input_cols; i++)
      if (schema->children[i]->name && strcmp(schema->children[i]->name, "_streaming_internal_metadata") == 0) meta_col = i;
    if (meta_col < 0) fail(DNZ_ERR_INVALID, "input schema lacks the `_streaming_internal_metadata` struct column");
    const ArrowSchema* ms = schema->children[meta_col];
    if (strcmp(ms->format, "+s") != 0) fail(DNZ_ERR_INVALID, "`_streaming_internal_metadata` must be a struct");
    ts_child = -1;
    for (int i = 0; i < ms->n_children; i++)
      if (ms->children[i]->name && strcmp(ms->children[i]->name, "canonical_timestamp") == 0) ts_child = i;
    if (ts_child < 0) fail(DNZ_ERR_INVALID, "`_streaming_internal_metadata` lacks `canonical_timestamp`");
    if (strncmp(ms->children[ts_child]->format, "tsm:", 4) != 0) fail(DNZ_ERR_INVALID, "`canonical_timestamp` must be Timestamp(Millisecond)");
  } else {
    // raw decoded batches: the canonical timestamp is derived here (kafka_stream_read.rs:236-268, utils/time.rs:59-94)
    if (ts_source < DNZ_TS_INT64_MILLIS || ts_source > DNZ_TS_STRING_ISO8601) fail(DNZ_ERR_INVALID, "bad ts_source %d", ts_source);
    if (c->ts_column < 0 || c->ts_column >= n_input_cols) fail(DNZ_ERR_INVALID, "ts_column out of range");
    ts_col = c->ts_column;
    const char* tf = schema->children[ts_col]->format;
    if (ts_source == DNZ_TS_STRING_ISO8601) {
      if (strcmp(tf, "u") != 0) fail(DNZ_ERR_INVALID, "timestamp column must be Utf8 for TimestampUnit::StringIso8601 (format '%s')", tf);
      std::string f = c->ts_format ? c->ts_format : "";
      for (const auto& kv : {std::pair<const char*, const char*>{"%F", "%Y-%m-%d"}, {"%T", "%H:%M:%S"}})
        for (size_t at; (at = f.find(kv.first)) != std::string::npos;) f.replace(at, 2, kv.second);
      if (!ts_format_supported(f.c_str())) fail(DNZ_ERR_UNSUPPORTED, "timestamp format '%s' is not supported (specifiers: %%Y %%m %%d %%H %%M %%S %%f %%.f %%3f %%6f %%9f %%.3f %%.6f %%.9f %%F %%T %%%%)", c->ts_format ? c->ts_format : "");
      memset(&ts_fmt, 0, sizeof ts_fmt); memcpy(ts_fmt.fmt, f.data(), f.size()); ts_fmt.len = (int32_t)f.size();
    } else if (strcmp(tf, "l") != 0) fail(DNZ_ERR_INVALID, "timestamp column must be Int64 for TimestampUnit::Int64Millis / Int64Seconds (format '%s')", tf);
  }
  if (c->has_filter && (c->filter_agg < 0 || c->filter_agg >= c->n_aggs || c->filter_op < DNZ_OP_GT || c->filter_op > DNZ_OP_NEQ))
    fail(DNZ_ERR_INVALID, "bad filter");

  // ---- window geometry (streaming_window.rs:1053-1094)
  L = c->window_ms; S = c->slide_ms;
  if (L <= 0 || S < 0) fail(DNZ_ERR_INVALID, "window length must be positive");
  if (L < 1000) fail(DNZ_ERR_DATA, "window length < 1 s: the reference divides by zero in snap_to_window_start");
  if (L % 1000 != 0) fail(DNZ_ERR_UNSUPPORTED, "window length must be whole seconds (the reference aligns windows in whole seconds)");
  if (S > 0 && L % S != 0) fail(DNZ_ERR_UNSUPPORTED, "sliding windows need window_ms %% slide_ms == 0 (pane sharing)");
  pane_ms = S > 0 ? S : L;
  panes_per_window = (int)(L / pane_ms);
  if (panes_per_window > MAX_WINDOW_PANES) fail(DNZ_ERR_UNSUPPORTED, "window/slide ratio %d exceeds %d", panes_per_window, MAX_WINDOW_PANES);
  if (c->max_rows_per_launch > 0) max_rows = c->max_rows_per_launch;

  if (c->cuda_stream) { stream = (cudaStream_t)c->cuda_stream; own_stream = false; }
  else { CK(cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking)); own_stream = true; }
  CK(cudaStreamCreateWithFlags(&copy_stream, cudaStreamNonBlocking));
  CK(cudaStreamCreateWithFlags(&d2h_stream, cudaStreamNonBlocking));
  for (auto& r : rs) { CK(cudaEventCreateWithFlags(&r.snap_ev, cudaEventDisableTiming)); r.snap.reserve(64); }
  for (int i = 0; i < PIPELINE_SLOTS; i++) {
    Slot& s = slot[i]; s.idx = i;
    CK(cudaEventCreateWithFlags(&s.copy_done, cudaEventDisableTiming));
    CK(cudaEventCreateWithFlags(&s.scan_done, cudaEventDisableTiming));
    CK(cudaEventCreateWithFlags(&s.done, cudaEventDisableTiming));
    CK(cudaEventCreate(&s.ev0)); CK(cudaEventCreate(&s.ev1));
    s.snap.reserve(sizeof(CtlBlock));
  }
  slot[0].state = Slot::FILLING; fill = 0;
  CK(agg_kernel_setup());

  d_ctl.alloc(sizeof(CtlBlock)); CK(cudaMemsetAsync(d_ctl.p, 0, sizeof(CtlBlock), stream));
  uint64_t eg = c->expected_groups > 0 ? (uint64_t)c->expected_groups : (1ull << 16);
  uint64_t g0 = 1024; while (g0 < eg + eg / 8) g0 <<= 1;
  if (g0 > (1ull << 29)) fail(DNZ_ERR_INVALID, "expected_groups too large");
  if (ungrouped) g0 = 1024;
  dict_alloc((uint32_t)g0);
  arena_cap = 1 << 20; arena.alloc(arena_cap);
  if (ungrouped) {
    need_nullrows = true;
    u_ring = 4096;
    d_uwins.alloc(u_ring * sizeof(UWindow)); d_ustates.alloc(u_ring * sizeof(UState));
    h_uwins.reserve(u_ring * sizeof(UWindow)); h_ustates.reserve(u_ring * sizeof(UState));
  }
  prealloc();
  CK(cudaStreamSynchronize(stream));
}

DictView dnz_window::dict_view() const {
  DictView d;
  d.slots = slots.as<DictSlot>(); d.mask = dict_cap - 1; d.gcap = gcap;
  DictCounters* c = &ctl()->dict;
  d.n_groups = &c->n_groups; d.null_gid = &c->null_gid;
  d.arena_used = &c->arena_used;
  d.key_bytes_total = &c->key_bytes_total;
  d.gid_key = gid_key.as<GidKey>();
  d.arena = arena.as<uint8_t>(); d.arena_cap = arena_cap;
  return d;
}

template <class F> void dnz_window::for_each_live_pane(F f) {
  for (auto& kv : panes) f(kv.second.get());
  for (auto& kv : late_panes) f(kv.second.get());
  for (Slot& s : slot) for (auto& p : s.retired) f(p.get());
}

// Slots per group id.  The first probe of a key misses its home slot with probability ~ load / 2; every miss costs a second
// scattered 32 B transaction (and a trip through the warp's retry queue), while an EMPTY slot is never touched by a lookup --
// the L2 footprint of the table is its occupied sectors, not its capacity.  So small and medium tables are kept very sparse.
static uint32_t dict_slots_per_group(uint32_t gcap_) { return gcap_ <= (1u << 20) ? 16u : gcap_ <= (1u << 23) ? 8u : 4u; }

// (re)allocate dictionary + per-pane state arrays for `new_gcap` groups, preserving contents
void dnz_window::dict_alloc(uint32_t new_gcap) {
  uint32_t new_cap = new_gcap * dict_slots_per_group(new_gcap);
  DevBuf ns, ng;
  ns.alloc((size_t)new_cap * sizeof(DictSlot)); CK(cudaMemsetAsync(ns.p, 0, ns.bytes, stream));
  ng.alloc((size_t)new_gcap * sizeof(GidKey)); CK(cudaMemsetAsync(ng.p, 0, ng.bytes, stream));
  if (dict_cap) {
    CK(cudaMemcpyAsync(ng.p, gid_key.p, (size_t)gcap * sizeof(GidKey), cudaMemcpyDeviceToDevice, stream));
    DictView nd = dict_view(); nd.slots = ns.as<DictSlot>(); nd.mask = new_cap - 1; nd.gcap = new_gcap; nd.gid_key = ng.as<GidKey>();
    CK(launch_dict_rehash(slots.as<DictSlot>(), dict_cap, nd, stream)); stats.total_launches++;
    // grow every live pane: the open ones, the one-batch late panes of a dirty run, and retired panes still awaiting their
    // (possibly re-issued) emission
    auto grow = [&](DevBuf& b, size_t elem, int fill_byte) {
      if (!b.p) return;
      DevBuf nb; nb.alloc((size_t)new_gcap * elem);
      CK(cudaMemcpyAsync(nb.p, b.p, (size_t)gcap * elem, cudaMemcpyDeviceToDevice, stream));
      CK(cudaMemsetAsync((char*)nb.p + (size_t)gcap * elem, fill_byte, (size_t)(new_gcap - gcap) * elem, stream));
      CK(cudaStreamSynchronize(stream));
      b = std::move(nb);
    };
    for_each_live_pane([&](Pane* p) { grow(p->st, sizeof(GroupState), 0); grow(p->nullrows, 8, 0); grow(p->fz, 8, 0xFF); });
    pane_pool.clear();
    CK(cudaStreamSynchronize(stream));
  }
  slots = std::move(ns); gid_key = std::move(ng);
  dict_cap = new_cap; gcap = new_gcap;
}
void dnz_window::dict_grow() {
  if (gcap >= (1u << 29)) fail(DNZ_ERR_NOMEM, "more than 2^29 groups");
  dict_alloc(gcap * 2);
}
// Long-key arena.  Inserters reserve space with an atomicAdd BEFORE they know whether it fits, so after an overflow the device
// counter has run past the capacity by the bytes of every failed attempt: an upper bound of what the deferred rows need.
void dnz_window::arena_grow(uint64_t at_least) {
  uint64_t ncap = std::max<uint64_t>(arena_cap * 2, at_least);
  ncap = round_up(ncap, 1 << 20);
  if (ncap > arena.bytes) {
    DevBuf na; na.alloc(ncap);
    CK(cudaMemcpyAsync(na.p, arena.p, arena_cap, cudaMemcpyDeviceToDevice, stream));
    CK(cudaStreamSynchronize(stream));
    arena = std::move(na);
  }
  arena_cap = ncap;
}
// After a replay the arena holds what it needs: pull the logical capacity back to "used + slack" so that the upper bounds
// derived from the free space (result sizing) stay tight; the memory stays allocated and the next overflow just raises it.
void dnz_window::arena_trim() {
  const uint64_t want = round_up(arena_used_host + std::max<uint64_t>(64ull << 20, arena_used_host / 4), 1 << 20);
  if (want < arena_cap && arena_used_host <= want) arena_cap = std::max<uint64_t>(want, 1 << 20);
}

void dnz_window::parse_ctl(const CtlBlock& h) {
  if (h.ts_err) fail(DNZ_ERR_DATA, "a timestamp string does not match the format (the reference unwraps the parse error and panics)");
  if (const uint32_t xe = h.merge_err) {
    if (xe & 8u) fail(DNZ_ERR_INVALID, "pane exchange: a rank sent keys of another type than this operator's group key (every rank must group by the same key type)");
    if (xe & 0x100u) fail(DNZ_ERR_NOMEM, "exchange ring overflow: an owner's ring is smaller than one step's packets (dnz_group_config.ring_entries / ring_key_bytes)");
    fail(DNZ_ERR_NOMEM, "pane merge failed (flags %u): the dictionary / key arena of this rank is too small for the keys it owns (in exchange mode expected_groups must cover the GLOBAL key set)", xe);
  }
  n_groups_host = std::min(h.dict.n_groups, gcap);
  arena_used_host = h.dict.arena_used;
  key_bytes_total_host = h.dict.key_bytes_total;
  for (const ResultCursor& r : h.result)
    if (r.overflow) fail(DNZ_ERR_NOMEM, "result buffer overflow (internal sizing error)");
  stats.groups = n_groups_host;
}
// one small D2H + sync: every launch enqueued so far has completed, the host view becomes exact
void dnz_window::fetch_ctl() {
  h_small.reserve(sizeof(CtlBlock));
  CK(cudaMemcpyAsync(h_small.p, d_ctl.p, sizeof(CtlBlock), cudaMemcpyDeviceToHost, stream));
  CK(cudaStreamSynchronize(stream));
  const CtlBlock& h = *h_small.as<CtlBlock>();
  parse_ctl(h);
  rows_since_known = 0;
  for (int k = 0; k < 2; k++) {
    const uint64_t c = h.result[k].cursor;
    rs[k].rows = c >> 32; rs[k].bytes = c & 0xFFFFFFFFull;
  }
  for (Slot& s : slot) { s.add_rows_bound = 0; s.add_bytes_bound = 0; }
}
// upper bounds of the device counters given what has been enqueued since the host last saw them
uint32_t dnz_window::groups_bound() const {
  if (world > 1) return gcap;      // the owner's merge interns keys the host has not seen
  return (uint32_t)std::min<uint64_t>(gcap, (uint64_t)n_groups_host + (uint64_t)std::max<int64_t>(rows_since_known, 0) + 1);   // + the NULL key
}
uint64_t dnz_window::key_bytes_bound() const {
  const uint64_t fresh = groups_bound() - std::min<uint32_t>(groups_bound(), n_groups_host);
  // long keys can only be interned by launches the host has not seen complete (or by the owner's merge)
  const bool interning = world > 1 || rows_since_known > 0;
  const uint64_t arena_free = interning ? arena_cap - std::min<uint64_t>(arena_used_host, arena_cap) : 0;
  return key_bytes_total_host + fresh * INLINE_KEY + arena_free + key_width;   // + the NULL key's value (integer keys)
}

std::unique_ptr<Pane> dnz_window::new_pane(int64_t id) {
  std::unique_ptr<Pane> p;
  while (!pane_pool.empty() && !p) {
    p = std::move(pane_pool.back()); pane_pool.pop_back();
    if (p->st.bytes < (size_t)gcap * sizeof(GroupState)) p.reset();      // never reuse a pane sized for a smaller dictionary
  }
  if (!p) { p.reset(new Pane()); p->st.alloc((size_t)gcap * sizeof(GroupState)); }
  if (p->nullrows.p && p->nullrows.bytes < (size_t)gcap * 8) p->nullrows.release();
  if (p->fz.p && p->fz.bytes < (size_t)gcap * 8) p->fz.release();
  p->id = id;
  if (next_tag >= (1ull << 31)) {     // tags live in [1, 2^31) so that "newer" is a signed 32-bit difference: drop every hint, restart
    CK(launch_clear_hints(slots.as<DictSlot>(), dict_cap, stream)); stats.total_launches++;
    next_tag = 1;
  }
  p->tag = next_tag++;
  CK(cudaMemsetAsync(p->st.p, 0, (size_t)gcap * sizeof(GroupState), stream));
  ensure_side_arrays(p.get());
  if (p->nullrows.p) CK(cudaMemsetAsync(p->nullrows.p, 0, (size_t)gcap * 8, stream));
  if (p->fz.p) CK(cudaMemsetAsync(p->fz.p, 0xFF, (size_t)gcap * 8, stream));
  return p;
}
void dnz_window::ensure_side_arrays(Pane* p) {
  if (need_nullrows && !p->nullrows.p) { p->nullrows.alloc((size_t)gcap * 8); CK(cudaMemsetAsync(p->nullrows.p, 0, (size_t)gcap * 8, stream)); }
  if (need_fz && !p->fz.p) { p->fz.alloc((size_t)gcap * 8); CK(cudaMemsetAsync(p->fz.p, 0xFF, (size_t)gcap * 8, stream)); }
}
Pane* dnz_window::get_pane(int64_t id, bool create) {
  auto it = panes.find(id);
  if (it != panes.end()) return it->second.get();
  if (!create) return nullptr;
  auto p = new_pane(id);
  Pane* r = p.get();
  panes[id] = std::move(p);
  return r;
}
// A pane is dropped once the last window that covers it (start == pane start) has been emitted.  Behind a speculative launch the
// pane is parked in the slot until the launch has been verified (its emission may have to be re-issued); otherwise stream order
// alone makes the reuse safe.
void dnz_window::retire_panes(Slot* sl) {
  if (!has_wm) return;
  for (auto it = panes.begin(); it != panes.end();) {
    if (it->first * pane_ms + L <= wm) {
      if (sl) sl->retired.push_back(std::move(it->second));
      else recycle_pane(std::move(it->second));
      it = panes.erase(it);
    } else ++it;
  }
}
void dnz_window::recycle_pane(std::unique_ptr<Pane> p) {
  if (pane_pool.size() < 16) pane_pool.push_back(std::move(p));
}
// the one-batch panes of a dirty run, once the stream has finished with them
void dnz_window::release_late_panes() {
  CK(cudaStreamSynchronize(stream));
  for (auto& kv : late_panes) recycle_pane(std::move(kv.second));
  late_panes.clear();
}
// an open pane, or one that was retired behind a launch that has not been verified yet (a replay of deferred rows still needs it)
Pane* dnz_window::find_pane(int64_t id) {
  auto it = panes.find(id);
  if (it != panes.end()) return it->second.get();
  for (Slot& s : slot) for (auto& p : s.retired) if (p->id == id) return p.get();
  return nullptr;
}
std::map<int64_t, Pane*> dnz_window::pane_sources() {
  std::map<int64_t, Pane*> src;
  for (Slot& s : slot) for (auto& p : s.retired) src[p->id] = p.get();
  for (auto& kv : panes) src[kv.first] = kv.second.get();
  return src;
}

// ------------------------------------------------------------------------------------------------
// input
static const void* buf_at(const ArrowArray* a, int i) { return a->n_buffers > i ? a->buffers[i] : nullptr; }

void dnz_window::push_host(ArrowArray* batch) {
  if (!batch || !batch->release) fail(DNZ_ERR_INVALID, "released or null ArrowArray");
  if (batch->n_children != n_input_cols) fail(DNZ_ERR_INVALID, "batch has %lld columns, schema has %d", (long long)batch->n_children, n_input_cols);
  int64_t n = batch->length;
  if (n < 0) fail(DNZ_ERR_INVALID, "negative batch length");
  if (n >= (1ll << 31)) fail(DNZ_ERR_UNSUPPORTED, "batch with >= 2^31 rows");
  if (cur().rows > 0 && cur().rows + n > max_rows) seal_current();
  Slot& c = cur();
  Arena& arena_in = c.arena;
  PendingBatch pb;
  pb.d.n_rows = n; pb.d.seq = next_seq++; pb.d.flags = BATCH_BULK_OK;
  if (n > 0) {
    const int64_t po = batch->offset;
    const ArrowArray* val = batch->children[val_col];
    const ArrowArray* key = ungrouped ? val : batch->children[key_col];
    const ArrowArray* meta = ts_source == DNZ_TS_CANONICAL ? batch->children[meta_col] : nullptr;
    const ArrowArray* ts = meta ? meta->children[ts_child] : batch->children[ts_col];
    if (key->length < po + n || val->length < po + n || ts->length < po + (meta ? meta->offset : 0) + n) fail(DNZ_ERR_INVALID, "child arrays shorter than the batch");
    // page-locked sources (dnz_host_alloc / cudaHostRegister) are device-readable: queue them for the gather kernel;
    // pageable sources go through cudaMemcpyAsync (staged by the driver)
    auto enqueue_copy = [&](void* d, const void* src, size_t bytes) {
      if (!bytes) return;
      cudaPointerAttributes at{};
      bool pinned = cudaPointerGetAttributes(&at, src) == cudaSuccess && at.type == cudaMemoryTypeHost && at.devicePointer;
      if (!pinned) cudaGetLastError();
      if (pinned && bytes >= 4096) {
        uint64_t fp = c.gather.empty() ? 0 : c.gather.back().first_piece + (c.gather.back().bytes + COPY_PIECE - 1) / COPY_PIECE;
        c.gather.push_back(CopyDesc{at.devicePointer, d, (uint64_t)bytes, fp});
      }
      else { CK(cudaMemcpyAsync(d, src, bytes, cudaMemcpyHostToDevice, copy_stream)); if (!pinned) stats.h2d_pageable_bytes += (int64_t)bytes; }
      stats.h2d_bytes += (int64_t)bytes;
    };
    auto copy_in = [&](const void* src, size_t bytes) -> void* {
      void* d = arena_in.alloc(bytes);
      enqueue_copy(d, src, bytes);
      return d;
    };
    auto copy_bitmap = [&](const ArrowArray* a, int64_t eff_off, const uint8_t*& dptr, int32_t& vbit) {
      dptr = nullptr; vbit = 0;
      const uint8_t* bm = (const uint8_t*)buf_at(a, 0);
      if (!bm || a->null_count == 0) return;
      int64_t b0 = eff_off >> 3, b1 = (eff_off + n + 7) >> 3;
      dptr = (const uint8_t*)copy_in(bm + b0, (size_t)(b1 - b0));
      vbit = (int32_t)(eff_off & 7);
    };
    // timestamps
    if (ts_source == DNZ_TS_CANONICAL) {
      int64_t to = po + meta->offset + ts->offset;
      pb.d.ts = (const int64_t*)copy_in((const int64_t*)buf_at(ts, 1) + to, (size_t)n * 8);
      copy_bitmap(ts, to, pb.d.ts_valid, pb.d.ts_vbit);
      if (meta->null_count != 0 && buf_at(meta, 0)) fail(DNZ_ERR_UNSUPPORTED, "null `_streaming_internal_metadata` structs are not supported");
    } else {
      // array_to_timestamp_array (utils/time.rs:59-94): Int64 values are taken as they are (the validity bitmap is ignored there
      // too); a NULL string is unwrapped -> panic
      const int64_t to = po + ts->offset;
      if (ts_source == DNZ_TS_INT64_MILLIS) {
        pb.d.ts = (const int64_t*)copy_in((const int64_t*)buf_at(ts, 1) + to, (size_t)n * 8);
      } else if (ts_source == DNZ_TS_INT64_SECONDS) {
        const void* raw = copy_in((const int64_t*)buf_at(ts, 1) + to, (size_t)n * 8);
        int64_t* dst = (int64_t*)arena_in.alloc((size_t)n * 8);
        c.ts_jobs.push_back(TsJob{raw, nullptr, nullptr, dst, n}); c.ts_max_rows = std::max(c.ts_max_rows, n);
        pb.d.ts = dst;
      } else {
        if (ts->null_count != 0 && buf_at(ts, 0)) fail(DNZ_ERR_DATA, "NULL timestamp string (the reference unwraps it and panics)");
        const int32_t* hoff = (const int32_t*)buf_at(ts, 1) + to;
        const int32_t* doff = (const int32_t*)copy_in(hoff, (size_t)(n + 1) * 4);
        const int64_t o0 = hoff[0], o1 = hoff[n];
        uint8_t* db = (uint8_t*)arena_in.alloc((size_t)(o1 - o0) + 16);
        if (o1 > o0) enqueue_copy(db, (const uint8_t*)buf_at(ts, 2) + o0, (size_t)(o1 - o0));
        int64_t* dst = (int64_t*)arena_in.alloc((size_t)n * 8);
        c.ts_jobs.push_back(TsJob{nullptr, doff, db - o0, dst, n}); c.ts_max_rows = std::max(c.ts_max_rows, n);
        pb.d.ts = dst;
      }
    }
    // values
    int64_t vo = po + val->offset;
    pb.d.val = (const double*)copy_in((const double*)buf_at(val, 1) + vo, (size_t)n * 8);
    copy_bitmap(val, vo, pb.d.val_valid, pb.d.val_vbit);
    // keys
    if (!ungrouped && key_width) {         // integer keys: the values (one per row, naturally aligned in the arena) and the bitmap
      const int64_t ko = po + key->offset;
      pb.d.bytes = (const uint8_t*)copy_in((const uint8_t*)buf_at(key, 1) + ko * key_width, (size_t)n * key_width);
      pb.d.off = nullptr;
      copy_bitmap(key, ko, pb.d.key_valid, pb.d.key_vbit);
    } else if (!ungrouped) {
    int64_t ko = po + key->offset;
    const int32_t* hoff = (const int32_t*)buf_at(key, 1) + ko;
    pb.d.off = (const int32_t*)copy_in(hoff, (size_t)(n + 1) * 4);
    int64_t o0 = hoff[0], o1 = hoff[n];
    int64_t a0 = o0 & ~(int64_t)15;
    pb.key_bytes = o1 - o0;
    const uint8_t* hb = (const uint8_t*)buf_at(key, 2);
    uint8_t* db = (uint8_t*)arena_in.alloc((size_t)(o1 - a0) + 16);
    if (o1 > a0) enqueue_copy(db, hb + a0, (size_t)(o1 - a0));
    pb.d.bytes = db - a0;     // only [o0, o1) is ever dereferenced
    copy_bitmap(key, ko, pb.d.key_valid, pb.d.key_vbit);
    }
    c.copies = true;
  }
  pb.has_moved = true; pb.moved = *batch; batch->release = nullptr;   // moved
  c.batches.push_back(pb);
  c.rows += n;
  stats.batches_in++; stats.rows_in += n;
  if (c.rows >= max_rows) seal_current();      // full: its transfer starts now, not when the next batch happens to arrive
}

void dnz_window::push_dev(const dnz_device_batch* b, int64_t nb) {
  for (int64_t i = 0; i < nb; i++) {
    const dnz_device_batch& s = b[i];
    if (s.n_rows < 0) fail(DNZ_ERR_INVALID, "device batch %lld: negative row count", (long long)i);
    if (s.n_rows >= (1ll << 31)) fail(DNZ_ERR_UNSUPPORTED, "batch with >= 2^31 rows");
    if (s.n_rows > 0 && (!s.ts || !s.val || (!ungrouped && ((!key_width && !s.key_off) || !s.key_bytes)))) fail(DNZ_ERR_INVALID, "device batch %lld: null column pointer", (long long)i);
    if (key_width && s.key_off) fail(DNZ_ERR_INVALID, "device batch %lld: key_off must be NULL for an integer key column (key_bytes holds the values)", (long long)i);
    if (key_width && (reinterpret_cast<uintptr_t>(s.key_bytes) % (uintptr_t)key_width) != 0)
      fail(DNZ_ERR_INVALID, "device batch %lld: integer key values must be aligned to their width (%d B)", (long long)i, key_width);
    if (cur().rows > 0 && cur().rows + s.n_rows > max_rows) seal_current();
    Slot& c = cur();
    PendingBatch pb;
    pb.d.ts = s.ts; pb.d.val = s.val; pb.d.off = ungrouped ? nullptr : s.key_off; pb.d.bytes = ungrouped ? nullptr : s.key_bytes;
    pb.d.ts_valid = s.ts_valid; pb.d.val_valid = s.val_valid; pb.d.key_valid = ungrouped ? nullptr : s.key_valid;
    pb.d.n_rows = s.n_rows; pb.d.seq = next_seq++; pb.d.flags = BATCH_BULK_OK;
    pb.key_bytes = -1;
    c.batches.push_back(pb);
    c.rows += s.n_rows;
    stats.batches_in++; stats.rows_in += s.n_rows;
    if (c.rows >= max_rows) seal_current();
  }
}

// ------------------------------------------------------------------------------------------------
// pipeline
// launch the gather copy of a superbatch's pinned sources and mark the point where all its bytes are on the device
void dnz_window::finish_copies(Slot& s) {
  if (!s.copies) return;
  if (!s.gather.empty()) {
    size_t nbytes = s.gather.size() * sizeof(CopyDesc);
    s.h_copy_descs.reserve(nbytes); s.d_copy_descs.reserve(nbytes);
    memcpy(s.h_copy_descs.p, s.gather.data(), nbytes);
    CK(cudaMemcpyAsync(s.d_copy_descs.p, s.h_copy_descs.p, nbytes, cudaMemcpyHostToDevice, copy_stream));
    CK(cudaMemsetAsync(d_copy_cursor.p, 0, 4, copy_stream));
    CK(launch_gather_copy(s.d_copy_descs.as<CopyDesc>(), (uint32_t)s.gather.size(), d_copy_cursor.as<unsigned int>(), copy_stream));
    stats.total_launches++;
    s.gather.clear();
  }
  CK(cudaEventRecord(s.copy_done, copy_stream));
}

// The filling superbatch is complete: start its transfer and its tile scan, enqueue the aggregation of the superbatch sealed
// before it (whose scan results are on the host by now, so nothing waits), and move on to the next slot -- which must have been
// verified: that is the only place where the host may wait for the device, two aggregate launches behind the one it just queued.
void dnz_window::seal_current() {
  Slot& f = cur();
  if (f.batches.empty()) return;
  InProcess scope(this);
  finish_copies(f);
  launch_scan(f);
  f.state = Slot::SEALED; sealed_order.push_back(f.idx);
  while (sealed_order.size() > 1) launch_slot(slot[sealed_order.front()]);
  if ((world > 1 && !fused) || (cfg.flags & DNZ_FLAG_SYNCHRONOUS)) while (!sealed_order.empty()) launch_slot(slot[sealed_order.front()]);
  const int next = (fill + 1) % PIPELINE_SLOTS;
  if (slot[next].state == Slot::SEALED) launch_slot(slot[next]);
  if (slot[next].state == Slot::LAUNCHED) { while (!launched_order.empty() && slot[next].state == Slot::LAUNCHED) verify(slot[launched_order.front()]); }
  fill = next; slot[next].state = Slot::FILLING;
}

// enqueue everything that has been pushed (no host wait for the results)
void dnz_window::process_pending() {
  InProcess scope(this);
  if (!cur().batches.empty()) seal_current();
  while (!sealed_order.empty()) launch_slot(slot[sealed_order.front()]);
}
// ... and make the host view exact: every launch verified, deferred rows replayed, input batches released
void dnz_window::drain() {
  InProcess scope(this);
  while (!sealed_order.empty()) launch_slot(slot[sealed_order.front()]);
  while (!launched_order.empty()) verify(slot[launched_order.front()]);
}

// Batch descriptors + tile scan (RecordBatchWatermark::try_from per batch, byte ranges per tile), asynchronously: the
// results land in the slot's pinned buffers and `scan_done` fires when they are readable.
void dnz_window::launch_scan(Slot& s) {
  const size_t nb = s.batches.size();
  s.bds.resize(nb); s.n_tiles = 0; s.scanned = true;
  for (size_t i = 0; i < nb; i++) { s.bds[i] = s.batches[i].d; s.bds[i].tile0 = s.n_tiles; s.n_tiles += (s.bds[i].n_rows + TILE - 1) / TILE; }
  if (s.n_tiles == 0) { s.ts_jobs.clear(); return; }            // only empty batches: no trigger (grouped_window_agg_stream.rs:331,:343-345)
  // the scan picks the LAST batch with tile0 <= t: empty batches in the middle share their successor's tile0 and are
  // never chosen; trailing empties get a tile0 past the end
  for (size_t i = nb; i-- > 0;) { if (s.bds[i].n_rows == 0) s.bds[i].tile0 = s.n_tiles + 1; else break; }
  s.d_batches.reserve(nb * sizeof(BatchDesc)); s.d_tiles.reserve((size_t)s.n_tiles * sizeof(TileDesc)); s.d_minmax.reserve(nb * sizeof(BatchMinMax));
  s.h_batches.reserve(nb * sizeof(BatchDesc)); s.h_minmax.reserve(nb * sizeof(BatchMinMax));
  memcpy(s.h_batches.p, s.bds.data(), nb * sizeof(BatchDesc));
  if (s.copies) CK(cudaStreamWaitEvent(stream, s.copy_done, 0));
  if (!s.ts_jobs.empty()) {           // canonical timestamps from the raw column: the step before the path (utils/time.rs:59-94)
    const size_t jb = s.ts_jobs.size() * sizeof(TsJob);
    s.h_ts_jobs.reserve(jb); s.d_ts_jobs.reserve(jb);
    memcpy(s.h_ts_jobs.p, s.ts_jobs.data(), jb);
    CK(cudaMemcpyAsync(s.d_ts_jobs.p, s.h_ts_jobs.p, jb, cudaMemcpyHostToDevice, stream));
    CK(launch_ts_convert(s.d_ts_jobs.as<TsJob>(), (int)s.ts_jobs.size(), s.ts_max_rows, ts_source, ts_fmt, &ctl()->ts_err, stream));
    stats.total_launches++;
    s.ts_jobs.clear(); s.ts_max_rows = 0;
  }
  CK(cudaMemcpyAsync(s.d_batches.p, s.h_batches.p, nb * sizeof(BatchDesc), cudaMemcpyHostToDevice, stream));
  bool allow_fast = !(cfg.flags & DNZ_FLAG_FORCE_GENERIC);
  CK(launch_tile_scan(s.d_batches.as<BatchDesc>(), (int64_t)nb, s.n_tiles, pane_ms, s.d_tiles.as<TileDesc>(), s.d_minmax.as<BatchMinMax>(), allow_fast, stream));
  stats.total_launches += 2;
  CK(cudaMemcpyAsync(s.h_minmax.p, s.d_minmax.p, nb * sizeof(BatchMinMax), cudaMemcpyDeviceToHost, stream));
  CK(cudaEventRecord(s.scan_done, stream));
}

// Everything a steady-state pass needs is allocated when the operator is created (cudaMalloc / cudaMallocHost cost
// milliseconds and must stay out of the per-batch path).
void dnz_window::prealloc() {
  const size_t nb_max = 4096 + (size_t)(max_rows / 8192), nt_max = (size_t)(max_rows / TILE) + nb_max;
  for (Slot& s : slot) {
    s.d_batches.reserve(nb_max * sizeof(BatchDesc)); s.d_tiles.reserve(nt_max * sizeof(TileDesc)); s.d_minmax.reserve(nb_max * sizeof(BatchMinMax));
    s.h_batches.reserve(nb_max * sizeof(BatchDesc)); s.h_minmax.reserve(nb_max * sizeof(BatchMinMax));
    s.d_copy_descs.reserve(8192 * sizeof(CopyDesc)); s.h_copy_descs.reserve(8192 * sizeof(CopyDesc));
    s.d_ptrs.reserve(7 * 1024 * sizeof(void*)); s.h_ptrs.reserve((size_t)7 * 1024 * sizeof(void*));
    s.d_defer[0].reserve((size_t)std::max<int64_t>(max_rows, 1) * sizeof(DeferEntry));
  }
  d_copy_cursor.alloc(64);
  h_small.reserve(sizeof(CtlBlock) + 64);
  // low cardinality: the per-CTA private pane copies (AggParams::priv) are needed by the first launch already
  if (gcap <= 8192) d_priv.reserve(256ull << 20);
  for (int i = 0; i < std::max(panes_per_window + 2, 8) && i < 16; i++) pane_pool.push_back(new_pane(0));
  {   // room for a few windows' worth of rows; grows on demand (one poll is limited to 2 GiB of key bytes by the 32-bit Utf8 offsets)
    // (upper bounds are reserved per emission: windows x group capacity, for every launch in flight and every unconsumed window)
    const uint64_t rows0 = std::min<uint64_t>((uint64_t)gcap * 24, 48ull << 20);
    for (wr = 1; wr >= 0; wr--) ensure_result_capacity(rows0, std::min<uint64_t>(rows0 * 16, (1ull << 31) - (1ull << 20)));
    wr = 0;
  }
}

// ---- runs: maximal sequences of batches without late rows are aggregated by ONE launch; a batch that contains rows for an
// already emitted window ("dirty") is aggregated alone so that the re-opened windows hold exactly its rows.  A run is also cut
// where its pane span would exceed the pane table (an idle gap in the stream), so the limit applies per batch, not per launch.
constexpr int64_t MAX_RUN_PANES = 1 << 16;
void dnz_window::plan_runs(Slot& s, const std::vector<BatchMinMax>& mm, std::vector<Run>& runs) {
  const size_t nb = s.batches.size();
  bool cur_has_wm = world > 1 ? has_lwm : has_wm; int64_t cur_wm = world > 1 ? lwm : wm;
  size_t run_start = nb; int64_t run_wm_after = 0, run_pmin = 0, run_pmax = 0;
  for (size_t i = 0; i < nb; i++) {
    if (s.bds[i].n_rows == 0) continue;
    const int64_t mn = mm[i].ts_min;
    const int64_t bp0 = floor_div(mn, pane_ms), bp1 = floor_div(mm[i].ts_max, pane_ms);
    if (bp1 - bp0 + 1 > MAX_RUN_PANES) fail(DNZ_ERR_UNSUPPORTED, "batch %lld spans %lld panes (timestamps too sparse); limit %lld", (long long)s.bds[i].seq, (long long)(bp1 - bp0 + 1), (long long)MAX_RUN_PANES);
    const int64_t first_pane_end = (bp0 + 1) * pane_ms;
    bool dirty = cur_has_wm && first_pane_end <= cur_wm;
    const int64_t new_wm = (!cur_has_wm || cur_wm <= mn) ? mn : cur_wm;     // process_watermark (:255-266)
    if (dirty && world > 1 && first_pane_end <= (exported_pane_upto == INT64_MIN ? INT64_MIN : (exported_pane_upto + 1) * pane_ms))
      fail(DNZ_ERR_UNSUPPORTED, "batch %lld is late for a pane that was already exchanged (exchange mode needs in-order input)", (long long)s.bds[i].seq);
    if (world > 1) dirty = false;      // nothing has been emitted locally: late rows simply join their (still local) panes
    if (dirty) {
      if (run_start != nb) { runs.push_back(Run{run_start, i, false, 0, run_wm_after}); run_start = nb; }
      runs.push_back(Run{i, i + 1, true, cur_wm, new_wm});
      stats.late_batches++;
    } else {
      if (run_start != nb && std::max(run_pmax, bp1) - std::min(run_pmin, bp0) + 1 > MAX_RUN_PANES) {
        runs.push_back(Run{run_start, i, false, 0, run_wm_after}); run_start = nb;
      }
      if (run_start == nb) { run_start = i; run_pmin = bp0; run_pmax = bp1; }
      else { run_pmin = std::min(run_pmin, bp0); run_pmax = std::max(run_pmax, bp1); }
      run_wm_after = new_wm;
    }
    cur_has_wm = true; cur_wm = new_wm;
  }
  if (run_start != nb) runs.push_back(Run{run_start, nb, false, 0, run_wm_after});
}

dnz_window::RunGeom dnz_window::run_geometry(Slot& s, const std::vector<BatchMinMax>& mm, const Run& r) {
  RunGeom g;
  int64_t acc = 0; int64_t fast = 0, generic = 0;
  for (size_t i = 0; i < r.b1; i++) {
    if (i == r.b0) g.t0 = acc;
    acc += (s.bds[i].n_rows + TILE - 1) / TILE;
  }
  g.t1 = acc;
  for (size_t i = r.b0; i < r.b1; i++) {
    const BatchMinMax& b = mm[i];
    const int64_t nr = s.bds[i].n_rows;
    if (nr == 0) continue;
    g.rows += nr; g.alg_bytes += (key_width ? 16.0 + key_width : 20.0) * nr + (double)b.key_bytes;    // see dnz_stats
    fast += b.n_fast; generic += b.n_tiles - b.n_fast;
    if (s.bds[i].val_valid) g.val_nulls = true;
    if (b.n_valid == 0) continue;
    g.pmin = std::min(g.pmin, floor_div(b.ts_min, pane_ms)); g.pmax = std::max(g.pmax, floor_div(b.ts_max, pane_ms));
  }
  stats.fast_tiles += fast; stats.generic_tiles += generic;
  return g;
}

// panes touched by the run (from the per-batch timestamp ranges of the tile scan)
void dnz_window::prepare_panes(Slot& s, const std::vector<BatchMinMax>& mm, const Run& r, const RunGeom& g) {
  if (g.pmin > g.pmax) return;
  const int64_t np = g.pmax - g.pmin + 1;
  if (g.val_nulls && !need_nullrows) { need_nullrows = true; for_each_live_pane([&](Pane* p) { ensure_side_arrays(p); }); }
  std::vector<uint8_t> touched((size_t)np, 0);
  for (size_t i = r.b0; i < r.b1; i++) {
    const BatchMinMax& b = mm[i];
    if (s.bds[i].n_rows == 0 || b.n_valid == 0) continue;
    for (int64_t p = floor_div(b.ts_min, pane_ms); p <= floor_div(b.ts_max, pane_ms); p++) touched[(size_t)(p - g.pmin)] = 1;
  }
  for (int64_t p = g.pmin; p <= g.pmax; p++) {
    if (!touched[(size_t)(p - g.pmin)]) continue;
    const bool need_main = !r.dirty || p * pane_ms + L > r.horizon;             // some covering window is still open
    const bool need_late = r.dirty && (p + 1) * pane_ms <= r.horizon;           // some covering window was already emitted
    if (need_main) get_pane(p, true);
    if (need_late) late_panes[p] = new_pane(p);
  }
}

// The pane table of panes [p0, p1]: its 7 x n_panes pointer arrays (PaneTable's, back to back) are staged at `hp` and copied to
// `dp` in stream order.  panes(p) names the main and the late pane of id p (either may be null).  The kernels update the side
// arrays of every pane in the table, so those are made to exist first.
PaneTable dnz_window::upload_pane_table(void** hp, char* dp, int64_t p0, int64_t p1, const PaneLookup& panes) {
  const int64_t np = p1 - p0 + 1;
  const size_t pb = (size_t)np * sizeof(void*);
  for (int64_t p = p0; p <= p1; p++) {
    const size_t k = (size_t)(p - p0);
    const std::pair<Pane*, Pane*> ml = panes(p);
    Pane* m = ml.first; Pane* l = ml.second;
    if (m) ensure_side_arrays(m);
    if (l) ensure_side_arrays(l);
    hp[0 * np + k] = m ? m->st.p : nullptr; hp[1 * np + k] = l ? l->st.p : nullptr;
    hp[2 * np + k] = m ? m->nullrows.p : nullptr; hp[3 * np + k] = l ? l->nullrows.p : nullptr;
    hp[4 * np + k] = m ? m->fz.p : nullptr; hp[5 * np + k] = l ? l->fz.p : nullptr;
    hp[6 * np + k] = reinterpret_cast<void*>((uintptr_t)(m ? (m->tag & 0xFFFFFFFFull) : 0));
  }
  CK(cudaMemcpyAsync(dp, hp, 7 * pb, cudaMemcpyHostToDevice, stream));
  PaneTable t;
  t.pane0 = p0; t.n_panes = (int32_t)np; t.pad = 0; t.pane_ms = pane_ms;
  t.main = (GroupState* const*)(dp + 0 * pb); t.late = (GroupState* const*)(dp + 1 * pb);
  t.nullrows_main = (unsigned long long* const*)(dp + 2 * pb); t.nullrows_late = (unsigned long long* const*)(dp + 3 * pb);
  t.fz_main = (unsigned long long* const*)(dp + 4 * pb); t.fz_late = (unsigned long long* const*)(dp + 5 * pb);
  t.tag_main = (const unsigned long long*)(dp + 6 * pb);
  return t;
}

// pane pointer table + launch parameters of one aggregate / replay pass over the run
AggParams dnz_window::build_agg_params(Slot& s, const RunGeom& g, bool dirty, int64_t horizon, int out_list) {
  const size_t pb = (size_t)(g.pmax - g.pmin + 1) * sizeof(void*);
  s.h_ptrs.reserve(7 * pb); s.d_ptrs.reserve(7 * pb);
  AggParams P;
  P.panes = upload_pane_table(s.h_ptrs.as<void*>(), s.d_ptrs.as<char>(), g.pmin, g.pmax, [&](int64_t p) {
    auto lit = late_panes.find(p);
    return std::make_pair((!dirty || p * pane_ms + L > horizon) ? find_pane(p) : nullptr, lit == late_panes.end() ? nullptr : lit->second.get());
  });
  SlotCtl& sc = ctl()->slot[s.idx];
  CK(cudaMemsetAsync(&sc, 0, offsetof(SlotCtl, emit_blocked), stream));        // deferred-row counter, flags, tile counter (not the emit-blocked flag)
  P.batches = s.d_batches.as<BatchDesc>(); P.tiles = s.d_tiles.as<TileDesc>(); P.tile_begin = g.t0; P.tile_end = g.t1;
  P.dict = dict_view();
  P.flags = ((cfg.flags & DNZ_FLAG_NO_HINTS) ? AGG_NO_HINTS : 0) | ((cfg.flags & DNZ_FLAG_NO_QUEUE) ? AGG_NO_QUEUE : 0) |
            ((cfg.flags & DNZ_FLAG_SCALAR_PROBE) ? AGG_SCALAR_PROBE : 0) | ((cfg.flags & DNZ_FLAG_STAGE_TS) ? AGG_STAGE_TS : 0);
  const size_t defer_cap = (size_t)std::max<int64_t>(g.rows, 1);
  s.d_defer[out_list].reserve(defer_cap * sizeof(DeferEntry));
  P.defer.entries = s.d_defer[out_list].as<DeferEntry>();
  P.defer.count = &sc.defer_count; P.defer.cap = defer_cap;
  P.defer.flags = &sc.defer_flags;
  P.tile_counter = &sc.tile_counter;
  P.priv = nullptr; P.priv_groups = 0;
  return P;
}

void dnz_window::launch_aggregate_pass(Slot& s, const RunGeom& g, AggParams& P, bool dirty) {
  // low cardinality: private pane copies per CTA (see AggParams::priv)
  const int64_t np = g.pmax - g.pmin + 1;
  const int agg_grid = aggregate_grid(g.t1 - g.t0, sm_count);
  const size_t priv_bytes = (size_t)agg_grid * (size_t)np * gcap * sizeof(GroupState);
  const bool use_priv = !ungrouped && !dirty && gcap <= 8192 && priv_bytes <= (256ull << 20) && !(cfg.flags & (DNZ_FLAG_FORCE_GENERIC | DNZ_FLAG_NO_PRIVATE));
  if (use_priv) {
    d_priv.reserve(priv_bytes);
    CK(cudaMemsetAsync(d_priv.p, 0, priv_bytes, stream));
    P.priv = d_priv.as<GroupState>(); P.priv_groups = gcap;
  }
  s.timed = (cfg.flags & DNZ_FLAG_KERNEL_TIMING) != 0; s.alg_bytes = g.alg_bytes;
  if (s.timed) CK(cudaEventRecord(s.ev0, stream));
  if (ungrouped) CK(launch_aggregate_ungrouped(P, sm_count, stream));
  else if (cfg.flags & DNZ_FLAG_FORCE_GENERIC) CK(launch_aggregate_generic(P, key_width, sm_count, stream));
  else CK(launch_aggregate(P, key_width, sm_count, stream));
  if (use_priv) { CK(launch_merge_private(P, agg_grid, stream)); stats.total_launches++; }
  if (s.timed) CK(cudaEventRecord(s.ev1, stream));
  stats.agg_launches++; stats.total_launches++;
  rows_since_known += g.rows;
}

// Rows the aggregate pass could not apply (a table was full, a side array was missing) sit in the slot's deferred-row list.
// Grow what was too small and replay exactly those rows until none is left.  Called with the stream idle and
// defer_count_host / defer_flags_host describing the slot's list 0.
void dnz_window::resolve_deferred(Slot& s, const RunGeom& g, bool dirty, int64_t horizon) {
  int in_list = 0; uint64_t n_in = defer_count_host; uint32_t flags = defer_flags_host;
  for (int iter = 0; n_in > 0; iter++) {
    if (iter > 64) fail(DNZ_ERR_NOMEM, "deferred rows did not converge");
    if (flags & DEFER_LIST_OVERFLOW) fail(DNZ_ERR_NOMEM, "deferred-row list overflow");
    stats.deferred_rows += (int64_t)n_in;
    if (flags & DEFER_GROUPS_FULL) {
      // The device counter ran past the table's capacity; ids >= gcap were never handed out, so it is pulled back to gcap.  A
      // launch queued behind a speculative one may have overflowed a table that the replay of the earlier launch has grown
      // since: then the counter is already below gcap and counts exactly the ids handed out; raising it to gcap would skip ids.
      CK(cudaMemcpyAsync(h_small.p, &ctl()->dict.n_groups, 4, cudaMemcpyDeviceToHost, stream));
      CK(cudaStreamSynchronize(stream));
      const uint32_t clamp = std::min(*h_small.as<uint32_t>(), gcap);
      CK(cudaMemcpyAsync(&ctl()->dict.n_groups, &clamp, 4, cudaMemcpyHostToDevice, stream));
      CK(cudaStreamSynchronize(stream));
      dict_grow();
    }
    if (flags & DEFER_ARENA_FULL) {
      // the counter ran past the capacity by the bytes of every failed reservation (>= what the deferred rows need, and
      // never more than the key bytes of the run): pull it back to the capacity (the tail gap stays unused) and grow by that
      const uint64_t over = arena_used_host > arena_cap ? arena_used_host - arena_cap : 0;
      const uint64_t old_cap = arena_cap;
      CK(cudaMemcpyAsync(&ctl()->dict.arena_used, &old_cap, 8, cudaMemcpyHostToDevice, stream));
      CK(cudaStreamSynchronize(stream));
      arena_grow(arena_cap + std::min<uint64_t>(over, (uint64_t)g.alg_bytes) + (1 << 20));
    }
    if (flags & DEFER_NEED_FZ) need_fz = true;
    if (flags & DEFER_NEED_NULLROWS) need_nullrows = true;
    if (flags & (DEFER_NEED_FZ | DEFER_NEED_NULLROWS)) for_each_live_pane([&](Pane* p) { ensure_side_arrays(p); });
    const int out_list = in_list ^ 1;
    AggParams P = build_agg_params(s, g, dirty, horizon, out_list);
    CK(launch_deferred(P, key_width, s.d_defer[in_list].as<DeferEntry>(), n_in, stream));   // replays the rows of the previous pass
    stats.total_launches++;
    fetch_ctl();
    const SlotCtl& h = h_small.as<CtlBlock>()->slot[s.idx];
    n_in = h.defer_count; flags = h.defer_flags;
    in_list = out_list;
  }
  arena_trim();
}

// Enqueues the aggregate launch of one run: its panes, its pane table and its parameters.  Returns the run's geometry; nothing
// is launched for a run without tiles (t1 <= t0) or without a valid timestamp (pmin > pmax).
dnz_window::RunGeom dnz_window::enqueue_run(Slot& s, const std::vector<BatchMinMax>& mm, const Run& r) {
  const RunGeom g = run_geometry(s, mm, r);
  if (g.t1 <= g.t0 || g.pmin > g.pmax) return g;
  prepare_panes(s, mm, r, g);
  g_tr.mark("panes");
  AggParams P = build_agg_params(s, g, r.dirty, r.horizon, 0);
  launch_aggregate_pass(s, g, P, r.dirty);
  g_tr.mark("agg_launch");
  return g;
}

// ---- process_watermark + trigger_windows of one run.  `gate`: the slot whose launch has not been verified yet, emission is
// gated on the device (see emit_windows); nullptr: the run's rows have all been applied, emission is not gated.
void dnz_window::advance_and_emit(const std::vector<BatchMinMax>& mm, const Run& r, Slot* gate) {
  if (world > 1) { if (!has_lwm || lwm <= r.wm_after) lwm = r.wm_after; has_lwm = true; }   // emission follows the GLOBAL watermark
  else if (ungrouped) {
    ungrouped_emit_run(gate, &mm, &r, 0);
    if (r.dirty) release_late_panes();
  } else {
    if (r.dirty) {
      // windows that were already emitted (end <= horizon) and received rows from this batch are re-opened and emitted
      // again immediately with ONLY this batch's rows (§8a-3)
      emit_closed(late_panes, INT64_MIN, r.horizon, nullptr);
      release_late_panes();
    }
    emit_normal(r.wm_after, gate);
  }
  g_tr.mark("emit");
}

void dnz_window::collect_kernel_time(Slot& s) {
  if (!s.timed) return;
  float ms = 0; CK(cudaEventElapsedTime(&ms, s.ev0, s.ev1)); stats.agg_kernel_ms += ms; stats.agg_algorithmic_bytes += s.alg_bytes; s.timed = false;
}

// Aggregates one run and triggers, waiting for the device after the launch (late batches, several runs in one superbatch,
// exchange mode): the path the speculative one falls back to.
void dnz_window::execute_run_sync(Slot& s, const std::vector<BatchMinMax>& mm, const Run& r) {
  const RunGeom g = enqueue_run(s, mm, r);
  if (g.t1 <= g.t0) return;
  if (g.pmin <= g.pmax) {
    fetch_ctl();
    g_tr.mark("agg_wait");
    collect_kernel_time(s);
    const SlotCtl& h = h_small.as<CtlBlock>()->slot[s.idx];
    defer_count_host = h.defer_count; defer_flags_host = h.defer_flags;
    if (defer_count_host) resolve_deferred(s, g, r.dirty, r.horizon);
  }
  g_tr.mark("post_agg");
  advance_and_emit(mm, r, nullptr);
}

// The host has the scan results of a sealed superbatch: replay the reference's per-batch watermark rule over its batches, enqueue
// the aggregation and the emission of every window it closes.  The common case -- one run, nothing late -- is enqueued without
// waiting for anything: emission is gated ON THE DEVICE by the deferred-row counters, and verify() inspects the outcome later.
void dnz_window::launch_slot(Slot& s) {
  if (s.state != Slot::SEALED) return;
  sealed_order.erase(std::find(sealed_order.begin(), sealed_order.end(), s.idx));
  s.speculative = false; s.emit_starts.clear(); s.add_rows_bound = s.add_bytes_bound = 0; s.rows_launched = 0; s.timed = false;
  g_tr.mark("pre");
  if (s.n_tiles > 0) {
    CK(cudaEventSynchronize(s.scan_done));
    g_tr.mark("scan_wait");
    const size_t nb = s.batches.size();
    std::vector<BatchMinMax> mm(s.h_minmax.as<BatchMinMax>(), s.h_minmax.as<BatchMinMax>() + nb);
    // ---- validation: inputs the reference panics on
    for (size_t i = 0; i < nb; i++) {
      if (s.bds[i].n_rows == 0) continue;
      if (mm[i].n_valid == 0) fail(DNZ_ERR_DATA, "batch %lld: all-null canonical_timestamp (the reference unwraps None and panics)", (long long)s.bds[i].seq);
      if (mm[i].ts_min < 0 || (S > 0 && mm[i].ts_min - L < 0)) fail(DNZ_ERR_DATA, "batch %lld: timestamp before epoch (+window): the reference panics in duration_since(UNIX_EPOCH)", (long long)s.bds[i].seq);
    }
    std::vector<Run> runs;
    plan_runs(s, mm, runs);
    const bool speculative = (world == 1 || fused) && runs.size() == 1 && !runs[0].dirty && !(cfg.flags & DNZ_FLAG_SYNCHRONOUS);
    if (!speculative) while (!launched_order.empty()) verify(slot[launched_order.front()]);
    if (res_consumed) reset_results();
    rotate_result_sets();
    if (speculative) {
      const Run& r = runs[0];
      const RunGeom g = enqueue_run(s, mm, r);
      if (g.t1 > g.t0) {
        if (g.pmin <= g.pmax) { s.speculative = true; s.t0 = g.t0; s.t1 = g.t1; s.pmin = g.pmin; s.pmax = g.pmax; s.rows_launched = g.rows; }
        advance_and_emit(mm, r, &s);
      }
    } else {
      for (const Run& r : runs) execute_run_sync(s, mm, r);
    }
  }
  CK(cudaMemcpyAsync(s.snap.p, d_ctl.p, sizeof(CtlBlock), cudaMemcpyDeviceToHost, stream));
  CK(cudaEventRecord(s.done, stream));
  s.state = Slot::LAUNCHED; launched_order.push_back(s.idx);
  g_tr.flush("superbatch");
}

// Inspect the snapshot taken behind a slot's launches (waits for it if it has not been written yet).
void dnz_window::verify(Slot& s) {
  if (s.state != Slot::LAUNCHED) return;
  CK(cudaEventSynchronize(s.done));
  const CtlBlock& h = *s.snap.as<CtlBlock>();
  parse_ctl(h);
  // what later launches may have added on top of this snapshot
  rows_since_known = 0;
  bool later = false;
  for (int i : launched_order) { if (i == s.idx) { later = true; continue; } if (later) rows_since_known += slot[i].rows_launched; }
  for (int k = 0; k < 2; k++) {
    const uint64_t c = h.result[k].cursor;
    uint64_t rows = c >> 32, bytes = c & 0xFFFFFFFFull;
    later = false;
    for (int i : launched_order) { if (i == s.idx) { later = true; continue; } if (later && slot[i].emit_set == k) { rows += slot[i].add_rows_bound; bytes += slot[i].add_bytes_bound; } }
    rs[k].rows = rows; rs[k].bytes = bytes;
  }
  collect_kernel_time(s);
  if (s.speculative) {
    const SlotCtl& hs = h.slot[s.idx];
    defer_count_host = hs.defer_count; defer_flags_host = hs.defer_flags;
    bool blocked = hs.emit_blocked != 0;
    if (defer_count_host && world > 1)
      fail(DNZ_ERR_NOMEM, "fused exchange: a table overflowed while launches were in flight (%llu rows deferred); size expected_groups for the GLOBAL key set", (unsigned long long)defer_count_host);
    if (defer_count_host) {
      // rare: a table was too small.  Let everything that is enqueued finish (emission behind this launch -- and behind later
      // ones -- found the gate closed and did nothing), replay the deferred rows, then issue the emission again.
      CK(cudaStreamSynchronize(stream));
      RunGeom g; g.t0 = s.t0; g.t1 = s.t1; g.pmin = s.pmin; g.pmax = s.pmax; g.rows = s.rows_launched; g.alg_bytes = s.alg_bytes;
      resolve_deferred(s, g, false, 0);
      blocked = true;
    }
    if (blocked) {
      CK(cudaMemsetAsync(&ctl()->slot[s.idx].emit_blocked, 0, 4, stream));
      if (!s.emit_starts.empty()) emit_windows(s.emit_starts, pane_sources(), nullptr);
    }
  }
  release_slot(s);
}

// verify every slot whose launches have completed, oldest first (never waits)
void dnz_window::verify_completed() {
  while (!launched_order.empty() && cudaEventQuery(slot[launched_order.front()].done) == cudaSuccess) verify(slot[launched_order.front()]);
  cudaGetLastError();
}

void dnz_window::release_slot(Slot& s) {
  if (s.copies) cudaEventSynchronize(s.copy_done);
  for (auto& pb : s.batches) if (pb.has_moved && pb.moved.release) pb.moved.release(&pb.moved);
  s.batches.clear(); s.gather.clear(); s.ts_jobs.clear(); s.ts_max_rows = 0; s.rows = 0; s.copies = false; s.arena.reset(); s.scanned = false; s.n_tiles = 0;
  for (auto& p : s.retired) recycle_pane(std::move(p));
  s.retired.clear(); s.emit_starts.clear(); s.speculative = false; s.add_rows_bound = s.add_bytes_bound = 0; s.rows_launched = 0;
  auto it = std::find(launched_order.begin(), launched_order.end(), s.idx);
  if (it != launched_order.end()) launched_order.erase(it);
  s.state = Slot::FREE;
}

// the windows with a pane in `ps` whose end lies in (end_after, end_upto], emitted from the panes of `ps`
void dnz_window::emit_closed(const PaneMap& ps, int64_t end_after, int64_t end_upto, Slot* gate) {
  std::set<int64_t> starts;
  for (auto& kv : ps)
    for (int j = 0; j < panes_per_window; j++) {
      int64_t s = (kv.first - j) * pane_ms;
      if (s >= 0 && s + L <= end_upto && s + L > end_after) starts.insert(s);
    }
  std::map<int64_t, Pane*> src;
  for (auto& kv : ps) src[kv.first] = kv.second.get();
  emit_windows(std::vector<int64_t>(starts.begin(), starts.end()), src, gate);
}

void dnz_window::emit_normal(int64_t wm_new, Slot* gate) {
  if (!has_wm || wm <= wm_new) { wm = wm_new; has_wm = true; }
  emit_closed(panes, emitted_upto, wm, gate);
  emitted_upto = std::max(emitted_upto, wm);
  retire_panes(gate);
}

// One k_emit launch per window: combine its panes, apply the fused FilterExec predicate, compact.  `gate` (nullptr: not gated):
// the launches do nothing (and raise that slot's emit-blocked flag) when any pipeline slot holds deferred rows at the time they run.
void dnz_window::emit_windows(const std::vector<int64_t>& starts, const std::map<int64_t, Pane*>& src, Slot* gate) {
  if (starts.empty()) return;
  uint32_t ng = groups_bound();
  if (ng == 0) return;
  uint64_t add_rows = (uint64_t)starts.size() * ng, add_bytes = (uint64_t)starts.size() * key_bytes_bound();
  if (R().bytes + add_bytes >= (1ull << 31)) {       // a bound per window adds up over thousands of windows: make it exact first
    fetch_ctl();                                     // every enqueued launch done: no key can be interned before these emits
    ng = groups_bound();
    add_rows = (uint64_t)starts.size() * ng; add_bytes = (uint64_t)starts.size() * key_bytes_bound();
  }
  ensure_result_capacity(add_rows, add_bytes);
  for (int64_t s : starts) {
    EmitParams E; memset(&E, 0, sizeof E);
    int64_t p0 = s / pane_ms; int k = 0;
    for (int j = 0; j < panes_per_window; j++) {
      auto it = src.find(p0 + j);
      if (it == src.end()) continue;
      E.panes[k] = it->second->st.as<GroupState>();
      E.nullrows[k] = it->second->nullrows.as<unsigned long long>();
      E.fz[k] = it->second->fz.as<unsigned long long>();
      k++;
    }
    if (k == 0) continue;
    E.n_panes = k; E.has_filter = cfg.has_filter;
    E.filter_col = cfg.has_filter ? aggs[cfg.filter_agg].kind : 0; E.filter_op = cfg.filter_op; E.filter_lit = cfg.filter_literal;
    E.wstart = s; E.wend = s + L; E.n_groups = ng; E.key_width = key_width; E.rank = rank; E.world = world;
    E.dict = dict_view();
    E.gate = gate ? ctl()->slot : nullptr;
    E.blocked = gate ? &ctl()->slot[gate->idx].emit_blocked : nullptr;
    E.out.key_off = R().key_off.as<int32_t>(); E.out.key_bytes = R().key_bytes.as<uint8_t>(); E.out.key_valid = R().key_valid.as<uint8_t>();
    E.out.count = R().count.as<int64_t>(); E.out.mn = R().mn.as<double>(); E.out.mx = R().mx.as<double>(); E.out.avg = R().avg.as<double>();
    E.out.sum = R().sum.as<double>(); E.out.agg_valid = R().agg_valid.as<uint8_t>(); E.out.wstart = R().wstart.as<int64_t>(); E.out.wend = R().wend.as<int64_t>();
    E.out.cursor = &ctl()->result[wr].cursor; E.out.row_cap = R().row_cap; E.out.byte_cap = R().byte_cap;
    E.out.overflow = &ctl()->result[wr].overflow;
    CK(launch_emit(E, stream));
    stats.total_launches++; stats.windows_emitted++;
  }
  R().rows += add_rows; R().bytes += add_bytes;
  if (gate) {
    gate->emit_starts.insert(gate->emit_starts.end(), starts.begin(), starts.end());
    gate->add_rows_bound += add_rows; gate->add_bytes_bound += add_bytes; gate->emit_set = wr;
  }
  snapshot_results();
}

// ------------------------------------------------------------------------------------------------
// checkpoint / restore (include/dnz_gpu.h)
namespace {
struct CkptHeader {
  char magic[8];                 // "DNZCKPT1"
  int64_t window_ms, slide_ms; int32_t n_aggs, flags;          // flags: 1 has_wm, 2 need_nullrows, 4 need_fz, 8 has_lwm,
                                                               //   bits 4-7 the key type (KEY_TYPES: 0 = Utf8)
  int64_t wm, emitted_upto, next_seq, lwm, exported_pane_upto;
  uint32_t n_groups, null_gid_plus1; uint64_t arena_used, key_bytes_total;
  int64_t n_panes;
  // followed by: GidKey[n_groups], arena bytes[round8(arena_used)], then per pane
  //   { int64 id; int64 has_nullrows; int64 has_fz; GroupState[n_groups]; u64 nullrows[n_groups] (if); u64 fz[n_groups] (if) }
};
}  // namespace

void dnz_window::checkpoint(std::vector<char>& blob) {
  if (ungrouped) fail(DNZ_ERR_UNSUPPORTED, "checkpoint of an ungrouped window is not implemented");
  process_pending(); drain();
  fetch_ctl();
  for (auto& r : rs) if (r.rows > r.exp_rows) fail(DNZ_ERR_INVALID, "checkpoint with emitted rows that have not been polled");
  CkptHeader H; memset(&H, 0, sizeof H);
  memcpy(H.magic, "DNZCKPT1", 8);
  H.window_ms = L; H.slide_ms = S; H.n_aggs = (int32_t)aggs.size();
  H.flags = (has_wm ? 1 : 0) | (need_nullrows ? 2 : 0) | (need_fz ? 4 : 0) | (has_lwm ? 8 : 0) | (key_type << 4);      // Utf8 (0): the blob is what it was before integer keys
  H.wm = wm; H.emitted_upto = emitted_upto; H.next_seq = next_seq; H.lwm = lwm; H.exported_pane_upto = exported_pane_upto;
  H.n_groups = n_groups_host; H.null_gid_plus1 = h_small.as<CtlBlock>()->dict.null_gid;
  H.arena_used = std::min<uint64_t>(arena_used_host, arena_cap); H.key_bytes_total = key_bytes_total_host;
  H.n_panes = (int64_t)panes.size();
  const size_t ng = H.n_groups, ab = round_up(H.arena_used, 8);
  size_t total = sizeof H + ng * sizeof(GidKey) + ab;
  for (auto& kv : panes) total += 24 + ng * sizeof(GroupState) + (kv.second->nullrows.p ? ng * 8 : 0) + (kv.second->fz.p ? ng * 8 : 0);
  blob.resize(total);
  char* p = blob.data();
  memcpy(p, &H, sizeof H); p += sizeof H;
  auto d2h = [&](const void* src, size_t n) { if (n) CK(cudaMemcpy(p, src, n, cudaMemcpyDeviceToHost)); p += n; };
  d2h(gid_key.p, ng * sizeof(GidKey));
  d2h(arena.p, ab);
  for (auto& kv : panes) {
    int64_t meta[3] = {kv.first, kv.second->nullrows.p ? 1 : 0, kv.second->fz.p ? 1 : 0};
    memcpy(p, meta, 24); p += 24;
    d2h(kv.second->st.p, ng * sizeof(GroupState));
    if (meta[1]) d2h(kv.second->nullrows.p, ng * 8);
    if (meta[2]) d2h(kv.second->fz.p, ng * 8);
  }
}

void dnz_window::restore(const char* blob, size_t bytes) {
  if (stats.rows_in != 0 || n_groups_host != 0 || !panes.empty()) fail(DNZ_ERR_INVALID, "restore needs a fresh operator");
  if (bytes < sizeof(CkptHeader)) fail(DNZ_ERR_INVALID, "checkpoint blob too short");
  CkptHeader H; memcpy(&H, blob, sizeof H);
  if (memcmp(H.magic, "DNZCKPT1", 8) != 0) fail(DNZ_ERR_INVALID, "not a checkpoint blob");
  if (H.window_ms != L || H.slide_ms != S || H.n_aggs != (int32_t)aggs.size()) fail(DNZ_ERR_INVALID, "checkpoint was taken with another window / aggregate configuration");
  if (((H.flags >> 4) & 0xF) != key_type) fail(DNZ_ERR_INVALID, "checkpoint was taken with another group key type");
  const size_t ng = H.n_groups, ab = round_up(H.arena_used, 8);
  const char* p = blob + sizeof H; const char* end = blob + bytes;
  auto need = [&](size_t n) { if ((size_t)(end - p) < n) fail(DNZ_ERR_INVALID, "checkpoint blob truncated"); };
  CK(cudaStreamSynchronize(stream));
  while (gcap < ng + ng / 8 + 1) dict_grow();                      // (nothing to rehash yet)
  if (ab + (1 << 20) > arena_cap) arena_grow(ab + (1 << 20));
  need(ng * sizeof(GidKey)); if (ng) CK(cudaMemcpy(gid_key.p, p, ng * sizeof(GidKey), cudaMemcpyHostToDevice)); p += ng * sizeof(GidKey);
  need(ab); if (ab) CK(cudaMemcpy(arena.p, p, ab, cudaMemcpyHostToDevice)); p += ab;
  const DictCounters c0{H.n_groups, 0u, H.arena_used, H.key_bytes_total};
  CK(cudaMemcpy(&ctl()->dict, &c0, sizeof c0, cudaMemcpyHostToDevice));
  CK(launch_dict_restore(dict_view(), H.n_groups, stream)); stats.total_launches++;      // sets null_gid for the NULL-key group
  need_nullrows = (H.flags & 2) != 0; need_fz = (H.flags & 4) != 0;
  for (int64_t i = 0; i < H.n_panes; i++) {
    need(24); int64_t meta[3]; memcpy(meta, p, 24); p += 24;
    Pane* pn = get_pane(meta[0], true);                              // zero-filled for gcap groups
    CK(cudaStreamSynchronize(stream));
    need(ng * sizeof(GroupState)); if (ng) CK(cudaMemcpy(pn->st.p, p, ng * sizeof(GroupState), cudaMemcpyHostToDevice)); p += ng * sizeof(GroupState);
    if (meta[1]) { if (!pn->nullrows.p) { need_nullrows = true; ensure_side_arrays(pn); CK(cudaStreamSynchronize(stream)); } need(ng * 8); if (ng) CK(cudaMemcpy(pn->nullrows.p, p, ng * 8, cudaMemcpyHostToDevice)); p += ng * 8; }
    if (meta[2]) { if (!pn->fz.p) { need_fz = true; ensure_side_arrays(pn); CK(cudaStreamSynchronize(stream)); } need(ng * 8); if (ng) CK(cudaMemcpy(pn->fz.p, p, ng * 8, cudaMemcpyHostToDevice)); p += ng * 8; }
  }
  has_wm = (H.flags & 1) != 0; wm = H.wm; emitted_upto = H.emitted_upto; next_seq = H.next_seq;
  has_lwm = (H.flags & 8) != 0; lwm = H.lwm; exported_pane_upto = H.exported_pane_upto;
  CK(cudaStreamSynchronize(stream));
  fetch_ctl();
}

// =================================================================================================
// C ABI
// =================================================================================================
extern "C" {

int32_t dnz_window_create(const dnz_window_config* cfg, const struct ArrowSchema* input_schema, dnz_window** out) {
  if (!out) { g_last_error = "null out"; return DNZ_ERR_INVALID; }
  *out = nullptr;
  dnz_window* w = nullptr;
  return create_guarded([&] {
    w = new dnz_window();
    w->init(cfg, input_schema);
    *out = w;
  }, [&] { delete w; });
}

int32_t dnz_window_push(dnz_window* w, struct ArrowArray* batch) {
  DNZ_TRY(w)
  w->push_host(batch);
  DNZ_CATCH(w)
}

int32_t dnz_window_push_device(dnz_window* w, const dnz_device_batch* batches, int64_t n) {
  DNZ_TRY(w)
  if (n < 0 || (n > 0 && !batches)) fail(DNZ_ERR_INVALID, "bad batch list");
  w->push_dev(batches, n);
  DNZ_CATCH(w)
}

int32_t dnz_window_poll(dnz_window* w, struct ArrowArray* out, struct ArrowSchema* out_schema, int32_t* has_output) {
  DNZ_TRY(w)
  if (!out) fail(DNZ_ERR_INVALID, "null out");
  w->process_pending(); w->drain();
  if (w->world > 1) w->fetch_ctl();          // exchange mode: surfaces merge / ring errors of the last step
  if (w->res_consumed) w->reset_results();
  w->export_arrow(out, out_schema, has_output, true);
  DNZ_CATCH(w)
}

int32_t dnz_window_poll_ready(dnz_window* w, struct ArrowArray* out, struct ArrowSchema* out_schema, int32_t* has_output) {
  DNZ_TRY(w)
  if (!out) fail(DNZ_ERR_INVALID, "null out");
  if (w->res_consumed) w->reset_results();
  w->async_polls = true;
  w->export_arrow(out, out_schema, has_output, false);
  DNZ_CATCH(w)
}

int32_t dnz_window_poll_device(dnz_window* w, dnz_device_result* out) {
  DNZ_TRY(w)
  if (!out) fail(DNZ_ERR_INVALID, "null out");
  w->process_pending(); w->drain();
  if (w->res_consumed) w->reset_results();
  w->export_device(out, true);
  DNZ_CATCH(w)
}

int32_t dnz_window_poll_device_ready(dnz_window* w, dnz_device_result* out) {
  DNZ_TRY(w)
  if (!out) fail(DNZ_ERR_INVALID, "null out");
  w->async_polls = true;
  w->export_device(out, false);
  DNZ_CATCH(w)
}

int32_t dnz_window_flush(dnz_window* w, int64_t watermark_ms) {
  DNZ_TRY(w)
  w->process_pending(); w->drain();
  if (w->res_consumed) w->reset_results();
  w->rotate_result_sets();
  if (w->ungrouped) w->ungrouped_emit_run(nullptr, nullptr, nullptr, watermark_ms);
  else w->emit_normal(watermark_ms, nullptr);
  DNZ_CATCH(w)
}

int32_t dnz_window_stats(const dnz_window* w, dnz_stats* out) {
  if (!w || !out) return DNZ_ERR_INVALID;
  *out = w->stats;
  return DNZ_OK;
}
int32_t dnz_window_reset_stats(dnz_window* w) {
  if (!w) return DNZ_ERR_INVALID;
  int64_t g = w->stats.groups;
  memset(&w->stats, 0, sizeof w->stats);
  w->stats.groups = g;
  return DNZ_OK;
}
int64_t dnz_window_watermark(const dnz_window* w) {
  if (!w) return INT64_MIN;
  if (w->world > 1) return w->has_lwm ? w->lwm : INT64_MIN;      // exchange mode: the LOCAL watermark (emission follows the global one)
  return w->has_wm ? w->wm : INT64_MIN;
}
const char* dnz_window_last_error(const dnz_window* w) { return w ? w->err.c_str() : g_last_error.c_str(); }
void dnz_window_destroy(dnz_window* w) { delete w; }

int32_t dnz_window_set_exchange(dnz_window* w, int32_t rank, int32_t world) {
  DNZ_TRY(w)
  if (world < 1 || rank < 0 || rank >= world) fail(DNZ_ERR_INVALID, "bad rank/world");
  if (w->ungrouped && world > 1) fail(DNZ_ERR_UNSUPPORTED, "ungrouped windows have no key to partition by");
  if (world > MAX_WORLD) fail(DNZ_ERR_UNSUPPORTED, "world > %d", MAX_WORLD);
  if (w->stats.rows_in > 0 && world != w->world) fail(DNZ_ERR_INVALID, "set_exchange must precede the first batch");
  w->rank = rank; w->world = world;
  if (world > 1) {
    w->need_nullrows = true; w->need_fz = true; for (auto& kv : w->panes) w->ensure_side_arrays(kv.second.get());
    // staging of the merge's pane table for the largest pane range of one step: page-locked allocations synchronise the device,
    // which must not happen while a peer rank of the same process spins in a wait kernel (dnz_group, local groups)
    w->h_xptrs.reserve((size_t)2 * 7 * (1 << 16) * sizeof(void*)); w->d_xptrs.reserve((size_t)2 * 7 * (1 << 16) * sizeof(void*));   // two halves (step parity)
  }
  DNZ_CATCH(w)
}
int32_t dnz_window_reserve_input(dnz_window* w, int64_t bytes_per_launch) {
  DNZ_TRY(w)
  if (bytes_per_launch < 0) fail(DNZ_ERR_INVALID, "negative size");
  for (Slot& s : w->slot) {
    Arena& a = s.arena;
    size_t have = 0; for (auto& b : a.slabs) have += b.bytes;
    if (have < (size_t)bytes_per_launch) { DevBuf b; b.alloc(round_up((size_t)bytes_per_launch - have, Arena::SLAB)); a.slabs.push_back(std::move(b)); }
  }
  DNZ_CATCH(w)
}
int32_t dnz_window_process(dnz_window* w, int64_t* local_watermark_ms) {
  DNZ_TRY(w)
  w->process_pending(); w->drain();
  if (local_watermark_ms) *local_watermark_ms = w->world > 1 ? (w->has_lwm ? w->lwm : INT64_MIN) : (w->has_wm ? w->wm : INT64_MIN);
  DNZ_CATCH(w)
}
int32_t dnz_window_export_partials(dnz_window* w, int64_t watermark_ms, dnz_partials* out) {
  DNZ_TRY(w)
  if (!out) fail(DNZ_ERR_INVALID, "null out");
  if (w->world <= 1) fail(DNZ_ERR_INVALID, "dnz_window_set_exchange was not called");
  w->export_partials(watermark_ms, out);
  DNZ_CATCH(w)
}
int32_t dnz_window_import_partials(dnz_window* w, const uint8_t* entries, const int64_t* src_counts, const uint8_t* key_bytes,
                                   const int64_t* src_key_bytes, int64_t pane_lo, int64_t pane_hi) {
  DNZ_TRY(w)
  if (w->world <= 1) fail(DNZ_ERR_INVALID, "dnz_window_set_exchange was not called");
  if (!src_counts || !src_key_bytes) fail(DNZ_ERR_INVALID, "null split arrays");
  w->import_partials(entries, src_counts, key_bytes, src_key_bytes, pane_lo, pane_hi);
  DNZ_CATCH(w)
}


int32_t dnz_window_checkpoint(dnz_window* w, void** blob, int64_t* bytes) {
  DNZ_TRY(w)
  if (!blob || !bytes) fail(DNZ_ERR_INVALID, "null out");
  std::vector<char> b;
  w->checkpoint(b);
  void* m = malloc(b.size() ? b.size() : 1);
  if (!m) fail(DNZ_ERR_NOMEM, "out of host memory");
  memcpy(m, b.data(), b.size());
  *blob = m; *bytes = (int64_t)b.size();
  DNZ_CATCH(w)
}
int32_t dnz_window_restore(dnz_window* w, const void* blob, int64_t bytes) {
  DNZ_TRY(w)
  if (!blob || bytes <= 0) fail(DNZ_ERR_INVALID, "null blob");
  w->restore(static_cast<const char*>(blob), (size_t)bytes);
  DNZ_CATCH(w)
}
void dnz_blob_free(void* blob) { free(blob); }

void* dnz_host_alloc(int64_t bytes) { void* p = nullptr; return cudaMallocHost(&p, (size_t)std::max<int64_t>(bytes, 64)) == cudaSuccess ? p : nullptr; }
void dnz_host_free(void* p) { if (p) cudaFreeHost(p); }
void* dnz_device_alloc(int32_t device, int64_t bytes) {
  void* p = nullptr;
  if (cudaSetDevice(device) != cudaSuccess) return nullptr;
  return cudaMalloc(&p, (size_t)std::max<int64_t>(bytes, 256)) == cudaSuccess ? p : nullptr;
}
void dnz_device_free(int32_t device, void* p) { if (p) { cudaSetDevice(device); cudaFree(p); } }
int32_t dnz_device_count(void) { int n = 0; return cudaGetDeviceCount(&n) == cudaSuccess ? n : 0; }
int32_t dnz_memcpy(void* dst, const void* src, int64_t bytes, int32_t kind) {
  if (bytes <= 0) return DNZ_OK;
  cudaError_t e = cudaMemcpy(dst, src, (size_t)bytes, kind == 1 ? cudaMemcpyHostToDevice : cudaMemcpyDeviceToHost);
  if (e != cudaSuccess) { g_last_error = cudaGetErrorString(e); return DNZ_ERR_CUDA; }
  return DNZ_OK;
}

}  // extern "C"
