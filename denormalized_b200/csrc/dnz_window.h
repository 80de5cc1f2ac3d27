// dnz_window.h -- internal declarations shared by the host-side translation units of the operator (dnz_window.cu,
// dnz_results.cu, dnz_ungrouped.cu, dnz_group.cu, dnz_synth.cu).  The public boundary is include/dnz_gpu.h.
#pragma once
#include <cuda_runtime.h>

#include <algorithm>
#include <chrono>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <deque>
#include <functional>
#include <map>
#include <memory>
#include <mutex>
#include <set>
#include <string>
#include <vector>

#include "../../include/dnz_gpu.h"
#include "dnz_kernels.h"

namespace dnz {

struct DnzError {
  int32_t code; std::string msg;
};
[[noreturn]] inline void fail(int32_t code, const char* fmt, ...) {
  char buf[512]; va_list ap; va_start(ap, fmt); vsnprintf(buf, sizeof buf, fmt, ap); va_end(ap);
  throw DnzError{code, buf};
}
#define CK(expr)                                                                                          \
  do {                                                                                                    \
    cudaError_t e__ = (expr);                                                                             \
    if (e__ != cudaSuccess) fail(DNZ_ERR_CUDA, "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(e__), __FILE__, __LINE__); \
  } while (0)

inline thread_local std::string g_last_error;       // one per thread for the whole library

// DNZ_TRACE=1: host-side phase timings per superbatch on stderr (debugging aid)
inline const bool g_trace = getenv("DNZ_TRACE") != nullptr;
struct Trace {
  std::chrono::steady_clock::time_point t0 = std::chrono::steady_clock::now();
  std::string line;
  void mark(const char* what) {
    if (!g_trace) return;
    auto t1 = std::chrono::steady_clock::now();
    char buf[64]; snprintf(buf, sizeof buf, " %s=%.3fms", what, std::chrono::duration<double, std::milli>(t1 - t0).count());
    line += buf; t0 = t1;
  }
  void flush(const char* tag) { if (g_trace) fprintf(stderr, "[dnz] %s:%s\n", tag, line.c_str()); line.clear(); }
};
inline Trace g_tr;

inline int64_t floor_div(int64_t a, int64_t b) { int64_t q = a / b; return (a % b != 0 && ((a < 0) != (b < 0))) ? q - 1 : q; }
inline size_t round_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

// device memory helpers (dnz_window.cu): the CUDA stream-ordered allocator of the current device
struct AllocCtx { cudaStream_t s = nullptr; bool async_ok = false; };
AllocCtx& alloc_ctx();
void* dev_alloc(size_t n);
void dev_free(void* p);          // callers free only after the work that used the block has completed

struct DevBuf {
  void* p = nullptr; size_t bytes = 0;
  DevBuf() = default;
  DevBuf(const DevBuf&) = delete; DevBuf& operator=(const DevBuf&) = delete;
  DevBuf(DevBuf&& o) noexcept : p(o.p), bytes(o.bytes) { o.p = nullptr; o.bytes = 0; }
  DevBuf& operator=(DevBuf&& o) noexcept { if (this != &o) { release(); p = o.p; bytes = o.bytes; o.p = nullptr; o.bytes = 0; } return *this; }
  ~DevBuf() { release(); }
  void release() { if (p) dev_free(p); p = nullptr; bytes = 0; }
  void alloc(size_t n) { release(); if (n == 0) n = 256; p = dev_alloc(n); bytes = n; }
  // grow without preserving contents
  void reserve(size_t n) { if (n > bytes) alloc(std::max(n, bytes + bytes / 2)); }
  // grow in stream order on `st`, keeping the first `keep` bytes: no host synchronisation (work enqueued on `st` before this call
  // still sees the old block, which is freed behind it)
  void regrow_on(cudaStream_t st, size_t n, size_t keep) {
    AllocCtx& c = alloc_ctx();
    if (!c.async_ok) {
      DevBuf nb; nb.alloc(n);
      if (keep && p) CK(cudaMemcpyAsync(nb.p, p, keep, cudaMemcpyDeviceToDevice, st));
      CK(cudaStreamSynchronize(st));
      *this = std::move(nb);
      return;
    }
    void* np = nullptr;
    CK(cudaMallocAsync(&np, n, st));
    if (keep && p) CK(cudaMemcpyAsync(np, p, keep, cudaMemcpyDeviceToDevice, st));
    if (p) cudaFreeAsync(p, st);
    p = np; bytes = n;
  }
  template <class T> T* as() const { return reinterpret_cast<T*>(p); }
};

struct PinnedBuf {
  void* p = nullptr; size_t bytes = 0;
  ~PinnedBuf() { if (p) cudaFreeHost(p); }
  void reserve(size_t n) {
    if (n <= bytes) return;
    const size_t want = std::max(n, bytes * 2);
    if (p) cudaFreeHost(p);
    p = nullptr; bytes = 0;
    CK(cudaMallocHost(&p, want)); bytes = want;
  }
  template <class T> T* as() const { return reinterpret_cast<T*>(p); }
};

// bump allocator for the device copies of pushed host batches
struct Arena {
  std::vector<DevBuf> slabs; size_t cur = 0, off = 0;
  static constexpr size_t SLAB = 256ull << 20;
  void* alloc(size_t n) {
    n = round_up(n + 32, 256);
    while (true) {
      if (cur < slabs.size() && off + n <= slabs[cur].bytes) { void* r = (char*)slabs[cur].p + off; off += n; return r; }
      if (cur + 1 < slabs.size() && n <= slabs[cur + 1].bytes) { cur++; off = 0; continue; }
      DevBuf b; b.alloc(std::max(n, SLAB));
      slabs.insert(slabs.begin() + (slabs.empty() ? 0 : cur + 1), std::move(b));
      if (slabs.size() > 1) cur++;
      off = 0;
    }
  }
  void reset() { cur = 0; off = 0; }
};

struct Pane {
  int64_t id = 0;
  uint64_t tag = 0;        // names this zero-initialised instance of `st` (DictSlot::hint); never reused
  DevBuf st, nullrows, fz;
};


struct PendingBatch {
  BatchDesc d{};
  int64_t key_bytes = 0;
  bool has_moved = false;
  ArrowArray moved{};
};

// One superbatch (<= max_rows_per_launch rows) travelling through the pipeline.  Three of them rotate:
//   FILLING   batches are being pushed; host batches are copied into the slot's arena as they arrive (copy stream)
//   SEALED    the tile scan (per-batch watermarks, per-tile byte ranges) has been enqueued
//   LAUNCHED  the aggregate launch and the emission of the windows it closes have been enqueued, a snapshot of the
//             control block follows them in stream order
//   FREE      the snapshot has been inspected on the host (`verify`): nothing was deferred, or it has been replayed
// so that in steady state the host never waits between a kernel and the next one: while slot k's aggregate runs, slot k+1's
// scan is already queued behind it and the host is one full superbatch ahead.
struct Slot {
  enum State { FREE, FILLING, SEALED, LAUNCHED };
  State state = FREE;
  int idx = 0;
  std::vector<PendingBatch> batches; int64_t rows = 0; bool copies = false;
  std::vector<CopyDesc> gather;       // pinned host buffers pulled by one k_gather_copy launch when the superbatch is sealed
  Arena arena; cudaEvent_t copy_done = nullptr;
  DevBuf d_copy_descs; PinnedBuf h_copy_descs;
  // tile scan
  DevBuf d_batches, d_tiles, d_minmax; PinnedBuf h_batches, h_minmax; cudaEvent_t scan_done = nullptr;
  std::vector<BatchDesc> bds; int64_t n_tiles = 0; bool scanned = false;
  // canonical timestamps still to be derived from raw columns of this superbatch (k_ts_convert, before the scan)
  std::vector<TsJob> ts_jobs; int64_t ts_max_rows = 0; DevBuf d_ts_jobs; PinnedBuf h_ts_jobs;
  // aggregate launch (its own staging: the async copies read these buffers when the stream gets there)
  DevBuf d_ptrs, d_defer[2]; PinnedBuf h_ptrs;
  PinnedBuf snap; cudaEvent_t done = nullptr; cudaEvent_t ev0 = nullptr, ev1 = nullptr;
  bool timed = false; double alg_bytes = 0;
  // what was enqueued speculatively behind the aggregate launch (replayed by verify() when rows were deferred)
  bool speculative = false;
  int64_t t0 = 0, t1 = 0, pmin = 0, pmax = -1;
  std::vector<int64_t> emit_starts;
  uint64_t add_rows_bound = 0, add_bytes_bound = 0; int emit_set = 0;
  int64_t rows_launched = 0;
  std::vector<std::unique_ptr<Pane>> retired;      // panes whose last window was emitted behind this launch
};

// Device columns of emitted rows.  Two sets: emission appends to one of them; a set whose rows have all been handed out is
// reset and becomes the next target, so a consumer that polls while input keeps streaming never makes the operator wait.
// What may be handed out is decided by SNAPSHOTS: after every group of emit launches the cursor is copied to pinned memory
// and an event is recorded; once the event has fired, rows below the snapshot are complete and stable (append-only).
struct ResultSet {
  DevBuf key_off, key_bytes, key_valid, count, mn, mx, avg, sum, agg_valid, wstart, wend;
  uint64_t row_cap = 0, byte_cap = 0;
  uint64_t rows = 0, bytes = 0;           // host view of the cursor: an UPPER BOUND while launches are in flight, exact after fetch_ctl
  uint64_t exp_rows = 0, exp_bytes = 0;   // prefix already handed to the consumer
  PinnedBuf snap; cudaEvent_t snap_ev = nullptr; bool snap_issued = false;   // snap: a ResultCursor
};


// ------------------------------------------------------------------------------------------------
// Arrow C-Data export plumbing
// Page-locked blocks for exported results are recycled: cudaMallocHost costs milliseconds, a poll must not.
struct PinnedPool {
  std::mutex m; std::multimap<size_t, void*> free_blocks;
  void* get(size_t n, size_t& cap) {
    {
      std::lock_guard<std::mutex> g(m);
      auto it = free_blocks.lower_bound(n);
      if (it != free_blocks.end() && it->first <= 4 * n + (1 << 20)) { void* p = it->second; cap = it->first; free_blocks.erase(it); return p; }
    }
    void* p = nullptr; cap = round_up(n + n / 4, 1 << 16);
    CK(cudaMallocHost(&p, cap));
    return p;
  }
  void put(void* p, size_t cap) {
    std::lock_guard<std::mutex> g(m);
    if (free_blocks.size() >= 8) { auto it = free_blocks.begin(); cudaFreeHost(it->second); free_blocks.erase(it); }
    free_blocks.emplace(cap, p);
  }
};
inline PinnedPool g_pinned_pool;

struct ExportPrivate {
  void* block = nullptr; size_t block_cap = 0;   // one pooled page-locked block holds every exported buffer
  ~ExportPrivate() { if (block) g_pinned_pool.put(block, block_cap); }
  std::vector<std::unique_ptr<ArrowArray>> children; std::vector<ArrowArray*> child_ptrs;
  std::vector<std::vector<const void*>> buffers;
};
inline void release_array(ArrowArray* a) {
  if (!a || !a->release) return;
  if (a->private_data) {
    delete static_cast<ExportPrivate*>(a->private_data);
  }
  a->release = nullptr;
}
inline void release_child(ArrowArray* a) { a->release = nullptr; }

// An exported RecordBatch of n rows being assembled: its buffers are carved from one pooled page-locked block of `block_bytes`
// (take), its children point into them (add_child).
struct ArrowBatch {
  std::unique_ptr<ExportPrivate> ep{new ExportPrivate()};
  int64_t n; size_t used = 0;
  ArrowBatch(uint64_t rows, size_t block_bytes, size_t n_children) : n((int64_t)rows) {
    ep->block = g_pinned_pool.get(block_bytes, ep->block_cap);
    ep->buffers.reserve(n_children + 1);
  }
  void* take(size_t bytes) { void* p = (char*)ep->block + used; used += round_up(std::max<size_t>(bytes, 8), 64); return p; }
  void add_child(std::vector<const void*> bufs, int64_t nulls) {
    ep->buffers.push_back(std::move(bufs));
    auto c = std::make_unique<ArrowArray>();
    memset(c.get(), 0, sizeof(ArrowArray));
    c->length = n; c->null_count = nulls; c->n_buffers = (int64_t)ep->buffers.back().size();
    c->buffers = ep->buffers.back().data(); c->release = release_child;
    ep->children.push_back(std::move(c));
  }
};
// host columns of the aggregates and the window bounds (validity: shared by every nullable aggregate, nullptr: no NULL)
struct ExportColumns {
  const uint8_t* validity; int64_t nulls;
  const int64_t* count; const double *mn, *mx, *avg, *sum; const int64_t *ws, *we;
};


}  // namespace dnz

using namespace dnz;

struct dnz_group;
struct dnz_window {
  dnz_window_config cfg{};
  std::vector<dnz_agg> aggs; std::vector<std::string> aliases;
  std::string key_name;
  // group key type: an index into KEY_TYPES (0 Utf8; Int64 / Int32 / UInt64 / UInt32, whose values are key_width = 8 or 4 bytes
  // each); key_width == 0 for Utf8 keys and for the ungrouped window.  key_nullable: the input field's nullability (integer keys
  // echo it in the emitted schema; Utf8 keys are emitted nullable, as they always were)
  int key_type = 0, key_width = 0; bool key_nullable = true;
  uint32_t key_tag() const { return (uint32_t)key_type << KEY_TYPE_SHIFT; }
  int key_col = -1, val_col = -1, meta_col = -1, ts_child = -1, n_input_cols = 0;
  int ts_source = DNZ_TS_CANONICAL, ts_col = -1; TsFormat ts_fmt{};      // input-contract producer (SURVEY §8 f1)
  int dev = 0; int sm_count = 148;
  cudaStream_t stream = nullptr; bool own_stream = false;
  cudaStream_t copy_stream = nullptr;
  int64_t L = 0, S = 0, pane_ms = 0; int panes_per_window = 1;
  int64_t max_rows = 64ll << 20;

  // dictionary
  DevBuf slots, gid_key, arena;
  DevBuf d_ctl;                       // the CtlBlock: every device counter the host reads back after a launch
  CtlBlock* ctl() const { return d_ctl.as<CtlBlock>(); }
  uint32_t dict_cap = 0, gcap = 0;
  uint64_t arena_cap = 0;     // LOGICAL capacity handed to the kernels (<= arena.bytes): bounds what launches in flight can add

  // host knowledge of the device counters: exact as of the last inspected snapshot ("known"), plus what launches enqueued since
  // then can have added at most ("bound")
  uint32_t n_groups_host = 0; uint64_t key_bytes_total_host = 0, arena_used_host = 0;
  int64_t rows_since_known = 0;
  uint64_t defer_count_host = 0; uint32_t defer_flags_host = 0;

  // panes
  std::map<int64_t, std::unique_ptr<Pane>> panes;
  std::map<int64_t, std::unique_ptr<Pane>> late_panes;     // one-batch panes of the exact late path (alive only inside a dirty run)
  std::vector<std::unique_ptr<Pane>> pane_pool;
  bool need_nullrows = false, need_fz = false;
  uint64_t next_tag = 1;   // pane instance tags (low 32 bits are stored in the hints)
  bool has_wm = false; int64_t wm = 0;
  int64_t emitted_upto = INT64_MIN;

  // pipeline
  Slot slot[PIPELINE_SLOTS]; int fill = 0; int64_t next_seq = 0;
  std::vector<int> sealed_order;      // SEALED slots, oldest first
  std::vector<int> launched_order;    // LAUNCHED slots, oldest first
  Slot& cur() { return slot[fill]; }
  bool in_process = false;            // an error thrown while true kills the stream (sticky), as the reference's panics do

  // scratch
  DevBuf d_priv, d_copy_cursor;
  PinnedBuf h_small;
  ResultSet rs[2]; int wr = 0; bool async_polls = false;
  ResultSet& R() { return rs[wr]; }
  cudaStream_t d2h_stream = nullptr;
  bool res_consumed = false;

  // ungrouped windows `.window([], aggs, ..)` (SURVEY §8 f2): the device reduces rows into panes; the Partial stage's per-batch
  // emission schedule and the whole Final stage (streaming_window.rs:882-1051) run on the host over one 40 B state per window
  bool ungrouped = false;
  std::set<int64_t> u_created;                  // Partial frames that exist (window starts)
  struct UEmission { std::vector<std::vector<int64_t>> pbs; size_t first = 0, count = 0; cudaEvent_t ev = nullptr; };
  std::deque<UEmission> u_pending;              // emissions whose partial states are on their way to the host
  std::vector<cudaEvent_t> u_event_pool;
  DevBuf d_uwins, d_ustates; PinnedBuf h_uwins, h_ustates; size_t u_ring = 0, u_head = 0;   // UState / UWindow slots, bump-allocated; reset when nothing is pending
  struct UFrame { int64_t end = 0; uint64_t cnt = 0; double sum = 0; bool has = false; double mn = 0, mx = 0; };
  std::map<int64_t, UFrame> u_final; std::set<int64_t> u_seen; bool u_has_fwm = false; int64_t u_fwm = 0;
  struct URow { int64_t ws, we; int64_t cnt; double mn, mx, avg, sum; bool valid; };
  std::vector<URow> u_out;
  void ungrouped_collect(bool wait);
  void ungrouped_final(const std::vector<URow>& pb);
  void export_ungrouped(ArrowArray* out, ArrowSchema* schema, int32_t* has_output, bool blocking);

  // multi-GPU pane exchange
  int rank = 0, world = 1;
  bool fused = false;                             // attached to a dnz_group: launches stay asynchronous, emission happens in the group step
  bool group_started = false;                     // this operator has taken part in a group step (its stream has begun in the group)
  bool has_lwm = false; int64_t lwm = 0;          // local watermark (exchange mode: emission follows the GLOBAL one)
  int64_t exported_pane_upto = INT64_MIN;
  DevBuf d_part_entries, d_part_keys, d_owner_cursor, d_pack_dest, d_xptrs; PinnedBuf h_xptrs;
  std::vector<int64_t> h_owner_counts, h_owner_bytes;
  void group_begin(struct dnz_group* g);
  void group_pack(struct dnz_group* g);
  void group_finish(struct dnz_group* g, int64_t* gwm_out);
  void export_partials(int64_t watermark, dnz_partials* out);
  void import_partials(const uint8_t* entries, const int64_t* src_counts, const uint8_t* key_bytes, const int64_t* src_key_bytes,
                       int64_t pane_lo, int64_t pane_hi);

  dnz_stats stats{};
  std::string err; int32_t sticky = 0;

  ~dnz_window();
  void init(const dnz_window_config* c, const ArrowSchema* schema);
  DictView dict_view() const;
  void dict_alloc(uint32_t new_gcap);
  void dict_grow();
  void arena_grow(uint64_t at_least);
  void arena_trim();
  void fetch_ctl();
  void parse_ctl(const CtlBlock& h);
  template <class F> void for_each_live_pane(F f);
  Pane* get_pane(int64_t id, bool create);
  Pane* find_pane(int64_t id);
  std::unique_ptr<Pane> new_pane(int64_t id);
  void ensure_side_arrays(Pane* p);
  void retire_panes(Slot* sl);
  void recycle_pane(std::unique_ptr<Pane> p);
  void release_late_panes();
  using PaneLookup = std::function<std::pair<Pane*, Pane*>(int64_t)>;     // pane id -> (main pane, late pane), either nullable
  PaneTable upload_pane_table(void** hp, char* dp, int64_t p0, int64_t p1, const PaneLookup& panes);
  void push_host(ArrowArray* batch);
  void push_dev(const dnz_device_batch* b, int64_t n);
  void process_pending();
  void drain();
  void seal_current();
  void finish_copies(Slot& s);
  void launch_scan(Slot& s);
  void launch_slot(Slot& s);
  void verify(Slot& s);
  void verify_completed();
  void release_slot(Slot& s);
  void prealloc();
  struct Run { size_t b0, b1; bool dirty; int64_t horizon, wm_after; };
  void plan_runs(Slot& s, const std::vector<BatchMinMax>& mm, std::vector<Run>& runs);
  void ungrouped_emit_run(Slot* sl, const std::vector<BatchMinMax>* mm, const Run* r, int64_t flush_wm);
  struct RunGeom { int64_t t0 = 0, t1 = 0, pmin = INT64_MAX, pmax = INT64_MIN, rows = 0; double alg_bytes = 0; bool val_nulls = false; };
  RunGeom run_geometry(Slot& s, const std::vector<BatchMinMax>& mm, const Run& r);
  void prepare_panes(Slot& s, const std::vector<BatchMinMax>& mm, const Run& r, const RunGeom& g);
  AggParams build_agg_params(Slot& s, const RunGeom& g, bool dirty, int64_t horizon, int out_list);
  void launch_aggregate_pass(Slot& s, const RunGeom& g, AggParams& P, bool dirty);
  void resolve_deferred(Slot& s, const RunGeom& g, bool dirty, int64_t horizon);
  RunGeom enqueue_run(Slot& s, const std::vector<BatchMinMax>& mm, const Run& r);
  void advance_and_emit(const std::vector<BatchMinMax>& mm, const Run& r, Slot* gate);
  void collect_kernel_time(Slot& s);
  void execute_run_sync(Slot& s, const std::vector<BatchMinMax>& mm, const Run& r);
  void emit_windows(const std::vector<int64_t>& starts, const std::map<int64_t, Pane*>& src, Slot* gate);
  using PaneMap = std::map<int64_t, std::unique_ptr<Pane>>;
  void emit_closed(const PaneMap& ps, int64_t end_after, int64_t end_upto, Slot* gate);
  void emit_normal(int64_t wm_new, Slot* gate);
  std::map<int64_t, Pane*> pane_sources();
  void ensure_result_capacity(uint64_t add_rows, uint64_t add_bytes);
  uint32_t groups_bound() const;
  uint64_t key_bytes_bound() const;
  void reset_results();
  void reset_set(int i);
  void snapshot_results();
  void rotate_result_sets();
  bool set_drained(ResultSet& r);
  bool ready_rows(ResultSet& r, uint64_t& rows, uint64_t& bytes);
  void hand_out(ArrowBatch& b, const ExportColumns& c, ArrowArray* out, ArrowSchema* schema, int32_t* has_output);
  void export_arrow(ArrowArray* out, ArrowSchema* schema, int32_t* has_output, bool blocking);
  void export_device(dnz_device_result* out, bool blocking);
  void checkpoint(std::vector<char>& blob);
  void restore(const char* blob, size_t bytes);
  void fill_schema(ArrowSchema* schema);
};

// marks the operator in_process for the lifetime of a scope (restoring the previous value: scopes nest)
struct InProcess {
  dnz_window* w; bool prev;
  explicit InProcess(dnz_window* w_) : w(w_), prev(w_->in_process) { w->in_process = true; }
  ~InProcess() { w->in_process = prev; }
};


// ------------------------------------------------------------------------------------------------
// C ABI helpers
#define DNZ_TRY(w)                                                                  \
  if (!(w)) { g_last_error = "null handle"; return DNZ_ERR_INVALID; }               \
  if ((w)->sticky) return (w)->sticky;                                              \
  cudaSetDevice((w)->dev);                                                          \
  try {
#define DNZ_CATCH(w)                                                                \
  } catch (const DnzError& e) {                                                     \
    (w)->err = e.msg; g_last_error = e.msg;                                         \
    if (e.code == DNZ_ERR_CUDA || (w)->in_process) (w)->sticky = e.code;            \
    return e.code;                                                                  \
  } catch (const std::exception& e) {                                               \
    (w)->err = e.what(); g_last_error = e.what(); return DNZ_ERR_NOMEM;             \
  }                                                                                 \
  return DNZ_OK;

// the create functions: an error thrown by `body` is recorded in g_last_error, `cleanup` frees what was made, its code is returned
template <class Body, class Cleanup> int32_t create_guarded(Body&& body, Cleanup&& cleanup) {
  try {
    body();
    return DNZ_OK;
  } catch (const DnzError& e) {
    g_last_error = e.msg; cleanup(); return e.code;
  } catch (const std::exception& e) {
    g_last_error = e.what(); cleanup(); return DNZ_ERR_NOMEM;
  }
}
