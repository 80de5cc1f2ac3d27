// dnz_window.cu -- host side of the H100 streaming-window operator behind the C ABI of include/dnz_gpu.h.
//
// Mirrors GroupedWindowAggStream (crates/core/src/physical_plan/continuous/grouped_window_agg_stream.rs):
//   push/poll           <-> poll_next_inner (:326-349): watermark -> windows -> frames.push -> process_watermark -> trigger
//   pipeline (Slot)     <-> the stream's poll loop, three superbatches deep: scan k+1 | aggregate + emit k | verify k-1
//   PaneStore           <-> window_frames: BTreeMap<SystemTime, GroupedAggWindowFrame> (:63-82), re-organised as hop-sized
//                           panes shared by the L/S windows that overlap them (SURVEY.md §5.7)
//   Dictionary          <-> GroupValues (one per frame in the reference; one per stream here, ids are stable)
//   plan_runs           <-> the per-batch watermark rule (:255-266) + late rows re-opening emitted windows (§8a-3)
// and the Arrow<->device buffer manager (host Arrow C-Data in, device columns, Arrow C-Data out).
#include <cuda_runtime.h>

#include <algorithm>
#include <chrono>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <deque>
#include <map>
#include <memory>
#include <mutex>
#include <set>
#include <string>
#include <vector>

#include "../../include/dnz_gpu.h"
#include "dnz_kernels.h"

using namespace dnz;

namespace {

struct DnzError {
  int32_t code; std::string msg;
};
[[noreturn]] void fail(int32_t code, const char* fmt, ...) {
  char buf[512]; va_list ap; va_start(ap, fmt); vsnprintf(buf, sizeof buf, fmt, ap); va_end(ap);
  throw DnzError{code, buf};
}
#define CK(expr)                                                                                          \
  do {                                                                                                    \
    cudaError_t e__ = (expr);                                                                             \
    if (e__ != cudaSuccess) fail(DNZ_ERR_CUDA, "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(e__), __FILE__, __LINE__); \
  } while (0)

thread_local std::string g_last_error;

// DNZ_TRACE=1: host-side phase timings per superbatch on stderr (debugging aid)
const bool g_trace = getenv("DNZ_TRACE") != nullptr;
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
Trace g_tr;

inline int64_t floor_div(int64_t a, int64_t b) { int64_t q = a / b; return (a % b != 0 && ((a < 0) != (b < 0))) ? q - 1 : q; }
inline size_t round_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

// ------------------------------------------------------------------------------------------------
// device memory helpers.  All device buffers come from the CUDA stream-ordered allocator with an unbounded release
// threshold: blocks freed by one operator stay cached in the process and are handed to the next one without a driver
// call (plain cudaMalloc/cudaFree cost milliseconds to seconds once tens of GB are mapped, and cudaFree synchronises
// the whole device).
struct AllocCtx { cudaStream_t s = nullptr; bool async_ok = false; };
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
constexpr int NSLOT = 3;
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
  size_t ctl_off() const { return 64 + 32 * (size_t)idx; }     // defer count (u64) flags (u32) tile counter (u32) emit-blocked (u32)
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
  size_t ctl_off = 192;                   // cursor (u64) + overflow flag (u32) inside the control block
  PinnedBuf snap; cudaEvent_t snap_ev = nullptr; bool snap_issued = false;
};

enum { COL_COUNT = 0, COL_MIN = 1, COL_MAX = 2, COL_AVG = 3, COL_SUM = 4 };
constexpr size_t CTL_BYTES = 256, CTL_MERGE_ERR = 224, CTL_TS_ERR = 228;

}  // namespace

struct dnz_group;
struct dnz_window {
  dnz_window_config cfg{};
  std::vector<dnz_agg> aggs; std::vector<std::string> aliases;
  std::string key_name;
  int key_col = -1, val_col = -1, meta_col = -1, ts_child = -1, n_input_cols = 0;
  int ts_source = DNZ_TS_CANONICAL, ts_col = -1; TsFormat ts_fmt{};      // input-contract producer (SURVEY §8 f1)
  int dev = 0; int sm_count = 148;
  cudaStream_t stream = nullptr; bool own_stream = false;
  cudaStream_t copy_stream = nullptr;
  int64_t L = 0, S = 0, pane_ms = 0; int panes_per_window = 1;
  int64_t max_rows = 64ll << 20;

  // dictionary
  DevBuf slots, gid_key, arena;
  // one 256 B device control block so that a single D2H copy fetches everything the host needs after a launch:
  //   +0    n_groups(u32) null_gid(u32) arena_used(u64) key_bytes_total(u64)
  //   +64 + 32 s   pipeline slot s: deferred-row count(u64) flags(u32) tile counter(u32) emit-blocked(u32)
  //   +192  result set 0: cursor(u64: rows<<32|bytes) overflow(u32);  +208 result set 1
  //   +224  pane-merge error flags (exchange)
  DevBuf d_ctl;
  char* ctl(size_t off) const { return d_ctl.as<char>() + off; }
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
  Slot slot[NSLOT]; int fill = 0; int64_t next_seq = 0;
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
  DevBuf d_part_entries, d_part_keys, d_owner_cursor, d_xptrs; PinnedBuf h_xptrs;
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
  void parse_ctl(const char* h);
  template <class F> void for_each_live_pane(F f);
  Pane* get_pane(int64_t id, bool create);
  Pane* find_pane(int64_t id);
  std::unique_ptr<Pane> new_pane(int64_t id);
  void ensure_side_arrays(Pane* p);
  void retire_panes(Slot* sl);
  void push_host(ArrowArray* batch);
  void push_dev(const dnz_device_batch* b, int64_t n);
  void process_pending();
  void drain();
  void seal_current();
  void finish_copies(Slot& s);
  void launch_scan(Slot& s);
  void launch_slot(Slot& s);
  void verify(Slot& s);
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
  void execute_run_sync(Slot& s, const std::vector<BatchMinMax>& mm, const Run& r);
  void emit_windows(const std::vector<int64_t>& starts, const std::map<int64_t, Pane*>& src, bool gated, Slot* sl);
  void emit_normal(int64_t wm_new, bool gated, Slot* sl);
  std::map<int64_t, Pane*> pane_sources();
  void ensure_result_capacity(uint64_t add_rows, uint64_t add_bytes);
  uint32_t groups_bound() const;
  uint64_t key_bytes_bound() const;
  void reset_results();
  void reset_set(int i);
  void snapshot_results();
  void rotate_result_sets();
  bool set_drained(ResultSet& r);
  void export_arrow(ArrowArray* out, ArrowSchema* schema, int32_t* has_output, bool blocking);
  void export_device(dnz_device_result* out, bool blocking);
  void checkpoint(std::vector<char>& blob);
  void restore(const char* blob, size_t bytes);
  void fill_schema(ArrowSchema* schema);
};

namespace {

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
PinnedPool g_pinned_pool;

struct ExportPrivate {
  void* block = nullptr; size_t block_cap = 0;   // one pooled page-locked block holds every exported buffer
  ~ExportPrivate() { if (block) g_pinned_pool.put(block, block_cap); }
  std::vector<std::unique_ptr<ArrowArray>> children; std::vector<ArrowArray*> child_ptrs;
  std::vector<std::vector<const void*>> buffers;
};
void release_array(ArrowArray* a) {
  if (!a || !a->release) return;
  if (a->private_data) {
    delete static_cast<ExportPrivate*>(a->private_data);
  }
  a->release = nullptr;
}
void release_child(ArrowArray* a) { a->release = nullptr; }

struct SchemaPrivate {
  std::vector<std::unique_ptr<ArrowSchema>> children; std::vector<ArrowSchema*> child_ptrs; std::vector<std::string> names;
};
void release_schema(ArrowSchema* s) {
  if (!s || !s->release) return;
  if (s->private_data) delete static_cast<SchemaPrivate*>(s->private_data);
  s->release = nullptr;
}
void release_child_schema(ArrowSchema* s) { s->release = nullptr; }

const char* agg_format(int kind) { return kind == DNZ_AGG_COUNT ? "l" : "g"; }

}  // namespace


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
    if (strcmp(ks->format, "u") != 0) fail(DNZ_ERR_UNSUPPORTED, "group key column '%s' has format '%s'; only Utf8 keys are implemented", ks->name, ks->format);
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
  rs[0].ctl_off = 192; rs[1].ctl_off = 208;
  for (auto& r : rs) { CK(cudaEventCreateWithFlags(&r.snap_ev, cudaEventDisableTiming)); r.snap.reserve(64); }
  for (int i = 0; i < NSLOT; i++) {
    Slot& s = slot[i]; s.idx = i;
    CK(cudaEventCreateWithFlags(&s.copy_done, cudaEventDisableTiming));
    CK(cudaEventCreateWithFlags(&s.scan_done, cudaEventDisableTiming));
    CK(cudaEventCreateWithFlags(&s.done, cudaEventDisableTiming));
    CK(cudaEventCreate(&s.ev0)); CK(cudaEventCreate(&s.ev1));
    s.snap.reserve(CTL_BYTES);
  }
  slot[0].state = Slot::FILLING; fill = 0;
  CK(agg_kernel_setup());

  d_ctl.alloc(CTL_BYTES); CK(cudaMemsetAsync(d_ctl.p, 0, CTL_BYTES, stream));
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
  uint32_t* c32 = reinterpret_cast<uint32_t*>(ctl(0));
  d.n_groups = c32; d.null_gid = c32 + 1;
  d.arena_used = reinterpret_cast<unsigned long long*>(c32 + 2);
  d.key_bytes_total = reinterpret_cast<unsigned long long*>(c32 + 4);
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

void dnz_window::parse_ctl(const char* h) {
  if (*reinterpret_cast<const uint32_t*>(h + CTL_TS_ERR)) fail(DNZ_ERR_DATA, "a timestamp string does not match the format (the reference unwraps the parse error and panics)");
  if (const uint32_t xe = *reinterpret_cast<const uint32_t*>(h + CTL_MERGE_ERR)) {
    if (xe & 0x100u) fail(DNZ_ERR_NOMEM, "exchange ring overflow: an owner's ring is smaller than one step's packets (dnz_group_config.ring_entries / ring_key_bytes)");
    fail(DNZ_ERR_NOMEM, "pane merge failed (flags %u): the dictionary / key arena of this rank is too small for the keys it owns (in exchange mode expected_groups must cover the GLOBAL key set)", xe);
  }
  n_groups_host = std::min(*reinterpret_cast<const uint32_t*>(h), gcap);
  arena_used_host = *reinterpret_cast<const uint64_t*>(h + 8);
  key_bytes_total_host = *reinterpret_cast<const uint64_t*>(h + 16);
  for (auto& r : rs)
    if (*reinterpret_cast<const uint32_t*>(h + r.ctl_off + 8)) fail(DNZ_ERR_NOMEM, "result buffer overflow (internal sizing error)");
  stats.groups = n_groups_host;
}
// one small D2H + sync: every launch enqueued so far has completed, the host view becomes exact
void dnz_window::fetch_ctl() {
  h_small.reserve(CTL_BYTES);
  CK(cudaMemcpyAsync(h_small.p, d_ctl.p, CTL_BYTES, cudaMemcpyDeviceToHost, stream));
  CK(cudaStreamSynchronize(stream));
  const char* h = h_small.as<char>();
  parse_ctl(h);
  rows_since_known = 0;
  for (auto& r : rs) {
    uint64_t c = *reinterpret_cast<const uint64_t*>(h + r.ctl_off);
    r.rows = c >> 32; r.bytes = c & 0xFFFFFFFFull;
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
  return key_bytes_total_host + fresh * INLINE_KEY + (arena_cap - std::min<uint64_t>(arena_used_host, arena_cap));
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
      else if (pane_pool.size() < 16) pane_pool.push_back(std::move(it->second));
      it = panes.erase(it);
    } else ++it;
  }
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
    if (!ungrouped) {
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
    if (s.n_rows > 0 && (!s.ts || !s.val || (!ungrouped && (!s.key_off || !s.key_bytes)))) fail(DNZ_ERR_INVALID, "device batch %lld: null column pointer", (long long)i);
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
  struct Guard { dnz_window* w; bool prev; ~Guard() { w->in_process = prev; } } guard{this, in_process};
  in_process = true;
  finish_copies(f);
  launch_scan(f);
  f.state = Slot::SEALED; sealed_order.push_back(f.idx);
  while (sealed_order.size() > 1) launch_slot(slot[sealed_order.front()]);
  if ((world > 1 && !fused) || (cfg.flags & DNZ_FLAG_SYNCHRONOUS)) while (!sealed_order.empty()) launch_slot(slot[sealed_order.front()]);
  const int next = (fill + 1) % NSLOT;
  if (slot[next].state == Slot::SEALED) launch_slot(slot[next]);
  if (slot[next].state == Slot::LAUNCHED) { while (!launched_order.empty() && slot[next].state == Slot::LAUNCHED) verify(slot[launched_order.front()]); }
  fill = next; slot[next].state = Slot::FILLING;
}

// enqueue everything that has been pushed (no host wait for the results)
void dnz_window::process_pending() {
  struct Guard { dnz_window* w; bool prev; ~Guard() { w->in_process = prev; } } guard{this, in_process};
  in_process = true;
  if (!cur().batches.empty()) seal_current();
  while (!sealed_order.empty()) launch_slot(slot[sealed_order.front()]);
}
// ... and make the host view exact: every launch verified, deferred rows replayed, input batches released
void dnz_window::drain() {
  struct Guard { dnz_window* w; bool prev; ~Guard() { w->in_process = prev; } } guard{this, in_process};
  in_process = true;
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
    CK(launch_ts_convert(s.d_ts_jobs.as<TsJob>(), (int)s.ts_jobs.size(), s.ts_max_rows, ts_source, ts_fmt, reinterpret_cast<uint32_t*>(ctl(CTL_TS_ERR)), stream));
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
  h_small.reserve(CTL_BYTES + 64);
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
    g.rows += nr; g.alg_bytes += 20.0 * nr + (double)b.key_bytes;
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

// pane pointer table + launch parameters of one aggregate / replay pass over the run
AggParams dnz_window::build_agg_params(Slot& s, const RunGeom& g, bool dirty, int64_t horizon, int out_list) {
  const int64_t np = g.pmax - g.pmin + 1;
  const size_t pb = (size_t)np * sizeof(void*);
  s.h_ptrs.reserve(7 * pb); s.d_ptrs.reserve(7 * pb);
  void** hp = s.h_ptrs.as<void*>();
  for (int64_t p = g.pmin; p <= g.pmax; p++) {
    const size_t k = (size_t)(p - g.pmin);
    Pane* m = (!dirty || p * pane_ms + L > horizon) ? find_pane(p) : nullptr;
    auto lit = late_panes.find(p); Pane* l = lit == late_panes.end() ? nullptr : lit->second.get();
    if (m) ensure_side_arrays(m);
    if (l) ensure_side_arrays(l);
    hp[0 * np + k] = m ? m->st.p : nullptr; hp[1 * np + k] = l ? l->st.p : nullptr;
    hp[2 * np + k] = m ? m->nullrows.p : nullptr; hp[3 * np + k] = l ? l->nullrows.p : nullptr;
    hp[4 * np + k] = m ? m->fz.p : nullptr; hp[5 * np + k] = l ? l->fz.p : nullptr;
    hp[6 * np + k] = reinterpret_cast<void*>((uintptr_t)(m ? (m->tag & 0xFFFFFFFFull) : 0));
  }
  CK(cudaMemcpyAsync(s.d_ptrs.p, hp, 7 * pb, cudaMemcpyHostToDevice, stream));
  CK(cudaMemsetAsync(ctl(s.ctl_off()), 0, 16, stream));        // deferred-row counter, flags, tile counter (not the emit-blocked flag)
  AggParams P;
  P.batches = s.d_batches.as<BatchDesc>(); P.tiles = s.d_tiles.as<TileDesc>(); P.tile_begin = g.t0; P.tile_end = g.t1;
  P.dict = dict_view();
  P.flags = ((cfg.flags & DNZ_FLAG_NO_HINTS) ? AGG_NO_HINTS : 0) | ((cfg.flags & DNZ_FLAG_NO_QUEUE) ? AGG_NO_QUEUE : 0);
  char* dp = s.d_ptrs.as<char>();
  P.panes.pane0 = g.pmin; P.panes.n_panes = (int32_t)np; P.panes.pad = 0; P.panes.pane_ms = pane_ms;
  P.panes.main = (GroupState* const*)(dp + 0 * pb); P.panes.late = (GroupState* const*)(dp + 1 * pb);
  P.panes.nullrows_main = (unsigned long long* const*)(dp + 2 * pb); P.panes.nullrows_late = (unsigned long long* const*)(dp + 3 * pb);
  P.panes.fz_main = (unsigned long long* const*)(dp + 4 * pb); P.panes.fz_late = (unsigned long long* const*)(dp + 5 * pb);
  P.panes.tag_main = (const unsigned long long*)(dp + 6 * pb);
  const size_t defer_cap = (size_t)std::max<int64_t>(g.rows, 1);
  s.d_defer[out_list].reserve(defer_cap * sizeof(DeferEntry));
  P.defer.entries = s.d_defer[out_list].as<DeferEntry>();
  P.defer.count = reinterpret_cast<unsigned long long*>(ctl(s.ctl_off())); P.defer.cap = defer_cap;
  P.defer.flags = reinterpret_cast<uint32_t*>(ctl(s.ctl_off() + 8));
  P.tile_counter = reinterpret_cast<uint32_t*>(ctl(s.ctl_off() + 12));
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
  else if (cfg.flags & DNZ_FLAG_FORCE_GENERIC) CK(launch_aggregate_generic(P, sm_count, stream));
  else CK(launch_aggregate(P, sm_count, stream));
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
      CK(cudaMemcpyAsync(h_small.p, ctl(0), 4, cudaMemcpyDeviceToHost, stream));
      CK(cudaStreamSynchronize(stream));
      const uint32_t clamp = std::min(*h_small.as<uint32_t>(), gcap);
      CK(cudaMemcpyAsync(ctl(0), &clamp, 4, cudaMemcpyHostToDevice, stream));
      CK(cudaStreamSynchronize(stream));
      dict_grow();
    }
    if (flags & DEFER_ARENA_FULL) {
      // the counter ran past the capacity by the bytes of every failed reservation (>= what the deferred rows need, and
      // never more than the key bytes of the run): pull it back to the capacity (the tail gap stays unused) and grow by that
      const uint64_t over = arena_used_host > arena_cap ? arena_used_host - arena_cap : 0;
      const uint64_t old_cap = arena_cap;
      CK(cudaMemcpyAsync(ctl(8), &old_cap, 8, cudaMemcpyHostToDevice, stream));
      CK(cudaStreamSynchronize(stream));
      arena_grow(arena_cap + std::min<uint64_t>(over, (uint64_t)g.alg_bytes) + (1 << 20));
    }
    if (flags & DEFER_NEED_FZ) need_fz = true;
    if (flags & DEFER_NEED_NULLROWS) need_nullrows = true;
    if (flags & (DEFER_NEED_FZ | DEFER_NEED_NULLROWS)) for_each_live_pane([&](Pane* p) { ensure_side_arrays(p); });
    const int out_list = in_list ^ 1;
    AggParams P = build_agg_params(s, g, dirty, horizon, out_list);
    CK(launch_deferred(P, s.d_defer[in_list].as<DeferEntry>(), n_in, stream));   // replays the rows of the previous pass
    stats.total_launches++;
    fetch_ctl();
    const char* h = h_small.as<char>() + s.ctl_off();
    n_in = *reinterpret_cast<const uint64_t*>(h); flags = *reinterpret_cast<const uint32_t*>(h + 8);
    in_list = out_list;
  }
  arena_trim();
}

// Aggregates one run and triggers, waiting for the device after the launch (late batches, several runs in one superbatch,
// exchange mode): the path the speculative one falls back to.
void dnz_window::execute_run_sync(Slot& s, const std::vector<BatchMinMax>& mm, const Run& r) {
  RunGeom g = run_geometry(s, mm, r);
  if (g.t1 <= g.t0) return;
  if (g.pmin <= g.pmax) {
    prepare_panes(s, mm, r, g);
    g_tr.mark("panes");
    AggParams P = build_agg_params(s, g, r.dirty, r.horizon, 0);
    launch_aggregate_pass(s, g, P, r.dirty);
    g_tr.mark("agg_launch");
    fetch_ctl();
    g_tr.mark("agg_wait");
    if (s.timed) { float ms = 0; CK(cudaEventElapsedTime(&ms, s.ev0, s.ev1)); stats.agg_kernel_ms += ms; stats.agg_algorithmic_bytes += s.alg_bytes; s.timed = false; }
    const char* h = h_small.as<char>() + s.ctl_off();
    defer_count_host = *reinterpret_cast<const uint64_t*>(h); defer_flags_host = *reinterpret_cast<const uint32_t*>(h + 8);
    if (defer_count_host) resolve_deferred(s, g, r.dirty, r.horizon);
  }
  g_tr.mark("post_agg");
  // ---- process_watermark + trigger_windows
  if (ungrouped) {
    ungrouped_emit_run(nullptr, &mm, &r, 0);
    if (r.dirty) {
      CK(cudaStreamSynchronize(stream));
      for (auto& kv : late_panes) if (pane_pool.size() < 16) pane_pool.push_back(std::move(kv.second));
      late_panes.clear();
    }
    g_tr.mark("emit");
    return;
  }
  if (r.dirty) {
    // windows that were already emitted (end <= horizon) and received rows from this batch are re-opened and emitted
    // again immediately with ONLY this batch's rows (§8a-3)
    std::set<int64_t> starts;
    for (auto& kv : late_panes)
      for (int j = 0; j < panes_per_window; j++) {
        int64_t st = (kv.first - j) * pane_ms;
        if (st >= 0 && st + L <= r.horizon) starts.insert(st);
      }
    std::map<int64_t, Pane*> src;
    for (auto& kv : late_panes) src[kv.first] = kv.second.get();
    emit_windows(std::vector<int64_t>(starts.begin(), starts.end()), src, false, nullptr);
    CK(cudaStreamSynchronize(stream));
    for (auto& kv : late_panes) if (pane_pool.size() < 16) pane_pool.push_back(std::move(kv.second));
    late_panes.clear();
  }
  if (world > 1) { if (!has_lwm || lwm <= r.wm_after) lwm = r.wm_after; has_lwm = true; }   // emission waits for the global watermark
  else emit_normal(r.wm_after, false, nullptr);
  g_tr.mark("emit");
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
      RunGeom g = run_geometry(s, mm, r);
      if (g.t1 > g.t0) {
        if (g.pmin <= g.pmax) {
          prepare_panes(s, mm, r, g);
          g_tr.mark("panes");
          AggParams P = build_agg_params(s, g, false, 0, 0);
          launch_aggregate_pass(s, g, P, false);
          g_tr.mark("agg_launch");
          s.speculative = true; s.t0 = g.t0; s.t1 = g.t1; s.pmin = g.pmin; s.pmax = g.pmax; s.rows_launched = g.rows;
        }
        if (world > 1) { if (!has_lwm || lwm <= r.wm_after) lwm = r.wm_after; has_lwm = true; }   // fused exchange: the group step emits under the GLOBAL watermark
        else if (ungrouped) ungrouped_emit_run(&s, &mm, &r, 0);
        else emit_normal(r.wm_after, true, &s);
        g_tr.mark("emit");
      }
    } else {
      for (const Run& r : runs) execute_run_sync(s, mm, r);
    }
  }
  CK(cudaMemcpyAsync(s.snap.p, d_ctl.p, CTL_BYTES, cudaMemcpyDeviceToHost, stream));
  CK(cudaEventRecord(s.done, stream));
  s.state = Slot::LAUNCHED; launched_order.push_back(s.idx);
  g_tr.flush("superbatch");
}

// Inspect the snapshot taken behind a slot's launches (waits for it if it has not been written yet).
void dnz_window::verify(Slot& s) {
  if (s.state != Slot::LAUNCHED) return;
  CK(cudaEventSynchronize(s.done));
  const char* h = s.snap.as<char>();
  parse_ctl(h);
  // what later launches may have added on top of this snapshot
  rows_since_known = 0;
  bool later = false;
  for (int i : launched_order) { if (i == s.idx) { later = true; continue; } if (later) rows_since_known += slot[i].rows_launched; }
  for (int k = 0; k < 2; k++) {
    uint64_t c = *reinterpret_cast<const uint64_t*>(h + rs[k].ctl_off);
    uint64_t rows = c >> 32, bytes = c & 0xFFFFFFFFull;
    later = false;
    for (int i : launched_order) { if (i == s.idx) { later = true; continue; } if (later && slot[i].emit_set == k) { rows += slot[i].add_rows_bound; bytes += slot[i].add_bytes_bound; } }
    rs[k].rows = rows; rs[k].bytes = bytes;
  }
  if (s.timed) { float ms = 0; CK(cudaEventElapsedTime(&ms, s.ev0, s.ev1)); stats.agg_kernel_ms += ms; stats.agg_algorithmic_bytes += s.alg_bytes; s.timed = false; }
  if (s.speculative) {
    const char* hs = h + s.ctl_off();
    defer_count_host = *reinterpret_cast<const uint64_t*>(hs); defer_flags_host = *reinterpret_cast<const uint32_t*>(hs + 8);
    bool blocked = *reinterpret_cast<const uint32_t*>(hs + 16) != 0;
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
      CK(cudaMemsetAsync(ctl(s.ctl_off() + 16), 0, 4, stream));
      if (!s.emit_starts.empty()) emit_windows(s.emit_starts, pane_sources(), false, nullptr);
    }
  }
  release_slot(s);
}

void dnz_window::release_slot(Slot& s) {
  if (s.copies) cudaEventSynchronize(s.copy_done);
  for (auto& pb : s.batches) if (pb.has_moved && pb.moved.release) pb.moved.release(&pb.moved);
  s.batches.clear(); s.gather.clear(); s.ts_jobs.clear(); s.ts_max_rows = 0; s.rows = 0; s.copies = false; s.arena.reset(); s.scanned = false; s.n_tiles = 0;
  for (auto& p : s.retired) if (pane_pool.size() < 16) pane_pool.push_back(std::move(p));
  s.retired.clear(); s.emit_starts.clear(); s.speculative = false; s.add_rows_bound = s.add_bytes_bound = 0; s.rows_launched = 0;
  auto it = std::find(launched_order.begin(), launched_order.end(), s.idx);
  if (it != launched_order.end()) launched_order.erase(it);
  s.state = Slot::FREE;
}

void dnz_window::emit_normal(int64_t wm_new, bool gated, Slot* sl) {
  if (!has_wm || wm <= wm_new) { wm = wm_new; has_wm = true; }
  std::set<int64_t> starts;
  for (auto& kv : panes)
    for (int j = 0; j < panes_per_window; j++) {
      int64_t s = (kv.first - j) * pane_ms;
      if (s >= 0 && s + L <= wm && s + L > emitted_upto) starts.insert(s);
    }
  std::map<int64_t, Pane*> src;
  for (auto& kv : panes) src[kv.first] = kv.second.get();
  emit_windows(std::vector<int64_t>(starts.begin(), starts.end()), src, gated, sl);
  emitted_upto = std::max(emitted_upto, wm);
  retire_panes(gated ? sl : nullptr);
}

void dnz_window::ensure_result_capacity(uint64_t add_rows, uint64_t add_bytes) {
  uint64_t need_rows = R().rows + add_rows, need_bytes = R().bytes + add_bytes;
  if (need_bytes >= (1ull << 31) || need_rows >= (1ull << 32)) {
    // the bound may be stale: make it exact before giving up
    drain(); fetch_ctl();
    need_rows = R().rows + add_rows; need_bytes = R().bytes + add_bytes;
    if (need_bytes >= (1ull << 31)) fail(DNZ_ERR_UNSUPPORTED, "more than 2 GiB of key bytes between polls (Utf8 offsets are 32-bit); poll more often");
  }
  if (need_rows <= R().row_cap && need_bytes <= R().byte_cap) return;
  auto grow = [&](DevBuf& b, size_t elem, uint64_t used, uint64_t cap) { b.regrow_on(stream, (size_t)cap * elem + 64, b.p ? (size_t)used * elem : 0); };
  if (need_rows > R().row_cap) {
    uint64_t cap = std::max<uint64_t>(need_rows, R().row_cap + R().row_cap / 2);
    const uint64_t used = std::min(R().rows, R().row_cap);
    grow(R().key_off, 4, used, cap + 1); grow(R().key_valid, 1, used, cap); grow(R().count, 8, used, cap);
    grow(R().mn, 8, used, cap); grow(R().mx, 8, used, cap); grow(R().avg, 8, used, cap); grow(R().sum, 8, used, cap);
    grow(R().agg_valid, 1, used, cap); grow(R().wstart, 8, used, cap); grow(R().wend, 8, used, cap);
    R().row_cap = cap;
  }
  if (need_bytes > R().byte_cap) {
    uint64_t cap = std::max<uint64_t>(need_bytes, R().byte_cap + R().byte_cap / 2);
    grow(R().key_bytes, 1, std::min(R().bytes, R().byte_cap), cap);
    R().byte_cap = cap;
  }
}

void dnz_window::reset_set(int i) {
  ResultSet& r = rs[i];
  CK(cudaMemsetAsync(ctl(r.ctl_off), 0, 16, stream));
  r.rows = 0; r.bytes = 0; r.exp_rows = 0; r.exp_bytes = 0; r.snap_issued = false;
  for (Slot& s : slot) if (s.emit_set == i) { s.add_rows_bound = 0; s.add_bytes_bound = 0; }
}
void dnz_window::reset_results() { reset_set(wr); res_consumed = false; }

// cursor of the current set -> pinned memory, in stream order behind the emit launches
void dnz_window::snapshot_results() {
  ResultSet& r = R();
  CK(cudaMemcpyAsync(r.snap.p, ctl(r.ctl_off), 16, cudaMemcpyDeviceToHost, stream));
  CK(cudaEventRecord(r.snap_ev, stream));
  r.snap_issued = true;
}
// every row of the set has been handed out and nothing is in flight for it
bool dnz_window::set_drained(ResultSet& r) {
  if (!r.snap_issued) return r.exp_rows == r.rows;
  if (cudaEventQuery(r.snap_ev) != cudaSuccess) { cudaGetLastError(); return false; }
  uint64_t c = *reinterpret_cast<volatile uint64_t*>(r.snap.p);
  return (c >> 32) == r.exp_rows;
}
// Called before a superbatch's emits are enqueued (only matters when the consumer uses the non-blocking poll): reuse the
// current set in place when it is drained, else switch to the other one if that is drained, else keep appending.
void dnz_window::rotate_result_sets() {
  if (!async_polls) return;
  if (set_drained(rs[wr])) { if (rs[wr].exp_rows) reset_set(wr); return; }
  if (set_drained(rs[wr ^ 1])) { if (rs[wr ^ 1].exp_rows || rs[wr ^ 1].rows) reset_set(wr ^ 1); wr ^= 1; }
}

// One k_emit launch per window: combine its panes, apply the fused FilterExec predicate, compact.  `gated`: the launches do
// nothing (and raise the slot's emit-blocked flag) when any pipeline slot holds deferred rows at the time they run.
void dnz_window::emit_windows(const std::vector<int64_t>& starts, const std::map<int64_t, Pane*>& src, bool gated, Slot* sl) {
  if (starts.empty()) return;
  const uint32_t ng = groups_bound();
  if (ng == 0) return;
  const uint64_t add_rows = (uint64_t)starts.size() * ng, add_bytes = (uint64_t)starts.size() * key_bytes_bound();
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
    E.wstart = s; E.wend = s + L; E.n_groups = ng; E.rank = rank; E.world = world;
    E.dict = dict_view();
    E.gate = gated ? reinterpret_cast<const unsigned long long*>(ctl(64)) : nullptr;
    E.blocked = gated && sl ? reinterpret_cast<uint32_t*>(ctl(sl->ctl_off() + 16)) : nullptr;
    E.out.key_off = R().key_off.as<int32_t>(); E.out.key_bytes = R().key_bytes.as<uint8_t>(); E.out.key_valid = R().key_valid.as<uint8_t>();
    E.out.count = R().count.as<int64_t>(); E.out.mn = R().mn.as<double>(); E.out.mx = R().mx.as<double>(); E.out.avg = R().avg.as<double>();
    E.out.sum = R().sum.as<double>(); E.out.agg_valid = R().agg_valid.as<uint8_t>(); E.out.wstart = R().wstart.as<int64_t>(); E.out.wend = R().wend.as<int64_t>();
    E.out.cursor = reinterpret_cast<unsigned long long*>(ctl(R().ctl_off)); E.out.row_cap = R().row_cap; E.out.byte_cap = R().byte_cap;
    E.out.overflow = reinterpret_cast<uint32_t*>(ctl(R().ctl_off + 8));
    CK(launch_emit(E, stream));
    stats.total_launches++; stats.windows_emitted++;
  }
  R().rows += add_rows; R().bytes += add_bytes;
  if (sl && gated) {
    sl->emit_starts.insert(sl->emit_starts.end(), starts.begin(), starts.end());
    sl->add_rows_bound += add_rows; sl->add_bytes_bound += add_bytes; sl->emit_set = wr;
  }
  snapshot_results();
}

// ------------------------------------------------------------------------------------------------
void dnz_window::fill_schema(ArrowSchema* schema) {
  auto* sp = new SchemaPrivate();
  size_t nc = (ungrouped ? 0 : 1) + aggs.size() + 2;
  sp->names.reserve(nc);
  auto add = [&](const std::string& name, const char* fmt, int64_t flags) {
    sp->names.push_back(name);
    auto c = std::make_unique<ArrowSchema>();
    memset(c.get(), 0, sizeof(ArrowSchema));
    c->format = fmt; c->flags = flags; c->release = release_child_schema;
    sp->children.push_back(std::move(c));
  };
  if (!ungrouped) add(key_name, "u", ARROW_FLAG_NULLABLE);
  for (size_t i = 0; i < aggs.size(); i++) add(aliases[i], agg_format(aggs[i].kind), aggs[i].kind == DNZ_AGG_COUNT ? 0 : ARROW_FLAG_NULLABLE);
  add("window_start_time", "tsm:", 0);     // continuous/mod.rs:42-62: Timestamp(ms, None), non-null
  add("window_end_time", "tsm:", 0);
  for (size_t i = 0; i < nc; i++) { sp->children[i]->name = sp->names[i].c_str(); sp->child_ptrs.push_back(sp->children[i].get()); }
  memset(schema, 0, sizeof(*schema));
  schema->format = "+s"; schema->name = ""; schema->n_children = (int64_t)nc; schema->children = sp->child_ptrs.data();
  schema->release = release_schema; schema->private_data = sp;
}


// Hands out every emitted row that is COMPLETE on the device: per result set, the rows between what was exported before and
// the newest snapshot whose event has fired (older set first).  `blocking` callers have synchronised the stream, so every
// snapshot has fired; the non-blocking poll simply leaves rows of still-running emits for the next call.  The device->host
// copies run on their own stream, never behind queued input.
void dnz_window::export_arrow(ArrowArray* out, ArrowSchema* schema, int32_t* has_output, bool blocking) {
  if (ungrouped) { export_ungrouped(out, schema, has_output, blocking); return; }
  if (blocking) { CK(cudaStreamSynchronize(stream)); }
  else {
    while (!launched_order.empty() && cudaEventQuery(slot[launched_order.front()].done) == cudaSuccess) verify(slot[launched_order.front()]);
    cudaGetLastError();
  }
  struct Range { ResultSet* r; uint64_t r0, r1, b0, b1; };
  std::vector<Range> ranges;
  for (int k = 0; k < 2; k++) {
    ResultSet& r = rs[k == 0 ? (wr ^ 1) : wr];
    if (!r.snap_issued) continue;
    if (cudaEventQuery(r.snap_ev) != cudaSuccess) { cudaGetLastError(); continue; }
    const volatile uint64_t* sp = reinterpret_cast<volatile uint64_t*>(r.snap.p);
    const uint64_t c = sp[0];
    if (static_cast<uint32_t>(sp[1])) fail(DNZ_ERR_NOMEM, "result buffer overflow (internal sizing error)");
    const uint64_t rows = c >> 32, bytes = c & 0xFFFFFFFFull;
    if (rows > r.exp_rows) ranges.push_back(Range{&r, r.exp_rows, rows, r.exp_bytes, bytes});
  }
  uint64_t n = 0, nbytes = 0;
  for (auto& g : ranges) { n += g.r1 - g.r0; nbytes += g.b1 - g.b0; }
  if (nbytes >= (1ull << 31)) fail(DNZ_ERR_UNSUPPORTED, "more than 2 GiB of key bytes in one poll (Utf8 offsets are 32-bit); poll more often");
  auto* ep = new ExportPrivate();
  std::unique_ptr<ExportPrivate> guard(ep);
  const size_t total = round_up((n + 1) * 4, 64) + round_up(nbytes, 64) + 2 * round_up(n, 64) + 7 * round_up(n * 8, 64) +
                       2 * round_up((n + 7) / 8 + 8, 64) + 1024;
  ep->block = g_pinned_pool.get(total, ep->block_cap);
  size_t used = 0;
  auto pinned = [&](size_t bytes) -> void* { void* p = (char*)ep->block + used; used += round_up(std::max<size_t>(bytes, 8), 64); return p; };
  // one column of every range, back to back
  auto fetch = [&](DevBuf ResultSet::*col, size_t elem, bool by_bytes, size_t extra) -> void* {
    char* h = (char*)pinned((by_bytes ? nbytes : n) * elem + extra);
    size_t at = 0;
    for (auto& g : ranges) {
      const uint64_t lo = by_bytes ? g.b0 : g.r0, hi = by_bytes ? g.b1 : g.r1;
      const size_t bytes = (size_t)(hi - lo) * elem;
      if (bytes) { CK(cudaMemcpyAsync(h + at, (g.r->*col).template as<char>() + lo * elem, bytes, cudaMemcpyDeviceToHost, d2h_stream)); stats.d2h_bytes += (int64_t)bytes; }
      at += bytes;
    }
    return h;
  };
  int32_t* koff = (int32_t*)fetch(&ResultSet::key_off, 4, false, 4);
  uint8_t* kbytes = (uint8_t*)fetch(&ResultSet::key_bytes, 1, true, 0);
  uint8_t* kvalid = (uint8_t*)fetch(&ResultSet::key_valid, 1, false, 0);
  int64_t* count = (int64_t*)fetch(&ResultSet::count, 8, false, 0);
  double* mn = (double*)fetch(&ResultSet::mn, 8, false, 0); double* mx = (double*)fetch(&ResultSet::mx, 8, false, 0);
  double* avg = (double*)fetch(&ResultSet::avg, 8, false, 0); double* sum = (double*)fetch(&ResultSet::sum, 8, false, 0);
  uint8_t* avalid = (uint8_t*)fetch(&ResultSet::agg_valid, 1, false, 0);
  int64_t* ws = (int64_t*)fetch(&ResultSet::wstart, 8, false, 0); int64_t* we = (int64_t*)fetch(&ResultSet::wend, 8, false, 0);
  CK(cudaStreamSynchronize(d2h_stream));
  {   // key offsets are relative to each set's byte buffer: rebase them onto the concatenated export
    uint64_t row_at = 0, byte_at = 0;
    for (auto& g : ranges) {
      const int64_t delta = (int64_t)byte_at - (int64_t)g.b0;
      if (delta != 0) for (uint64_t i = row_at; i < row_at + (g.r1 - g.r0); i++) koff[i] = (int32_t)(koff[i] + delta);
      row_at += g.r1 - g.r0; byte_at += g.b1 - g.b0;
    }
  }
  koff[n] = (int32_t)nbytes;
  // byte-per-row validity -> Arrow bitmaps
  auto pack = [&](const uint8_t* v, int64_t& nulls) -> uint8_t* {
    nulls = 0;
    for (uint64_t i = 0; i < n; i++) nulls += !v[i];
    if (!nulls) return nullptr;
    uint8_t* bm = (uint8_t*)pinned((n + 7) / 8 + 8);
    memset(bm, 0, (n + 7) / 8 + 8);
    for (uint64_t i = 0; i < n; i++) if (v[i]) bm[i >> 3] |= (uint8_t)(1u << (i & 7));
    return bm;
  };
  int64_t key_nulls = 0, agg_nulls = 0;
  uint8_t* kbm = pack(kvalid, key_nulls);
  uint8_t* abm = pack(avalid, agg_nulls);
  size_t nc = 1 + aggs.size() + 2;
  auto add_child = [&](std::vector<const void*> bufs, int64_t nulls) {
    ep->buffers.push_back(std::move(bufs));
    auto c = std::make_unique<ArrowArray>();
    memset(c.get(), 0, sizeof(ArrowArray));
    c->length = (int64_t)n; c->null_count = nulls; c->n_buffers = (int64_t)ep->buffers.back().size();
    c->buffers = ep->buffers.back().data(); c->release = release_child;
    ep->children.push_back(std::move(c));
  };
  ep->buffers.reserve(nc + 1);
  add_child({kbm, koff, kbytes}, key_nulls);
  for (auto& a : aggs) {
    switch (a.kind) {
      case DNZ_AGG_COUNT: add_child({nullptr, count}, 0); break;
      case DNZ_AGG_MIN: add_child({abm, mn}, agg_nulls); break;
      case DNZ_AGG_MAX: add_child({abm, mx}, agg_nulls); break;
      case DNZ_AGG_AVG: add_child({abm, avg}, agg_nulls); break;
      default: add_child({abm, sum}, agg_nulls); break;
    }
  }
  add_child({nullptr, ws}, 0);
  add_child({nullptr, we}, 0);
  for (auto& c : ep->children) ep->child_ptrs.push_back(c.get());
  ep->buffers.push_back({nullptr});
  memset(out, 0, sizeof(*out));
  out->length = (int64_t)n; out->null_count = 0; out->n_buffers = 1; out->buffers = ep->buffers.back().data();
  out->n_children = (int64_t)nc; out->children = ep->child_ptrs.data(); out->release = release_array;
  out->private_data = guard.release();
  if (schema) fill_schema(schema);
  if (has_output) *has_output = n > 0;
  stats.rows_out += (int64_t)n;
  for (auto& g : ranges) { g.r->exp_rows = g.r1; g.r->exp_bytes = g.b1; }
  if (blocking) {         // stream idle: drained sets can be recycled right away
    for (int i = 0; i < 2; i++) if (rs[i].exp_rows && set_drained(rs[i])) reset_set(i);
  }
}

// Device-resident hand-over: the oldest range of emitted rows that has not been handed out yet, one result set per call (call
// again until n_rows == 0 when both sets may hold rows).  blocking: everything has been aggregated and the stream is idle, so
// every emitted row is eligible.  Non-blocking: only rows whose emission is COMPLETE on the device; nothing queued is forced.
// key_off entries are offsets into `key_bytes` (the set's byte buffer); key_bytes_len is the offset at which the last returned
// key ends.
void dnz_window::export_device(dnz_device_result* out, bool blocking) {
  if (ungrouped) fail(DNZ_ERR_UNSUPPORTED, "ungrouped windows finish on the host (Final stage): use dnz_window_poll / dnz_window_poll_ready");
  memset(out, 0, sizeof *out);
  ResultSet* r = nullptr; uint64_t r0 = 0, r1 = 0, b1 = 0;
  if (blocking) fetch_ctl();
  else {
    // release the input of launches that have completed (never waits)
    while (!launched_order.empty() && cudaEventQuery(slot[launched_order.front()].done) == cudaSuccess) verify(slot[launched_order.front()]);
    cudaGetLastError();
  }
  for (int k = 0; k < 2 && !r; k++) {
    ResultSet& c = rs[k == 0 ? (wr ^ 1) : wr];
    uint64_t rows = c.rows, bytes = c.bytes;
    if (!blocking) {
      if (!c.snap_issued) continue;
      if (cudaEventQuery(c.snap_ev) != cudaSuccess) { cudaGetLastError(); continue; }
      const volatile uint64_t* sp = reinterpret_cast<volatile uint64_t*>(c.snap.p);
      const uint64_t cur = sp[0];
      if (static_cast<uint32_t>(sp[1])) fail(DNZ_ERR_NOMEM, "result buffer overflow (internal sizing error)");
      rows = cur >> 32; bytes = cur & 0xFFFFFFFFull;
    }
    if (rows > c.exp_rows) { r = &c; r0 = c.exp_rows; r1 = rows; b1 = bytes; }
  }
  if (!r) return;
  r->exp_rows = r1; r->exp_bytes = b1;
  if (blocking) {          // stream idle: a set that has been handed out completely restarts at row 0 with the next emission
    for (int i = 0; i < 2; i++) if (rs[i].exp_rows && rs[i].exp_rows == rs[i].rows) reset_set(i);
  }
  out->n_rows = (int64_t)(r1 - r0); out->key_bytes_len = (int64_t)b1;
  out->key_off = r->key_off.as<int32_t>() + r0; out->key_bytes = r->key_bytes.as<uint8_t>(); out->key_valid = r->key_valid.as<uint8_t>() + r0;
  out->count = r->count.as<int64_t>() + r0; out->min = r->mn.as<double>() + r0; out->max = r->mx.as<double>() + r0;
  out->avg = r->avg.as<double>() + r0; out->sum = r->sum.as<double>() + r0; out->agg_valid = r->agg_valid.as<uint8_t>() + r0;
  out->window_start_ms = r->wstart.as<int64_t>() + r0; out->window_end_ms = r->wend.as<int64_t>() + r0;
  stats.rows_out += (int64_t)(r1 - r0);
}


// ------------------------------------------------------------------------------------------------

// ------------------------------------------------------------------------------------------------
// ungrouped windows (include/dnz_gpu.h, DNZ_NO_KEY)
namespace {
// get_windows_for_watermark (streaming_window.rs:1053-1086), whole-second snap (:1088-1094): the frames a batch creates
void reference_windows(int64_t mn, int64_t mx, int64_t L, int64_t S, std::vector<int64_t>& out) {
  auto snap = [&](int64_t ts) { const int64_t wl = L / 1000, t = ts / 1000; return (t / wl) * wl * 1000; };
  if (S > 0) { for (int64_t cur = snap(mn - L); cur <= mx; cur += S) { const int64_t end = cur + L; if (mn > end || mx < cur) continue; out.push_back(cur); } }
  else for (int64_t cur = snap(mn); cur <= mx; cur += L) out.push_back(cur);
}
inline unsigned long long unord_bits_h(unsigned long long o) { return (o & 0x8000000000000000ull) ? (o & ~0x8000000000000000ull) : ~o; }
inline int total_cmp_d(double a, double b) {
  long long x, y; memcpy(&x, &a, 8); memcpy(&y, &b, 8);
  x ^= (long long)(((unsigned long long)(x >> 63)) >> 1); y ^= (long long)(((unsigned long long)(y >> 63)) >> 1);
  return x < y ? -1 : x > y ? 1 : 0;
}
}  // namespace

// The Partial stage's emission schedule for one run (or a flush): per batch, the frames it creates and the frames its watermark
// closes -- one "partial batch" (PB) per batch, exactly what WindowAggStream::trigger_windows hands to the Final stage -- and the
// collection of the closed windows' states from the device (one kernel + one small D2H per run).
void dnz_window::ungrouped_emit_run(Slot* sl, const std::vector<BatchMinMax>* mm, const Run* r, int64_t flush_wm) {
  UEmission em;
  std::vector<std::pair<int64_t, bool>> wins;          // (window start, from the late panes)
  auto close_upto = [&](int64_t w, int64_t horizon, bool dirty) {
    std::vector<int64_t> pb;
    for (auto it = u_created.begin(); it != u_created.end();) {
      if (*it + L <= w) { pb.push_back(*it); wins.emplace_back(*it, dirty && *it + L <= horizon); it = u_created.erase(it); } else ++it;
    }
    if (!pb.empty()) em.pbs.push_back(std::move(pb));
  };
  if (r) {
    std::vector<int64_t> tmp;
    for (size_t i = r->b0; i < r->b1; i++) {
      const BatchMinMax& b = (*mm)[i];
      if (b.n_valid == 0) continue;
      tmp.clear(); reference_windows(b.ts_min, b.ts_max, L, S, tmp);
      for (int64_t st : tmp) u_created.insert(st);
      if (!has_wm || wm <= b.ts_min) { wm = b.ts_min; has_wm = true; }       // process_watermark
      close_upto(wm, r->horizon, r->dirty);
    }
  } else {                                             // dnz_window_flush (tests): one trigger at the given watermark
    if (!has_wm || wm <= flush_wm) { wm = flush_wm; has_wm = true; }
    close_upto(wm, 0, false);
  }
  if (!wins.empty()) {
    const size_t n = wins.size();
    if (n > u_ring) fail(DNZ_ERR_UNSUPPORTED, "%zu windows closed by one run (limit %zu)", n, u_ring);
    if (u_head + n > u_ring) { ungrouped_collect(true); u_head = 0; }              // staging full: take in what is on its way first
    const size_t at = u_head;
    UWindow* hw = h_uwins.as<UWindow>() + at;
    for (size_t i = 0; i < n; i++) {
      UWindow& W = hw[i]; memset(&W, 0, sizeof W);
      const int64_t p0 = wins[i].first / pane_ms;
      W.n = panes_per_window;
      for (int j = 0; j < panes_per_window; j++) {
        Pane* pn = nullptr;
        if (wins[i].second) { auto it = late_panes.find(p0 + j); if (it != late_panes.end()) pn = it->second.get(); }
        else pn = find_pane(p0 + j);
        W.st[j] = pn ? pn->st.as<GroupState>() : nullptr; W.nr[j] = pn ? pn->nullrows.as<unsigned long long>() : nullptr;
      }
    }
    CK(cudaMemcpyAsync(d_uwins.as<UWindow>() + at, hw, n * sizeof(UWindow), cudaMemcpyHostToDevice, stream));
    CK(launch_ungrouped_collect(d_uwins.as<UWindow>() + at, (int)n, d_ustates.as<UState>() + at, stream)); stats.total_launches++;
    CK(cudaMemcpyAsync(h_ustates.as<UState>() + at, d_ustates.as<UState>() + at, n * sizeof(UState), cudaMemcpyDeviceToHost, stream));
    if (u_event_pool.empty()) { cudaEvent_t e; CK(cudaEventCreateWithFlags(&e, cudaEventDisableTiming)); u_event_pool.push_back(e); }
    em.ev = u_event_pool.back(); u_event_pool.pop_back();
    CK(cudaEventRecord(em.ev, stream));
    em.first = at; em.count = n; u_head += n;
    stats.windows_emitted += (int64_t)n;
    u_pending.push_back(std::move(em));
  }
  emitted_upto = std::max(emitted_upto, wm);
  retire_panes(sl);
}

// FullWindowAggStream::poll_next_inner (streaming_window.rs:934-1032) for one partial batch
void dnz_window::ungrouped_final(const std::vector<URow>& pb) {
  if (pb.empty()) return;
  int64_t start = pb[0].ws, end = pb[0].we;
  for (const URow& x : pb) { start = std::max(start, x.ws); end = std::max(end, x.we); }      // "these batches should only have 1 row"
  const bool cached = u_final.count(start) != 0;
  if (u_seen.count(start) && !cached) return;                                                // late data for a finalized window: dropped
  UFrame& f = u_final[start];
  if (!cached) f.end = end;
  u_seen.insert(start);
  for (const URow& x : pb) {                               // merge_batch of every row of the batch into THAT frame
    f.cnt += (uint64_t)x.cnt;
    if (x.valid) {
      f.sum += x.sum;
      if (!f.has) { f.mn = x.mn; f.mx = x.mx; f.has = true; }
      else { if (total_cmp_d(x.mn, f.mn) < 0) f.mn = x.mn; if (total_cmp_d(x.mx, f.mx) > 0) f.mx = x.mx; }
    }
  }
  if (!u_has_fwm || start > u_fwm) { u_fwm = start; u_has_fwm = true; }
  for (auto it = u_final.begin(); it != u_final.end();) {                                    // finalize_windows: watermark > window end
    if (u_fwm > it->second.end) {
      const UFrame& g = it->second;
      u_out.push_back(URow{it->first, g.end, (int64_t)g.cnt, g.has ? g.mn : 0.0, g.has ? g.mx : 0.0, g.has ? g.sum / (double)g.cnt : 0.0, g.sum, g.has});
      it = u_final.erase(it);
    } else ++it;
  }
}

// feed the partial batches whose states have arrived to the Final stage (in emission order)
void dnz_window::ungrouped_collect(bool wait) {
  while (!u_pending.empty()) {
    UEmission& em = u_pending.front();
    if (wait) CK(cudaEventSynchronize(em.ev));
    else if (cudaEventQuery(em.ev) != cudaSuccess) { cudaGetLastError(); break; }
    const UState* st = h_ustates.as<UState>() + em.first;
    size_t k = 0;
    for (const auto& pb : em.pbs) {
      std::vector<URow> rows;
      for (int64_t ws : pb) {
        const UState& u = st[k++];
        URow x; x.ws = ws; x.we = ws + L; x.cnt = (int64_t)u.cnt; x.valid = u.cnt != 0; x.sum = u.sum; x.avg = 0;
        unsigned long long bmn = unord_bits_h(~u.mink), bmx = unord_bits_h(u.maxk);
        memcpy(&x.mn, &bmn, 8); memcpy(&x.mx, &bmx, 8);
        rows.push_back(x);
      }
      ungrouped_final(rows);
    }
    u_event_pool.push_back(em.ev);
    u_pending.pop_front();
    if (u_pending.empty()) u_head = 0;
  }
}

void dnz_window::export_ungrouped(ArrowArray* out, ArrowSchema* schema, int32_t* has_output, bool blocking) {
  if (blocking) CK(cudaStreamSynchronize(stream));
  else { while (!launched_order.empty() && cudaEventQuery(slot[launched_order.front()].done) == cudaSuccess) verify(slot[launched_order.front()]); cudaGetLastError(); }
  ungrouped_collect(blocking);
  const size_t n = u_out.size();
  auto* ep = new ExportPrivate();
  std::unique_ptr<ExportPrivate> guard(ep);
  const size_t total = 8 * round_up(n * 8 + 8, 64) + round_up((n + 7) / 8 + 8, 64) + 1024;
  ep->block = g_pinned_pool.get(total, ep->block_cap);
  size_t used = 0;
  auto take = [&](size_t bytes) -> void* { void* p = (char*)ep->block + used; used += round_up(std::max<size_t>(bytes, 8), 64); return p; };
  int64_t* cnt = (int64_t*)take(n * 8); double* mn = (double*)take(n * 8); double* mx = (double*)take(n * 8); double* avg = (double*)take(n * 8);
  double* sum = (double*)take(n * 8); int64_t* ws = (int64_t*)take(n * 8); int64_t* we = (int64_t*)take(n * 8);
  uint8_t* bm = (uint8_t*)take((n + 7) / 8 + 8); memset(bm, 0, (n + 7) / 8 + 8);
  int64_t nulls = 0;
  for (size_t i = 0; i < n; i++) {
    const URow& x = u_out[i];
    cnt[i] = x.cnt; mn[i] = x.mn; mx[i] = x.mx; avg[i] = x.avg; sum[i] = x.valid ? x.sum : 0.0; ws[i] = x.ws; we[i] = x.we;
    if (x.valid) bm[i >> 3] |= (uint8_t)(1u << (i & 7)); else nulls++;
  }
  uint8_t* abm = nulls ? bm : nullptr;
  auto add_child = [&](std::vector<const void*> bufs, int64_t nl) {
    ep->buffers.push_back(std::move(bufs));
    auto c = std::make_unique<ArrowArray>(); memset(c.get(), 0, sizeof(ArrowArray));
    c->length = (int64_t)n; c->null_count = nl; c->n_buffers = (int64_t)ep->buffers.back().size();
    c->buffers = ep->buffers.back().data(); c->release = release_child;
    ep->children.push_back(std::move(c));
  };
  ep->buffers.reserve(aggs.size() + 4);
  for (auto& a : aggs) {
    switch (a.kind) {
      case DNZ_AGG_COUNT: add_child({nullptr, cnt}, 0); break;
      case DNZ_AGG_MIN: add_child({abm, mn}, nulls); break;
      case DNZ_AGG_MAX: add_child({abm, mx}, nulls); break;
      case DNZ_AGG_AVG: add_child({abm, avg}, nulls); break;
      default: add_child({abm, sum}, nulls); break;
    }
  }
  add_child({nullptr, ws}, 0); add_child({nullptr, we}, 0);
  for (auto& c : ep->children) ep->child_ptrs.push_back(c.get());
  ep->buffers.push_back({nullptr});
  memset(out, 0, sizeof(*out));
  out->length = (int64_t)n; out->n_buffers = 1; out->buffers = ep->buffers.back().data();
  out->n_children = (int64_t)ep->children.size(); out->children = ep->child_ptrs.data(); out->release = release_array;
  out->private_data = guard.release();
  if (schema) fill_schema(schema);
  if (has_output) *has_output = n > 0;
  stats.rows_out += (int64_t)n;
  u_out.clear();
}

// ------------------------------------------------------------------------------------------------
// checkpoint / restore (include/dnz_gpu.h)
namespace {
struct CkptHeader {
  char magic[8];                 // "DNZCKPT1"
  int64_t window_ms, slide_ms; int32_t n_aggs, flags;          // flags: 1 has_wm, 2 need_nullrows, 4 need_fz, 8 has_lwm
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
  const char* h = h_small.as<char>();
  CkptHeader H; memset(&H, 0, sizeof H);
  memcpy(H.magic, "DNZCKPT1", 8);
  H.window_ms = L; H.slide_ms = S; H.n_aggs = (int32_t)aggs.size();
  H.flags = (has_wm ? 1 : 0) | (need_nullrows ? 2 : 0) | (need_fz ? 4 : 0) | (has_lwm ? 8 : 0);
  H.wm = wm; H.emitted_upto = emitted_upto; H.next_seq = next_seq; H.lwm = lwm; H.exported_pane_upto = exported_pane_upto;
  H.n_groups = n_groups_host; H.null_gid_plus1 = *reinterpret_cast<const uint32_t*>(h + 4);
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
  const size_t ng = H.n_groups, ab = round_up(H.arena_used, 8);
  const char* p = blob + sizeof H; const char* end = blob + bytes;
  auto need = [&](size_t n) { if ((size_t)(end - p) < n) fail(DNZ_ERR_INVALID, "checkpoint blob truncated"); };
  CK(cudaStreamSynchronize(stream));
  while (gcap < ng + ng / 8 + 1) dict_grow();                      // (nothing to rehash yet)
  if (ab + (1 << 20) > arena_cap) arena_grow(ab + (1 << 20));
  need(ng * sizeof(GidKey)); if (ng) CK(cudaMemcpy(gid_key.p, p, ng * sizeof(GidKey), cudaMemcpyHostToDevice)); p += ng * sizeof(GidKey);
  need(ab); if (ab) CK(cudaMemcpy(arena.p, p, ab, cudaMemcpyHostToDevice)); p += ab;
  struct { uint32_t n_groups, null_gid; uint64_t arena_used, key_bytes_total; } c0{H.n_groups, 0u, H.arena_used, H.key_bytes_total};
  CK(cudaMemcpy(ctl(0), &c0, sizeof c0, cudaMemcpyHostToDevice));
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

// ------------------------------------------------------------------------------------------------
// pane exchange (see include/dnz_gpu.h)
void dnz_window::export_partials(int64_t watermark, dnz_partials* out) {
  process_pending(); drain();
  memset(out, 0, sizeof *out);
  h_owner_counts.assign((size_t)world, 0); h_owner_bytes.assign((size_t)world, 0);
  out->owner_counts = h_owner_counts.data(); out->owner_key_bytes = h_owner_bytes.data();
  out->pane_lo = 0; out->pane_hi = -1;
  if (watermark == INT64_MIN) return;
  const int64_t hi = floor_div(watermark, pane_ms) - 1;          // panes with end <= watermark
  int64_t lo = exported_pane_upto == INT64_MIN ? (panes.empty() ? hi + 1 : panes.begin()->first) : exported_pane_upto + 1;
  if (hi < lo) return;
  std::vector<Pane*> send;
  for (auto& kv : panes) if (kv.first >= lo && kv.first <= hi) send.push_back(kv.second.get());
  out->pane_lo = lo; out->pane_hi = hi;
  exported_pane_upto = hi;
  if (send.empty()) return;
  fetch_ctl();
  if (n_groups_host == 0) return;
  d_owner_cursor.reserve((size_t)world * 8);
  h_small.reserve((size_t)std::max(256, world * 8));
  PackParams P; memset(&P, 0, sizeof P);
  P.n_groups = n_groups_host; P.rank = rank; P.world = world; P.dict = dict_view();
  P.owner_cursor = d_owner_cursor.as<unsigned long long>();
  auto run_pass = [&](int pass) {
    CK(cudaMemsetAsync(d_owner_cursor.p, 0, (size_t)world * 8, stream));
    P.pass = pass;
    for (Pane* p : send) {
      P.st = p->st.as<GroupState>(); P.nullrows = p->nullrows.as<unsigned long long>(); P.fz = p->fz.as<unsigned long long>(); P.pane = p->id;
      CK(launch_pack_partials(P, stream)); stats.total_launches++;
    }
  };
  run_pass(0);
  CK(cudaMemcpyAsync(h_small.p, d_owner_cursor.p, (size_t)world * 8, cudaMemcpyDeviceToHost, stream));
  CK(cudaStreamSynchronize(stream));
  uint64_t n_total = 0, b_total = 0;
  for (int o = 0; o < world; o++) {
    uint64_t c = h_small.as<uint64_t>()[o];
    h_owner_counts[(size_t)o] = (int64_t)(c >> 32); h_owner_bytes[(size_t)o] = (int64_t)(c & 0xFFFFFFFFull);
    P.owner_base[o] = (n_total << 32) | b_total;
    n_total += c >> 32; b_total += c & 0xFFFFFFFFull;
    if (n_total >= (1ull << 31) || b_total >= (1ull << 31)) fail(DNZ_ERR_UNSUPPORTED, "more than 2^31 packets or key bytes in one exchange step");
  }
  if (n_total == 0) return;
  d_part_entries.reserve((size_t)n_total * sizeof(PartialEntry)); d_part_keys.reserve((size_t)b_total + 64);
  P.entries = d_part_entries.as<PartialEntry>(); P.key_bytes = d_part_keys.as<uint8_t>();
  run_pass(1);
  CK(cudaStreamSynchronize(stream));
  out->n_entries = (int64_t)n_total; out->entries = d_part_entries.as<uint8_t>();
  out->key_bytes_len = (int64_t)b_total; out->key_bytes = d_part_keys.as<uint8_t>();
  stats.exchanged_out += (int64_t)n_total;
}

void dnz_window::import_partials(const uint8_t* entries, const int64_t* src_counts, const uint8_t* key_bytes,
                                 const int64_t* src_key_bytes, int64_t pane_lo, int64_t pane_hi) {
  MergeParams M; memset(&M, 0, sizeof M);
  int64_t n = 0, kb = 0;
  for (int r = 0; r < world; r++) {
    if (src_counts[r] < 0 || src_key_bytes[r] < 0) fail(DNZ_ERR_INVALID, "negative split size");
    M.src_key_base[r] = kb; n += src_counts[r]; kb += src_key_bytes[r]; M.src_entry_end[r] = n;
  }
  if (n == 0) return;
  if (!entries || (kb && !key_bytes)) fail(DNZ_ERR_INVALID, "null packet buffers");
  if (pane_hi < pane_lo || pane_hi - pane_lo >= (1 << 16)) fail(DNZ_ERR_INVALID, "bad pane range");
  // every received key may be new here: size the dictionary and the long-key arena first so that the merge cannot fail
  fetch_ctl();
  while ((uint64_t)n_groups_host + (uint64_t)n > gcap) dict_grow();
  {
    if (arena_used_host + (uint64_t)kb + 64 > arena_cap) arena_grow(arena_used_host + (uint64_t)kb + 64);
  }
  const int64_t np = pane_hi - pane_lo + 1;
  for (int64_t p = pane_lo; p <= pane_hi; p++) ensure_side_arrays(get_pane(p, true));
  const size_t pb = (size_t)np * sizeof(void*);
  h_xptrs.reserve(7 * pb); d_xptrs.reserve(7 * pb);
  void** hp = h_xptrs.as<void*>();
  for (int64_t p = pane_lo; p <= pane_hi; p++) {
    const size_t k = (size_t)(p - pane_lo);
    Pane* m = get_pane(p, false);
    hp[0 * np + k] = m->st.p; hp[1 * np + k] = nullptr; hp[2 * np + k] = m->nullrows.p; hp[3 * np + k] = nullptr;
    hp[4 * np + k] = m->fz.p; hp[5 * np + k] = nullptr; hp[6 * np + k] = reinterpret_cast<void*>((uintptr_t)(m->tag & 0xFFFFFFFFull));
  }
  CK(cudaMemcpyAsync(d_xptrs.p, hp, 7 * pb, cudaMemcpyHostToDevice, stream));
  CK(cudaMemsetAsync(ctl(CTL_MERGE_ERR), 0, 4, stream));
  char* dp = d_xptrs.as<char>();
  M.panes.pane0 = pane_lo; M.panes.n_panes = (int32_t)np; M.panes.pane_ms = pane_ms;
  M.panes.main = (GroupState* const*)(dp + 0 * pb); M.panes.late = (GroupState* const*)(dp + 1 * pb);
  M.panes.nullrows_main = (unsigned long long* const*)(dp + 2 * pb); M.panes.nullrows_late = (unsigned long long* const*)(dp + 3 * pb);
  M.panes.fz_main = (unsigned long long* const*)(dp + 4 * pb); M.panes.fz_late = (unsigned long long* const*)(dp + 5 * pb);
  M.panes.tag_main = (const unsigned long long*)(dp + 6 * pb);
  M.entries = reinterpret_cast<const PartialEntry*>(entries); M.n_entries = n; M.key_bytes = key_bytes; M.world = world;
  M.dict = dict_view(); M.error = reinterpret_cast<uint32_t*>(ctl(CTL_MERGE_ERR));
  CK(launch_merge_partials(M, stream)); stats.total_launches++;
  fetch_ctl();
  uint32_t err = *reinterpret_cast<const uint32_t*>(h_small.as<char>() + CTL_MERGE_ERR);
  if (err) fail(DNZ_ERR_NOMEM, "pane merge failed (flags %u): table sizing error", err);
  stats.exchanged_in += n;
}

// =================================================================================================
// C ABI
// =================================================================================================
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

extern "C" {

int32_t dnz_window_create(const dnz_window_config* cfg, const struct ArrowSchema* input_schema, dnz_window** out) {
  if (!out) { g_last_error = "null out"; return DNZ_ERR_INVALID; }
  *out = nullptr;
  dnz_window* w = nullptr;
  try {
    w = new dnz_window();
    w->init(cfg, input_schema);
    *out = w;
    return DNZ_OK;
  } catch (const DnzError& e) {
    g_last_error = e.msg; delete w; return e.code;
  } catch (const std::exception& e) {
    g_last_error = e.what(); delete w; return DNZ_ERR_NOMEM;
  }
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
  else w->emit_normal(watermark_ms, false, nullptr);
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

struct dnz_synth {
  int dev; void* ts; void* val; void* off; void* bytes; int64_t alg_bytes;
};

int32_t dnz_synth_generate(int32_t device, int64_t row0, int64_t n_rows, int64_t batch_rows, uint64_t seed, int64_t groups,
                           int64_t rows_per_ms, int64_t t0_ms, int32_t uuid_keys, int64_t key_mul, int64_t key_add, dnz_synth** arena,
                           dnz_device_batch* out, int64_t n_batches) {
  if (!arena || !out || n_rows <= 0 || batch_rows <= 0 || groups <= 0 || rows_per_ms <= 0) { g_last_error = "bad synth arguments"; return DNZ_ERR_INVALID; }
  int64_t nb = (n_rows + batch_rows - 1) / batch_rows;
  if (n_batches < nb) { g_last_error = "batch array too small"; return DNZ_ERR_INVALID; }
  if (cudaSetDevice(device) != cudaSuccess) { g_last_error = "no such CUDA device"; return DNZ_ERR_CUDA; }
  int maxlen = 36;
  if (key_mul < 1) key_mul = 1;
  if (!uuid_keys) { maxlen = 8; for (int64_t v = (groups - 1) * key_mul + key_add; v >= 10; v /= 10) maxlen++; }
  int64_t off_stride = (batch_rows + 1 + 3) & ~(int64_t)3;
  int64_t bytes_stride = (batch_rows * maxlen + 15 + 16) & ~(int64_t)15;
  dnz_synth* a = new dnz_synth{device, nullptr, nullptr, nullptr, nullptr, 0};
  auto bail = [&](const char* m) { g_last_error = m; dnz_synth_free(a); return DNZ_ERR_CUDA; };
  if (cudaMalloc(&a->ts, (size_t)n_rows * 8 + 64) != cudaSuccess) return bail("cudaMalloc(ts) failed");
  if (cudaMalloc(&a->val, (size_t)n_rows * 8 + 64) != cudaSuccess) return bail("cudaMalloc(val) failed");
  if (cudaMalloc(&a->off, (size_t)nb * off_stride * 4 + 64) != cudaSuccess) return bail("cudaMalloc(off) failed");
  if (cudaMalloc(&a->bytes, (size_t)nb * bytes_stride + 64) != cudaSuccess) return bail("cudaMalloc(bytes) failed");
  if (launch_synth(row0, n_rows, batch_rows, seed, groups, rows_per_ms, t0_ms, uuid_keys, key_mul, key_add, (int64_t*)a->ts, (double*)a->val,
                   (int32_t*)a->off, (uint8_t*)a->bytes, bytes_stride, nullptr) != cudaSuccess) return bail("synth launch failed");
  if (cudaDeviceSynchronize() != cudaSuccess) return bail("synth kernel failed");
  // algorithmic bytes: 20 B/row + key bytes (last offset of every batch)
  std::vector<int32_t> last((size_t)nb);
  for (int64_t b = 0; b < nb; b++) {
    int64_t n = std::min(batch_rows, n_rows - b * batch_rows);
    if (cudaMemcpy(&last[(size_t)b], (int32_t*)a->off + b * off_stride + n, 4, cudaMemcpyDeviceToHost) != cudaSuccess) return bail("memcpy failed");
  }
  a->alg_bytes = 20 * n_rows;
  for (int64_t b = 0; b < nb; b++) {
    int64_t n = std::min(batch_rows, n_rows - b * batch_rows);
    a->alg_bytes += last[(size_t)b];
    dnz_device_batch& d = out[b];
    memset(&d, 0, sizeof d);
    d.n_rows = n; d.ts = (int64_t*)a->ts + b * batch_rows; d.val = (double*)a->val + b * batch_rows;
    d.key_off = (int32_t*)a->off + b * off_stride; d.key_bytes = (uint8_t*)a->bytes + b * bytes_stride;
  }
  *arena = a;
  return DNZ_OK;
}
int64_t dnz_synth_bytes(const dnz_synth* a) { return a ? a->alg_bytes : 0; }
void dnz_synth_free(dnz_synth* a) {
  if (!a) return;
  cudaSetDevice(a->dev);
  cudaFree(a->ts); cudaFree(a->val); cudaFree(a->off); cudaFree(a->bytes);
  delete a;
}

}  // extern "C"

// =================================================================================================
// dnz_group: the library-owned communicator of the fused pane exchange (SURVEY.md §8b "dnz_group_create"; §8e).
// One rank per GPU.  Multi-process groups (one process per GPU, the production shape) map every rank's receive region into every
// peer with CUDA IPC, order the streams of different ranks with INTERPROCESS CUDA EVENTS (no kernel ever spins) and exchange the
// per-step host scalars (local watermark, first pane) through a POSIX shared-memory block; the rendezvous needs two all-gathers
// of a few hundred bytes at creation, which the host application supplies as a callback (the role the ncclUniqueId broadcast
// plays for NCCL).  Local groups put all ranks into one process (tests; several GPUs driven by one process): same kernels,
// same protocol, plain events.
// =================================================================================================
#include <fcntl.h>
#include <sys/mman.h>
#include <unistd.h>

#include <atomic>

namespace {
struct HostCtl {          // shared by all ranks (POSIX shm or heap); four slots by step & 3: a rank is never more than two steps ahead
  std::atomic<int64_t> arrived[4][MAX_WORLD];     // phase 1: the local watermark of the step is published
  std::atomic<int64_t> packed[4][MAX_WORLD];      // phase 2: the "my packets are written" event of the step is recorded
  std::atomic<int64_t> finished[4][MAX_WORLD];    // phase 3: the step is issued completely ("merged" event recorded)
  std::atomic<int64_t> lwm[4][MAX_WORLD];
  std::atomic<int64_t> first_pane[4][MAX_WORLD];
  std::atomic<int32_t> failed;
};
struct GroupShared { HostCtl ctl; };
}  // namespace

struct dnz_group {
  int rank = 0, world = 1, dev = 0;
  uint64_t ring_entries = 0, ring_key_bytes = 0;
  size_t region_bytes = 0;
  void* region = nullptr;                       // this rank's receive region (cudaMalloc: IPC-exportable)
  std::vector<void*> peer_base;                 // mapped peers (nullptr for self)
  bool ipc = false;
  HostCtl* hctl = nullptr; size_t shm_bytes = 0; std::string shm_name; bool shm_owner = false;
  std::shared_ptr<GroupShared> local_shared;
  // ev_packed[r][p] / ev_merged[r][p]: rank r's events of step parity p (own rank: created here; peers: opened / shared)
  cudaEvent_t ev_packed[MAX_WORLD][2] = {}, ev_merged[MAX_WORLD][2] = {};
  XchgView view{};
  unsigned long long step = 0;
  DevBuf d_owner_cursor, d_owner_base, d_totals;   // totals: [0] packets sent, [1] packets merged
  PinnedBuf h_totals; cudaEvent_t totals_ev = nullptr; bool totals_issued = false;
  int phase = 0;                                 // 0 idle, 1 begun, 2 packed
  // DNZ_TRACE: device timestamps of the step phases (pack start, packed, peers' packets seen, merged, emitted)
  static constexpr int TSTEPS = 48; cudaEvent_t tev[TSTEPS][5] = {}; int tcount = 0;
  void tmark(int k, cudaStream_t st) { if (!g_trace || tcount >= TSTEPS) return; if (!tev[tcount][k]) cudaEventCreate(&tev[tcount][k]); cudaEventRecord(tev[tcount][k], st); if (k == 4) tcount++; }
  struct Range { int64_t gwm = INT64_MIN, first = INT64_MAX, hi = INT64_MIN; bool any = false; };
  Range sent[2];                                 // what pack of step s sent (by step parity): merged by finish of step s+1
  bool staged[2] = {false, false};
  unsigned long long attach_step = 0;            // the step count when the current STREAM began (first step of a fresh operator): what was published before belongs to another stream

  static XchgRegion carve(void* base, uint64_t ring_entries) {
    XchgRegion r;
    char* p = static_cast<char*>(base);
    r.ctl = reinterpret_cast<XchgCtl*>(p);
    r.entries = reinterpret_cast<PartialEntry*>(p + 4096);
    r.keys = reinterpret_cast<uint8_t*>(p + 4096 + 2 * ring_entries * sizeof(PartialEntry));
    return r;
  }
  ~dnz_group() {
    cudaSetDevice(dev);
    cudaDeviceSynchronize();
    if (g_trace) for (int i = 0; i < tcount; i++) {
      float a = 0, b = 0, c = 0, d = 0, gap = 0;
      cudaEventElapsedTime(&a, tev[i][0], tev[i][1]); cudaEventElapsedTime(&b, tev[i][1], tev[i][2]); cudaEventElapsedTime(&c, tev[i][2], tev[i][3]); cudaEventElapsedTime(&d, tev[i][3], tev[i][4]);
      if (i) cudaEventElapsedTime(&gap, tev[i - 1][4], tev[i][0]);
      fprintf(stderr, "[dnz] rank %d xstep %d device: since_prev=%.3f pack=%.3f wait_peers=%.3f merge=%.3f emit=%.3f ms\n", rank, i, gap, a, b, c, d);
    }
    if (totals_ev) cudaEventDestroy(totals_ev);
    for (int p = 0; p < 2; p++) { if (ev_packed[rank][p]) cudaEventDestroy(ev_packed[rank][p]); if (ev_merged[rank][p]) cudaEventDestroy(ev_merged[rank][p]); }
    if (ipc) {
      for (int r = 0; r < world; r++) if (r != rank) for (int p = 0; p < 2; p++) { if (ev_packed[r][p]) cudaEventDestroy(ev_packed[r][p]); if (ev_merged[r][p]) cudaEventDestroy(ev_merged[r][p]); }
      for (size_t r = 0; r < peer_base.size(); r++) if (peer_base[r]) cudaIpcCloseMemHandle(peer_base[r]);
    }
    if (region) cudaFree(region);
    if (hctl && !local_shared) { munmap(hctl, shm_bytes); if (shm_owner) shm_unlink(shm_name.c_str()); }
  }
};

namespace {

void group_alloc_region(dnz_group* g, unsigned event_flags) {
  if (g->ring_entries < 1024) g->ring_entries = 1024;
  if (g->ring_key_bytes < 65536) g->ring_key_bytes = 65536;
  g->ring_key_bytes = round_up(g->ring_key_bytes, 256);
  if (g->ring_entries >= (1ull << 31) || g->ring_key_bytes >= (1ull << 31)) fail(DNZ_ERR_INVALID, "exchange ring larger than 2^31 packets / key bytes per step");
  g->region_bytes = 4096 + 2 * g->ring_entries * sizeof(PartialEntry) + 2 * g->ring_key_bytes;
  CK(cudaSetDevice(g->dev));
  CK(cudaMalloc(&g->region, g->region_bytes));
  CK(cudaMemset(g->region, 0, 4096));
  g->d_owner_cursor.alloc(MAX_WORLD * 8); g->d_owner_base.alloc(MAX_WORLD * 8); g->d_totals.alloc(64);
  CK(cudaMemset(g->d_totals.p, 0, 64));
  g->h_totals.reserve(64); memset(g->h_totals.p, 0, 64);
  CK(cudaEventCreateWithFlags(&g->totals_ev, cudaEventDisableTiming));
  for (int p = 0; p < 2; p++) {
    CK(cudaEventCreateWithFlags(&g->ev_packed[g->rank][p], cudaEventDisableTiming | event_flags));
    CK(cudaEventCreateWithFlags(&g->ev_merged[g->rank][p], cudaEventDisableTiming | event_flags));
  }
  CK(cudaDeviceSynchronize());
}

void group_finish_view(dnz_group* g) {
  XchgView& v = g->view;
  memset(&v, 0, sizeof v);
  v.rank = g->rank; v.world = g->world; v.ring_entries = g->ring_entries; v.ring_key_bytes = g->ring_key_bytes;
  v.self = dnz_group::carve(g->region, g->ring_entries);
  for (int r = 0; r < g->world; r++) v.peer[r] = dnz_group::carve(r == g->rank ? g->region : g->peer_base[(size_t)r], g->ring_entries);
}

// host barrier on one of the per-step counters.  A process that drives all ranks itself must call the phases in order for
// ALL ranks (begin x world, pack x world, finish x world): waiting would never end there, so it is an error instead.
void group_wait(dnz_group* g, std::atomic<int64_t> (*ctr)[MAX_WORLD], unsigned long long step, const char* what) {
  const int s = (int)(step & 3);
  const auto t0 = std::chrono::steady_clock::now();
  for (int r = 0; r < g->world; r++) {
    int spins = 0;
    while (ctr[s][r].load(std::memory_order_acquire) != (int64_t)step) {
      if (g->local_shared) fail(DNZ_ERR_INVALID, "exchange group: rank %d has not reached '%s' of step %llu (a process driving several ranks calls each phase for all ranks before the next phase)", r, what, step);
      if (g->hctl->failed.load(std::memory_order_relaxed)) fail(DNZ_ERR_INVALID, "exchange group: another rank failed or left");
      if (++spins > 2000) {
        usleep(50);
        if (std::chrono::steady_clock::now() - t0 > std::chrono::seconds(300)) fail(DNZ_ERR_INVALID, "exchange group: rank %d did not reach '%s' of step %llu within 300 s", r, what, step);
      }
    }
  }
}

}  // namespace

// The step protocol is PIPELINED over three steps so that no phase waits for something a peer does "now" (a rank whose host
// thread is descheduled for a millisecond would otherwise idle every GPU of the group -- each has about one aggregate launch
// queued):
//     step s   begin   publish this rank's local watermark                                        -> lwm(s)
//     step s+1 pack    global watermark = min over ranks of lwm(s); the panes it closes are packed and written into the owners'
//                      rings (half (s+1) & 1)
//     step s+2 finish  the owners merge what step s+1 wrote, and emit the windows closed under that watermark
// The only host wait is "every rank has ISSUED step s-1" (finished[s-1]), checked in pack of step s: it orders the interprocess
// event waits (an event wait captures the record that exists when it is issued) and was normally satisfied a whole step ago.
// Every rank computes the same watermark / pane range sequence, so `exported_pane_upto` agrees everywhere without being exchanged.

// ---- phase 1: seal what is filling, publish the local watermark of the step
void dnz_window::group_begin(dnz_group* g) {
  if (world != g->world || rank != g->rank) fail(DNZ_ERR_INVALID, "operator is not attached to this group");
  if (g->phase != 0) fail(DNZ_ERR_INVALID, "dnz_group_step_begin: the previous step of this rank is not finished");
  // Nothing is waited for.  A filling superbatch is sealed (its scan is enqueued, the superbatch sealed before it is launched: its
  // scan results are on the host), but the NEWEST sealed superbatch is not forced -- its scan sits behind the previous aggregate
  // on the device, waiting for it here would idle the GPU every step.  The local watermark is that of the LAUNCHED batches;
  // dnz_window_process before the step includes everything pushed.
  // Errors of earlier steps (ring / table overflow) surface when their launches are verified.
  if (!group_started) {
    // The first step of a fresh operator begins a new stream in the group (collective: every rank's operator is fresh in the same
    // step; operators may have been attached long before).  Watermarks published and pane ranges sent before this step belong to
    // the previous stream: the pipeline restarts empty.
    group_started = true;
    g->attach_step = g->step; g->sent[0] = g->sent[1] = dnz_group::Range{};
  }
  if (!cur().batches.empty()) seal_current();
  while (!launched_order.empty() && cudaEventQuery(slot[launched_order.front()].done) == cudaSuccess) verify(slot[launched_order.front()]);
  cudaGetLastError();
  if (g->totals_issued && cudaEventQuery(g->totals_ev) == cudaSuccess) {
    stats.exchanged_out = (int64_t)g->h_totals.as<unsigned long long>()[0]; stats.exchanged_in = (int64_t)g->h_totals.as<unsigned long long>()[1];
  }
  cudaGetLastError();
  const unsigned long long step = g->step + 1;
  HostCtl* h = g->hctl; const int q = (int)(step & 3);
  h->lwm[q][g->rank].store(has_lwm ? lwm : INT64_MIN, std::memory_order_relaxed);
  h->first_pane[q][g->rank].store(panes.empty() ? INT64_MAX : panes.begin()->first, std::memory_order_relaxed);
  h->arrived[q][g->rank].store((int64_t)step, std::memory_order_release);
  g->phase = 1;
  g_tr.mark("x_begin");
}

// ---- phase 2: the panes closed under the watermark published one step ago go straight into the owners' rings
void dnz_window::group_pack(dnz_group* g) {
  if (g->phase != 1) fail(DNZ_ERR_INVALID, "dnz_group_step_pack without dnz_group_step_begin");
  const unsigned long long step = g->step + 1;
  const int par = (int)(step & 1);
  int64_t gwm = INT64_MIN, gfirst = INT64_MAX;
  if (step >= 2) {
    group_wait(g, g->hctl->finished, step - 1, "finish");
    g_tr.mark("x_wait_prev_step");
    const int q = (int)((step - 1) & 3);
    if (step - 1 > g->attach_step) gwm = INT64_MAX;          // (the watermarks of step-1 were published by THIS stream's operators)
    if (step - 1 > g->attach_step) for (int r = 0; r < world; r++) { gwm = std::min(gwm, g->hctl->lwm[q][r].load(std::memory_order_relaxed)); gfirst = std::min(gfirst, g->hctl->first_pane[q][r].load(std::memory_order_relaxed)); }
  }
  if (exported_pane_upto != INT64_MIN) gfirst = exported_pane_upto + 1;
  const int64_t hi = gwm == INT64_MIN ? INT64_MIN : floor_div(gwm, pane_ms) - 1;          // panes with end <= global watermark
  const bool any = gwm != INT64_MIN && gfirst != INT64_MAX && hi >= gfirst;
  g->sent[par].gwm = gwm; g->sent[par].first = gfirst; g->sent[par].hi = hi; g->sent[par].any = any;
  XchgView X = g->view; X.step = step;
  std::vector<Pane*> send;
  if (any) {
    if (hi - gfirst + 1 > (1 << 16)) fail(DNZ_ERR_UNSUPPORTED, "one exchange step spans %lld panes", (long long)(hi - gfirst + 1));
    for (auto& kv : panes) if (kv.first >= gfirst && kv.first <= hi) send.push_back(kv.second.get());
    exported_pane_upto = hi;                                                                // the same on every rank
  }
  // the owners must have merged what step-2 wrote into the same half of their rings (recorded in their finish of step-1)
  if (step > 2) for (int r = 0; r < world; r++) if (r != rank) CK(cudaStreamWaitEvent(stream, g->ev_merged[r][par], 0));
  g->tmark(0, stream);
  CK(cudaMemsetAsync(g->d_owner_cursor.p, 0, MAX_WORLD * 8, stream));
  PackParams P; memset(&P, 0, sizeof P);
  P.n_groups = gcap; P.rank = rank; P.world = world; P.dict = dict_view();      // grid bound; the kernels clamp to the device counter
  P.owner_cursor = g->d_owner_cursor.as<unsigned long long>();
  auto for_pane_chunks = [&](auto&& launch) {                 // up to PACK_PANES panes per launch (one thread per group id walks them)
    for (size_t i0 = 0; i0 < send.size(); i0 += PACK_PANES) {
      P.n_multi = (int32_t)std::min<size_t>(PACK_PANES, send.size() - i0);
      for (int j = 0; j < P.n_multi; j++) {
        Pane* p = send[i0 + j];
        P.mst[j] = p->st.as<GroupState>(); P.mnull[j] = p->nullrows.as<unsigned long long>(); P.mfz[j] = p->fz.as<unsigned long long>(); P.mpane[j] = p->id;
      }
      launch(); stats.total_launches++;
    }
  };
  P.pass = 0;
  for_pane_chunks([&]() { CK(launch_pack_partials(P, stream)); });
  CK(launch_xchg_reserve(X, g->d_owner_cursor.as<unsigned long long>(), g->d_owner_base.as<unsigned long long>(), g->d_totals.as<unsigned long long>(), reinterpret_cast<uint32_t*>(ctl(CTL_MERGE_ERR)), stream));
  stats.total_launches++;
  for_pane_chunks([&]() { CK(launch_pack_write_peer(P, X, g->d_owner_base.as<unsigned long long>(), stream)); });
  CK(cudaEventRecord(g->ev_packed[rank][par], stream));                    // "all my packets of this step are in the owners' rings"
  g->tmark(1, stream);
  g->hctl->packed[(int)(step & 3)][g->rank].store((int64_t)step, std::memory_order_release);
  g->phase = 2;
  g_tr.mark("x_pack");
}

// ---- phase 3: merge what the peers wrote ONE STEP AGO, emit the windows of this rank's keys closed under that step's watermark
void dnz_window::group_finish(dnz_group* g, int64_t* gwm_out) {
  if (g->phase != 2) fail(DNZ_ERR_INVALID, "dnz_group_step_finish without dnz_group_step_pack");
  const unsigned long long step = ++g->step;
  g->phase = 0;
  if (gwm_out) *gwm_out = INT64_MIN;
  if (step >= 2) {
    const unsigned long long mstep = step - 1;                            // the step whose packets are merged now
    const int mp = (int)(mstep & 1);
    const dnz_group::Range R = g->sent[mp];
    if (gwm_out) *gwm_out = R.gwm;
    XchgView X = g->view; X.step = mstep;
    // every peer issued pack(mstep) before its finish(mstep), which pack of this step waited for: the records exist
    for (int r = 0; r < world; r++) if (r != rank) CK(cudaStreamWaitEvent(stream, g->ev_packed[r][mp], 0));
    g->tmark(2, stream);
    if (R.any) {
      const int64_t gfirst = R.first, hi = R.hi;
      const int64_t np = hi - gfirst + 1;
      for (int64_t p = gfirst; p <= hi; p++) ensure_side_arrays(get_pane(p, true));
      const size_t pb = (size_t)np * sizeof(void*);
      // The pane table is staged in page-locked memory and copied by the stream when it gets there: the staging half may only be
      // rewritten once the copy issued two steps ago (same half) has executed -- its merge has been recorded in ev_merged[rank][mp].
      const size_t half_bytes = (size_t)7 * (1 << 16) * sizeof(void*);
      if (g->staged[mp]) CK(cudaEventSynchronize(g->ev_merged[rank][mp]));
      g->staged[mp] = true;
      g_tr.mark("x_sync_merged");
      void** hp = reinterpret_cast<void**>(h_xptrs.as<char>() + (size_t)mp * half_bytes);
      char* dxp = d_xptrs.as<char>() + (size_t)mp * half_bytes;
      for (int64_t p = gfirst; p <= hi; p++) {
        const size_t k = (size_t)(p - gfirst);
        Pane* m = get_pane(p, false);
        hp[0 * np + k] = m->st.p; hp[1 * np + k] = nullptr; hp[2 * np + k] = m->nullrows.p; hp[3 * np + k] = nullptr;
        hp[4 * np + k] = m->fz.p; hp[5 * np + k] = nullptr; hp[6 * np + k] = reinterpret_cast<void*>((uintptr_t)(m->tag & 0xFFFFFFFFull));
      }
      CK(cudaMemcpyAsync(dxp, hp, 7 * pb, cudaMemcpyHostToDevice, stream));
      MergeParams M; memset(&M, 0, sizeof M);
      char* dp = dxp;
      M.panes.pane0 = gfirst; M.panes.n_panes = (int32_t)np; M.panes.pane_ms = pane_ms;
      M.panes.main = (GroupState* const*)(dp + 0 * pb); M.panes.late = (GroupState* const*)(dp + 1 * pb);
      M.panes.nullrows_main = (unsigned long long* const*)(dp + 2 * pb); M.panes.nullrows_late = (unsigned long long* const*)(dp + 3 * pb);
      M.panes.fz_main = (unsigned long long* const*)(dp + 4 * pb); M.panes.fz_late = (unsigned long long* const*)(dp + 5 * pb);
      M.panes.tag_main = (const unsigned long long*)(dp + 6 * pb);
      M.world = world; M.dict = dict_view(); M.error = reinterpret_cast<uint32_t*>(ctl(CTL_MERGE_ERR));
      CK(launch_merge_ring(M, X, g->d_totals.as<unsigned long long>() + 1, sm_count, stream)); stats.total_launches++;
    }
    CK(cudaMemsetAsync(&g->view.self.ctl->cursor[mp], 0, 8, stream));       // the ring half is free again ...
    CK(cudaEventRecord(g->ev_merged[rank][mp], stream));                    // ... once this has happened
    CK(cudaMemcpyAsync(g->h_totals.p, g->d_totals.p, 16, cudaMemcpyDeviceToHost, stream));   // packet counters for dnz_stats (read when complete)
    CK(cudaEventRecord(g->totals_ev, stream)); g->totals_issued = true;
    g->tmark(3, stream);
    // ---- every rank emits the windows of ITS keys that closed under that watermark
    if (R.gwm != INT64_MIN) {
      if (res_consumed) reset_results();
      rotate_result_sets();
      emit_normal(R.gwm, false, nullptr);
    }
    g->tmark(4, stream);
  }
  g->hctl->finished[(int)(step & 3)][g->rank].store((int64_t)step, std::memory_order_release);
  g_tr.mark("x_finish");
  g_tr.flush("xstep");
}

namespace {
struct GroupHello { cudaIpcMemHandle_t mem; cudaIpcEventHandle_t packed[2], merged[2]; char shm[64]; int64_t ring_entries, ring_key_bytes; int32_t dev, pad; };
}

extern "C" {

int32_t dnz_group_create(const dnz_group_config* cfg, dnz_allgather_fn allgather, void* ctx, dnz_group** out) {
  if (!out) { g_last_error = "null out"; return DNZ_ERR_INVALID; }
  *out = nullptr;
  dnz_group* g = nullptr;
  try {
    if (!cfg || !allgather) fail(DNZ_ERR_INVALID, "null config or all-gather callback");
    if (cfg->abi_version != DNZ_ABI_VERSION) fail(DNZ_ERR_INVALID, "abi_version %u != %u", cfg->abi_version, DNZ_ABI_VERSION);
    if (cfg->world < 1 || cfg->world > MAX_WORLD || cfg->rank < 0 || cfg->rank >= cfg->world) fail(DNZ_ERR_INVALID, "bad rank/world (world <= %d)", MAX_WORLD);
    g = new dnz_group();
    g->rank = cfg->rank; g->world = cfg->world; g->dev = cfg->device; g->ipc = true;
    g->ring_entries = (uint64_t)std::max<int64_t>(cfg->ring_entries, 0); g->ring_key_bytes = (uint64_t)std::max<int64_t>(cfg->ring_key_bytes, 0);
    if (!g->ring_entries) g->ring_entries = 8ull << 20;
    if (!g->ring_key_bytes) g->ring_key_bytes = 256ull << 20;
    group_alloc_region(g, cudaEventInterprocess);
    GroupHello mine; memset(&mine, 0, sizeof mine);
    CK(cudaIpcGetMemHandle(&mine.mem, g->region));
    for (int p = 0; p < 2; p++) { CK(cudaIpcGetEventHandle(&mine.packed[p], g->ev_packed[g->rank][p])); CK(cudaIpcGetEventHandle(&mine.merged[p], g->ev_merged[g->rank][p])); }
    mine.ring_entries = (int64_t)g->ring_entries; mine.ring_key_bytes = (int64_t)g->ring_key_bytes; mine.dev = g->dev;
    g->shm_bytes = round_up(sizeof(HostCtl), 4096);
    if (g->rank == 0) {       // the block of per-step scalars shared by all ranks
      snprintf(mine.shm, sizeof mine.shm, "/dnz_group_%d_%lld", (int)getpid(), (long long)std::chrono::steady_clock::now().time_since_epoch().count());
      int fd = shm_open(mine.shm, O_CREAT | O_EXCL | O_RDWR, 0600);
      if (fd < 0 || ftruncate(fd, (off_t)g->shm_bytes) != 0) fail(DNZ_ERR_NOMEM, "shm_open(%s) failed", mine.shm);
      void* p = mmap(nullptr, g->shm_bytes, PROT_READ | PROT_WRITE, MAP_SHARED, fd, 0); close(fd);
      if (p == MAP_FAILED) fail(DNZ_ERR_NOMEM, "mmap of the group control block failed");
      g->hctl = static_cast<HostCtl*>(p); g->shm_name = mine.shm; g->shm_owner = true;
    }
    std::vector<GroupHello> all((size_t)g->world);
    if (allgather(ctx, &mine, all.data(), (int64_t)sizeof(GroupHello)) != 0) fail(DNZ_ERR_INVALID, "the rendezvous all-gather failed");
    if (g->rank != 0) {
      int fd = shm_open(all[0].shm, O_RDWR, 0600);
      if (fd < 0) fail(DNZ_ERR_INVALID, "cannot open the group control block %s (ranks must share one node)", all[0].shm);
      void* p = mmap(nullptr, g->shm_bytes, PROT_READ | PROT_WRITE, MAP_SHARED, fd, 0); close(fd);
      if (p == MAP_FAILED) fail(DNZ_ERR_NOMEM, "mmap of the group control block failed");
      g->hctl = static_cast<HostCtl*>(p); g->shm_name = all[0].shm;
    }
    g->peer_base.assign((size_t)g->world, nullptr);
    for (int r = 0; r < g->world; r++) {
      const GroupHello& o = all[(size_t)r];
      if (o.ring_entries != mine.ring_entries || o.ring_key_bytes != mine.ring_key_bytes) fail(DNZ_ERR_INVALID, "ranks disagree on the ring size");
      if (r == g->rank) continue;
      int can = 0; CK(cudaDeviceCanAccessPeer(&can, g->dev, o.dev));
      if (!can && o.dev != g->dev) fail(DNZ_ERR_UNSUPPORTED, "GPU %d cannot access GPU %d directly (the fused exchange needs NVLink / P2P)", g->dev, o.dev);
      CK(cudaIpcOpenMemHandle(&g->peer_base[(size_t)r], o.mem, cudaIpcMemLazyEnablePeerAccess));
      for (int p = 0; p < 2; p++) { CK(cudaIpcOpenEventHandle(&g->ev_packed[r][p], o.packed[p])); CK(cudaIpcOpenEventHandle(&g->ev_merged[r][p], o.merged[p])); }
    }
    group_finish_view(g);
    GroupHello again = mine; std::vector<GroupHello> all2((size_t)g->world);          // barrier: everybody has mapped everything
    if (allgather(ctx, &again, all2.data(), (int64_t)sizeof(GroupHello)) != 0) fail(DNZ_ERR_INVALID, "the rendezvous all-gather failed");
    if (g->shm_owner) { shm_unlink(g->shm_name.c_str()); g->shm_owner = false; }      // the mappings stay; the name is gone
    *out = g;
    return DNZ_OK;
  } catch (const DnzError& e) {
    g_last_error = e.msg; delete g; return e.code;
  } catch (const std::exception& e) {
    g_last_error = e.what(); delete g; return DNZ_ERR_NOMEM;
  }
}

int32_t dnz_group_create_local(int32_t world, const int32_t* devices, int64_t ring_entries, int64_t ring_key_bytes, dnz_group** out) {
  if (!out || !devices) { g_last_error = "null argument"; return DNZ_ERR_INVALID; }
  std::vector<dnz_group*> gs;
  try {
    if (world < 1 || world > MAX_WORLD) fail(DNZ_ERR_INVALID, "bad world (<= %d)", MAX_WORLD);
    auto shared = std::make_shared<GroupShared>();
    memset(static_cast<void*>(&shared->ctl), 0, sizeof(HostCtl));
    for (int r = 0; r < world; r++) {
      dnz_group* g = new dnz_group(); gs.push_back(g);
      g->rank = r; g->world = world; g->dev = devices[r];
      g->ring_entries = ring_entries > 0 ? (uint64_t)ring_entries : (1ull << 20); g->ring_key_bytes = ring_key_bytes > 0 ? (uint64_t)ring_key_bytes : (32ull << 20);
      g->local_shared = shared; g->hctl = &shared->ctl;
      group_alloc_region(g, 0);
    }
    for (int r = 0; r < world; r++) {
      dnz_group* g = gs[(size_t)r];
      g->peer_base.assign((size_t)world, nullptr);
      for (int q = 0; q < world; q++) {
        if (q == r) continue;
        g->peer_base[(size_t)q] = gs[(size_t)q]->region;
        for (int p = 0; p < 2; p++) { g->ev_packed[q][p] = gs[(size_t)q]->ev_packed[q][p]; g->ev_merged[q][p] = gs[(size_t)q]->ev_merged[q][p]; }
        if (devices[q] != devices[r]) { CK(cudaSetDevice(devices[r])); cudaError_t e = cudaDeviceEnablePeerAccess(devices[q], 0); if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled) CK(e); cudaGetLastError(); }
      }
      group_finish_view(g);
    }
    for (int r = 0; r < world; r++) out[r] = gs[(size_t)r];
    return DNZ_OK;
  } catch (const DnzError& e) {
    g_last_error = e.msg; for (auto* g : gs) delete g; return e.code;
  } catch (const std::exception& e) {
    g_last_error = e.what(); for (auto* g : gs) delete g; return DNZ_ERR_NOMEM;
  }
}

void dnz_group_destroy(dnz_group* g) {
  if (!g) return;
  if (g->hctl && !g->local_shared) g->hctl->failed.store(1);
  delete g;
}

int32_t dnz_group_attach(dnz_group* g, dnz_window* w) {
  if (!g) { g_last_error = "null group"; return DNZ_ERR_INVALID; }
  const int32_t rc = dnz_window_set_exchange(w, g->rank, g->world);
  if (rc == DNZ_OK) w->fused = g->world > 1;
  return rc;
}

#define DNZ_GROUP_PHASE(call)                                                       \
  DNZ_TRY(w)                                                                        \
  if (!g) fail(DNZ_ERR_INVALID, "null group");                                      \
  struct Guard { dnz_window* w; bool prev; ~Guard() { w->in_process = prev; } } guard{w, w->in_process};   \
  w->in_process = true;                                                             \
  call;                                                                             \
  DNZ_CATCH(w)

int32_t dnz_group_step_begin(dnz_group* g, dnz_window* w) { DNZ_GROUP_PHASE(w->group_begin(g)) }
int32_t dnz_group_step_pack(dnz_group* g, dnz_window* w) { DNZ_GROUP_PHASE(w->group_pack(g)) }
int32_t dnz_group_step_finish(dnz_group* g, dnz_window* w, int64_t* global_watermark_ms) { DNZ_GROUP_PHASE(w->group_finish(g, global_watermark_ms)) }
int32_t dnz_group_step(dnz_group* g, dnz_window* w, int64_t* global_watermark_ms) {
  int32_t rc = dnz_group_step_begin(g, w);
  if (rc == DNZ_OK) rc = dnz_group_step_pack(g, w);
  return rc != DNZ_OK ? rc : dnz_group_step_finish(g, w, global_watermark_ms);
}
int32_t dnz_group_flush(dnz_group* g, dnz_window* w, int64_t* global_watermark_ms) {
  int32_t rc = dnz_window_process(w, nullptr);
  for (int i = 0; i < 3 && rc == DNZ_OK; i++) rc = dnz_group_step(g, w, global_watermark_ms);
  return rc;
}

}  // extern "C"
