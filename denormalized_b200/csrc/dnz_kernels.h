// dnz_kernels.h -- device data layout + kernel launch wrappers (internal; the public boundary is include/dnz_gpu.h)
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

namespace dnz {

// ------------------------------------------------------------------------------------------------
// Tiling of the input.  One tile = up to TILE consecutive rows of ONE RecordBatch.
constexpr int TILE = 416;             // rows per tile = consumer threads of one CTA (a multiple of 4: 16 B aligned column slices)
constexpr int STAGES = 4;             // TMA ring depth per CTA
constexpr int BCAP = 6656;            // staged key bytes per tile (16 B/row average); longer tiles take the generic path (a 16 KB budget with 3 stages was tried: cfg 2 -1.5 %, cfg 5 no gain)
constexpr int CONSUMER_WARPS = 13;   // 416 consumer threads x 1 row = TILE; + 1 producer warp = 448 threads; two CTAs per SM at 72 registers (no spills)
constexpr int AGG_THREADS = (CONSUMER_WARPS + 1) * 32;  // + 1 producer warp
constexpr int INLINE_KEY = 16;        // key bytes stored inline in a dictionary slot

enum : int32_t {
  TILE_FAST = 1,          // all four column slices can be staged with cp.async.bulk (16 B aligned, fits BCAP, no bitmaps)
  TILE_PANE_UNIFORM = 2,  // every valid timestamp of the tile falls in pane_lo
  TILE_EMPTY = 4,         // no valid timestamp
  TILE_END = 8,           // (stage header only) no more tiles for this CTA
  TILE_KEYS_GLOBAL = 16,  // with TILE_FAST: timestamps / values / offsets are staged, but the key bytes exceed the stage (long keys): read from global
};

struct BatchDesc {
  const int64_t* ts; const double* val; const int32_t* off; const uint8_t* bytes;
  const uint8_t* ts_valid; const uint8_t* val_valid; const uint8_t* key_valid;
  int32_t ts_vbit, val_vbit, key_vbit;   // bit offset of row 0 inside the bitmaps (sliced arrays)
  int32_t flags;                          // bit0: buffers are padded/aligned for bulk copies
  int64_t n_rows;
  int64_t seq;                            // arrival sequence number of the batch
  int64_t tile0;                          // first tile of the batch inside the launch set
};
enum : int32_t { BATCH_BULK_OK = 1 };

struct TileDesc {
  int32_t batch, row0, n_rows, flags;
  int64_t byte0;        // off[row0]
  int32_t byte_len;     // off[row0+n_rows] - off[row0]
  int32_t pad;
  int64_t ts_min, ts_max;
  int64_t pane_lo;      // floor(ts_min / pane_ms)
};

struct BatchMinMax { int64_t ts_min, ts_max, n_valid, key_bytes, n_fast, n_tiles; };   // per RecordBatch, filled by k_tile_scan

// ------------------------------------------------------------------------------------------------
// Key dictionary: open addressing, one 32 B sector per slot, keys <= 16 B inline.
struct __align__(32) DictSlot {
  uint64_t k0, k1;       // inline: zero padded key bytes; long keys: k0 = hash64, k1 = arena offset
  uint64_t hint;         // min/max reduction filter of this group (see below); rides along with every probe for free
  uint32_t len;          // key length in bytes
  uint32_t state;        // 0 empty, 0xFFFFFFFF locked (insert in flight), else gid + 1
};
// hint = tag:32 | hmin:16 | hmax:16.  `tag` names ONE zero-initialised pane state array (Pane::tag, never reused);
// hmin / hmax are the top 16 bits of a minkey / maxkey that some thread HAS reduced (or is about to reduce) into that
// array for this group.  A row whose key is smaller in its top 16 bits cannot change the state and skips the reduction.
// Plain racy stores keep it conservative: every value ever stored is backed by a reduction, a mismatching tag reads
// as "no hint".
constexpr uint32_t SLOT_EMPTY = 0u, SLOT_LOCKED = 0xFFFFFFFFu;

// key of a group id: inline words (or hash64 / arena offset for keys > INLINE_KEY) and length; len == 0xFFFFFFFF: the NULL key
struct GidKey { uint64_t k0, k1; uint32_t len, pad; };

struct DictView {
  DictSlot* slots; uint32_t mask;     // capacity - 1 (power of two, 4 * gcap)
  uint32_t gcap;                      // group ids must stay < gcap (capacity of the per-pane state arrays)
  uint32_t* n_groups;                 // device counter
  uint32_t* null_gid;                 // 0 = unassigned, 0xFFFFFFFF locked, else gid + 1 (group of the NULL key)
  GidKey* gid_key;                    // gid -> key (dense, written at insert: emission and the pane exchange read keys coalesced)
  uint8_t* arena; unsigned long long* arena_used; uint64_t arena_cap;   // bytes of keys longer than INLINE_KEY
  unsigned long long* key_bytes_total;                                  // sum of key lengths over all groups
};

// ------------------------------------------------------------------------------------------------
// One 256 B device control block per operator, so that a single D2H copy fetches everything the host needs after a launch.
constexpr int PIPELINE_SLOTS = 3;     // superbatches in flight on the host side (dnz_window.h, Slot)
struct DictCounters {                 // DictView's device counters
  uint32_t n_groups, null_gid;
  unsigned long long arena_used, key_bytes_total;
};
struct SlotCtl {                      // one pipeline slot's aggregate launch
  unsigned long long defer_count;     // DeferList::count
  uint32_t defer_flags;               // DeferList::flags
  uint32_t tile_counter;              // AggParams::tile_counter
  uint32_t emit_blocked;              // EmitParams::blocked (not cleared with the three above)
  uint32_t pad[3];
};
struct ResultCursor {                 // one result set: EmitOut::cursor and EmitOut::overflow
  unsigned long long cursor;
  uint32_t overflow, pad;
};
struct CtlBlock {
  DictCounters dict; uint8_t pad0[40];
  SlotCtl slot[PIPELINE_SLOTS]; uint8_t pad1[32];
  ResultCursor result[2];
  uint32_t merge_err;                 // pane-merge / exchange-ring error flags (MergeParams::error)
  uint32_t ts_err;                    // a timestamp string did not match the format (launch_ts_convert)
  uint8_t pad2[24];
};
static_assert(sizeof(SlotCtl) == 32 && sizeof(ResultCursor) == 16, "control block entries");
static_assert(sizeof(CtlBlock) == 256 && offsetof(CtlBlock, slot) == 64 && offsetof(CtlBlock, result) == 192 &&
              offsetof(CtlBlock, merge_err) == 224 && offsetof(CtlBlock, ts_err) == 228, "control block layout");

// Per (pane, group) partial aggregate: exactly one 32 B sector.
struct __align__(32) GroupState {
  double cnt;                  // non-null values, kept as f64 (exact below 2^53) so that {cnt, sum} is ONE red.add.f64 pair
  double sum;
  unsigned long long minkey;   // ORD(f64::MAX) - ord(v): 0 == f64::MAX (accumulator start), larger == smaller value
  unsigned long long maxkey;   // ord(v) - ORD(f64::MIN): 0 == f64::MIN
};

// ord(): monotone map f64 -> u64 over IEEE totalOrder.  min/max accumulators are kept as distances from the
// DataFusion starting values (f64::MAX for min, f64::MIN for max) so that a zero-filled state IS the start.
constexpr unsigned long long SIGN64 = 0x8000000000000000ull;
constexpr unsigned long long BITS_F64_MAX = 0x7FEFFFFFFFFFFFFFull;
constexpr unsigned long long ORD_F64_MAX = BITS_F64_MAX | SIGN64;        // ord(+MAX)
constexpr unsigned long long ORD_F64_MIN = ~(BITS_F64_MAX | SIGN64);     // ord(-MAX)
__host__ __device__ __forceinline__ unsigned long long ord_bits(unsigned long long b) { return (b & SIGN64) ? ~b : (b | SIGN64); }
__host__ __device__ __forceinline__ unsigned long long unord_bits(unsigned long long o) { return (o & SIGN64) ? (o & ~SIGN64) : ~o; }
// IEEE totalOrder key (arrow-ord cmp on floats == f64::total_cmp)
__host__ __device__ __forceinline__ long long total_key(unsigned long long b) {
  long long s = (long long)b; return s ^ (long long)(((unsigned long long)(s >> 63)) >> 1);
}

struct PaneTable {             // uploaded per launch
  int64_t pane0;               // pane id of entry 0
  int32_t n_panes; int32_t pad;
  int64_t pane_ms;
  GroupState* const* main;     // [n_panes] nullable: pane no longer needed by any open window
  GroupState* const* late;     // [n_panes] nullable: rows re-opening already emitted windows (exact late path)
  unsigned long long* const* nullrows_main; unsigned long long* const* nullrows_late;   // rows with NULL value, nullable
  unsigned long long* const* fz_main; unsigned long long* const* fz_late;               // first +-0.0 row (seq<<1|sign), nullable
  const unsigned long long* tag_main;   // [n_panes] instance tag of main[i] (low 32 bits, never 0), see DictSlot::hint
};

struct DeferEntry { uint32_t tile, row; };
struct DeferList { DeferEntry* entries; unsigned long long* count; uint64_t cap; uint32_t* flags; };
enum : uint32_t { DEFER_GROUPS_FULL = 1, DEFER_ARENA_FULL = 2, DEFER_NEED_FZ = 4, DEFER_LIST_OVERFLOW = 8, DEFER_NEED_NULLROWS = 16 };

struct AggParams {
  const BatchDesc* batches; const TileDesc* tiles; int64_t tile_begin, tile_end;
  DictView dict; PaneTable panes; DeferList defer;
  uint32_t flags;
  uint32_t* tile_counter;   // zeroed per launch: CTAs claim tiles in stream order (keeps the tiles in flight within ~1 % of a pane)
  // Low cardinality: with a few thousand groups every state sector is hit by thousands of reductions per launch and the L2
  // atomic unit serialises per address (18 G rows/s at 1 K groups, profiles/microbench).  The paired / hinted reductions then
  // go to a PRIVATE zero-initialised copy of the pane per CTA, priv[(cta * n_panes + pane) * priv_groups + gid], which
  // k_merge_private folds into the pane afterwards (everything is commutative).  nullptr: disabled.
  GroupState* priv; uint32_t priv_groups;
};
// experiments: reduce min/max for every row; loop on collisions; both slot halves loaded by the row's own lane; stage the
// timestamps of every tile
enum : uint32_t { AGG_NO_HINTS = 1, AGG_NO_QUEUE = 2, AGG_SCALAR_PROBE = 4, AGG_STAGE_TS = 8 };

// ------------------------------------------------------------------------------------------------
// Emission: combine the panes of one window, evaluate the predicate, compact into Arrow-shaped columns.
constexpr int MAX_WINDOW_PANES = 64;
struct EmitOut {
  int32_t* key_off; uint8_t* key_bytes; uint8_t* key_valid;
  int64_t* count; double* mn; double* mx; double* avg; double* sum; uint8_t* agg_valid;
  int64_t* wstart; int64_t* wend;
  unsigned long long* cursor;    // (rows << 32) | key bytes reserved so far
  uint64_t row_cap, byte_cap;
  uint32_t* overflow;
};
struct EmitParams {
  const GroupState* panes[MAX_WINDOW_PANES];
  const unsigned long long* nullrows[MAX_WINDOW_PANES];
  const unsigned long long* fz[MAX_WINDOW_PANES];
  int32_t n_panes; int32_t has_filter; int32_t filter_col /*0 count 1 min 2 max 3 avg 4 sum*/; int32_t filter_op;
  double filter_lit;
  int64_t wstart, wend;
  uint32_t n_groups;             // upper bound (grid size); the kernel clamps to the device counter
  int32_t key_width;             // 0: Utf8 keys; 4 / 8: integer keys, every row (the NULL key too) emits key_width bytes
  int32_t rank, world;           // multi-GPU: emit only keys with hash64 % world == rank (world <= 1: all)
  // speculative pipeline: gate[0 .. PIPELINE_SLOTS) are the control block's pipeline slots (nullptr: not gated).  While any
  // of their deferred-row counters is non-zero some rows of an earlier launch have not been applied yet: the launch does
  // nothing and raises *blocked so that the host issues it again after the replay.
  const SlotCtl* gate; uint32_t* blocked;
  DictView dict;
  EmitOut out;
};

// Multi-GPU pane exchange: one packet per (pane, group) partial state a rank holds for a key it does not own
// (DNZ_PARTIAL_BYTES = 64).  owner(key) = key hash % world (the NULL key belongs to rank 0).
struct __align__(16) PartialEntry {
  int64_t pane;
  unsigned long long cnt; double sum; unsigned long long minkey, maxkey;
  unsigned long long nullrows, fz;
  uint32_t key_off, key_len;     // bytes at key_off inside the sender's key segment FOR THIS OWNER; key_len == 0xFFFFFFFF: NULL key,
                                 // integer keys: width | key type << KEY_TYPE_SHIFT (below)
};
static_assert(sizeof(PartialEntry) == 64, "packet size");
// Group-key types: index = key type code (0 Utf8, 1 Int64, 2 Int32, 3 UInt64, 4 UInt32), the code a checkpoint records.  A packet
// of an integer key carries key_len = width | code << KEY_TYPE_SHIFT, so that the owner's merge detects a rank that groups by
// another key type; Utf8 packets carry the plain length (keys of 256 MiB or more are refused by the merge).
struct KeyType { const char* format; int32_t width; };           // format: the Arrow C format string (a literal)
constexpr KeyType KEY_TYPES[] = {{"u", 0}, {"l", 8}, {"i", 4}, {"L", 8}, {"I", 4}};
constexpr int N_KEY_TYPES = 5;
constexpr int KEY_TYPE_SHIFT = 28;
constexpr int MAX_WORLD = 32;
constexpr int PACK_PANES = 32;       // panes per pack launch (a 32-bit mask per group id)
// Where the write pass puts one owner's packets and key bytes: its segment of the local export buffers, or its reserved range
// of the owner's receive ring.  `entries` is the first packet of the range; its key bytes start at keys + key_off0, and a
// packet's key_off counts from `keys` (the segment: key_off0 = 0; the ring half: the reserved base).  entries == nullptr:
// write nothing for this owner.
struct PackDest { PartialEntry* entries; uint8_t* keys; uint32_t key_off0, pad; };
struct PackParams {
  uint32_t n_groups; int32_t rank, world, n_panes;
  const GroupState* st[PACK_PANES]; const unsigned long long* nullrows[PACK_PANES]; const unsigned long long* fz[PACK_PANES];
  int64_t pane[PACK_PANES];                      // up to PACK_PANES panes in one launch: one thread per group id walks them
  DictView dict;
  unsigned long long* owner_cursor;              // [world] (entries << 32) | key bytes, running over all launches of a pass
  const PackDest* dest;                          // [world] write pass: every owner's destination
  int32_t pass;                                  // 0: count, 1: write
  uint32_t key_tag;                              // key type code << KEY_TYPE_SHIFT, or'ed into key_len (0: Utf8)
};
struct MergeParams {
  const PartialEntry* entries; int64_t n_entries; const uint8_t* key_bytes;
  int32_t world;
  int32_t key_width;                             // 0: Utf8 keys; 4 / 8: integer keys (a packet's key bytes are the value, int_key)
  uint32_t key_tag;                              // what a packet of this key type carries above KEY_TYPE_SHIFT in key_len
  int64_t src_entry_end[MAX_WORLD];              // prefix sums over the sending ranks
  int64_t src_key_base[MAX_WORLD];
  DictView dict; PaneTable panes;
  uint32_t* error;                               // set when a table was full (the host sizes them beforehand)
};

// ------------------------------------------------------------------------------------------------
// launch wrappers (dnz_kernels.cu)
cudaError_t launch_tile_scan(const BatchDesc* batches, int64_t n_batches, int64_t n_tiles, int64_t pane_ms,
                             TileDesc* tiles, BatchMinMax* minmax, bool allow_fast, cudaStream_t s);
// key_width: 0 = Utf8 keys, 4 / 8 = integer keys (the instantiation of the kernel that matches the stream)
cudaError_t launch_aggregate(const AggParams& p, int key_width, int sm_count, cudaStream_t s);
int aggregate_grid(int64_t n_tiles, int sm_count);
cudaError_t launch_merge_private(const AggParams& p, int grid, cudaStream_t s);
cudaError_t launch_aggregate_generic(const AggParams& p, int key_width, int sm_count, cudaStream_t s);
cudaError_t launch_aggregate_ungrouped(const AggParams& p, int sm_count, cudaStream_t s);
// ungrouped windows: the panes of one closed window -> one partial state (read back by the host-side Final stage)
struct UWindow { const GroupState* st[MAX_WINDOW_PANES]; const unsigned long long* nr[MAX_WINDOW_PANES]; int32_t n, pad; };
struct UState { unsigned long long cnt; double sum; unsigned long long mink, maxk, nulls; };
cudaError_t launch_ungrouped_collect(const UWindow* wins, int n, UState* out, cudaStream_t s);
cudaError_t launch_deferred(const AggParams& p, int key_width, const DeferEntry* in, uint64_t n_entries, cudaStream_t s);
cudaError_t launch_emit(const EmitParams& p, cudaStream_t s);
cudaError_t launch_dict_rehash(const DictSlot* old_slots, uint32_t old_cap, DictView nd, cudaStream_t s);
cudaError_t launch_clear_hints(DictSlot* slots, uint32_t cap, cudaStream_t s);
cudaError_t launch_dict_restore(DictView d, uint32_t n, cudaStream_t s);
cudaError_t agg_kernel_setup();

// exchange (multi-GPU, dnz_exchange.cu)
cudaError_t launch_pack_partials(const PackParams& p, cudaStream_t s);
cudaError_t launch_merge_partials(const MergeParams& p, cudaStream_t s);

// fused exchange over peer memory: a rank's receive region (device memory of that rank, mapped into every peer)
struct XchgCtl {
  unsigned long long cursor[2];               // per ring half: (packets << 32) | key bytes reserved so far (remote atomicAdd by the senders)
  unsigned int error; unsigned int pad;
};
struct XchgRegion { XchgCtl* ctl; PartialEntry* entries; uint8_t* keys; };      // entries: 2 x ring_entries, keys: 2 x ring_key_bytes
struct XchgView {
  XchgRegion self; XchgRegion peer[MAX_WORLD];
  uint64_t ring_entries, ring_key_bytes;
  unsigned long long step;                    // 1, 2, ... (same on every rank)
  int32_t rank, world;
};
cudaError_t launch_xchg_reserve(const XchgView& X, unsigned long long* owner_cursor, PackDest* dest, unsigned long long* sent_total, uint32_t* err, cudaStream_t s);
cudaError_t launch_merge_ring(const MergeParams& p, const XchgView& X, unsigned long long* merged_total, int sm_count, cudaStream_t s);

// Arrow<->device buffer manager: one launch pulls every pinned host buffer of a superbatch over PCIe with 128-bit loads
// (hundreds of 0.5 MiB cudaMemcpyAsync calls reach only ~25 GB/s on this platform; see profiles/h2d_probe.py)
struct CopyDesc { const void* src; void* dst; uint64_t bytes; uint64_t first_piece; };   // pieces of 256 KiB, prefix over the list
constexpr uint64_t COPY_PIECE = 256 * 1024;
cudaError_t launch_gather_copy(const CopyDesc* descs, uint32_t n, unsigned int* cursor, cudaStream_t s);

// input-contract producer: canonical timestamps from a raw column (array_to_timestamp_array, utils/time.rs:59-94)
struct TsJob { const void* src; const int32_t* off; const uint8_t* bytes; int64_t* dst; int64_t n; };    // src: i64 values (kinds 2); off/bytes: Utf8 (kind 3)
constexpr int TS_FMT_MAX = 64;
struct TsFormat { char fmt[TS_FMT_MAX]; int32_t len; };
cudaError_t launch_ts_convert(const TsJob* jobs, int n_jobs, int64_t max_rows, int kind, const TsFormat& fmt, uint32_t* error, cudaStream_t s);
bool ts_format_supported(const char* fmt);

// synthetic generator (dnz_synth.cu)
cudaError_t launch_synth(int64_t row0, int64_t n_rows, int64_t batch_rows, uint64_t seed, int64_t groups,
                         int64_t rows_per_ms, int64_t t0_ms, int key_kind, int64_t key_mul, int64_t key_add, int64_t* ts, double* val, int32_t* off,
                         uint8_t* bytes, int64_t bytes_stride, cudaStream_t s);

}  // namespace dnz
