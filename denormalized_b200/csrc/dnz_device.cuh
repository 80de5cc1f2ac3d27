// dnz_device.cuh -- device helpers: PTX wrappers (mbarrier, cp.async.bulk, wide loads, reductions),
// key loading / hashing, dictionary probe+insert, per-row state update, fold of partial states.
#pragma once
#include "dnz_kernels.h"

namespace dnz {

// ---------------------------------------------------------------- PTX wrappers
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
// Releasing a ring slot only has to order the consumer's shared-memory READS of the slot before the producer's refill;
// those reads have completed once their values were used.  The default .release form also waits for every outstanding
// global reduction of the warp (an L2 round trip per tile).
__device__ __forceinline__ void mbar_arrive_relaxed(uint64_t* bar) {
  asm volatile("mbarrier.arrive.relaxed.cta.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, %3;\n\t"     // %3: suspend-time hint (ns): park the warp
      "selp.u32 %0, 1, 0, p;\n\t}"                                          // instead of spinning through issue slots
      : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity), "r"(0x989680u) : "memory");
  return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  while (!mbar_try_wait(bar, parity)) {}
}
// TMA 1-D bulk copy global -> shared, completion signalled on an mbarrier (SASS: UBLKCP.S.G).
__device__ __forceinline__ void bulk_g2s(void* dst_smem, const void* src_gmem, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(smem_u32(dst_smem)), "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}

// 16 B single accesses (SASS: LDG.E.128.STRONG.GPU / STG.E.128.STRONG.GPU), always served by L2: slots are written by
// other SMs (atomicCAS + release store) while we probe, and the per-SM L1 is not coherent -- an L1-cached copy of an
// EMPTY/LOCKED slot would make the probe loop spin forever.
__device__ __forceinline__ void ld_relaxed_b128(const void* p, uint64_t& lo, uint64_t& hi) {
  asm volatile("{\n\t.reg .b128 t;\n\tld.relaxed.gpu.global.b128 t, [%2];\n\tmov.b128 {%0, %1}, t;\n\t}" : "=l"(lo), "=l"(hi) : "l"(p) : "memory");
}
__device__ __forceinline__ void ld_acquire_b128(const void* p, uint64_t& lo, uint64_t& hi) {
  asm volatile("{\n\t.reg .b128 t;\n\tld.acquire.gpu.global.b128 t, [%2];\n\tmov.b128 {%0, %1}, t;\n\t}" : "=l"(lo), "=l"(hi) : "l"(p) : "memory");
}
__device__ __forceinline__ void st_relaxed_b128(void* p, uint64_t lo, uint64_t hi) {
  asm volatile("{\n\t.reg .b128 t;\n\tmov.b128 t, {%1, %2};\n\tst.relaxed.gpu.global.b128 [%0], t;\n\t}" :: "l"(p), "l"(lo), "l"(hi) : "memory");
}
// A slot is one 32 B sector; the widest load is 16 B, so a probe issues two independent loads in the same sector: the key
// words {k0, k1} (a, b) and {hint, len | state << 32} (c, d).  The two are not ordered, so a slot published between them
// reads as a published state with the key words it had before the insert.  Slots start zeroed and an insert writes the
// key words once, with one 16 B store, before it publishes: such a torn read always shows a == b == 0, and
// slot_keys_unsettled() sends it to ld_slot_ordered, which reads the key words behind an acquire of the state.
__device__ __forceinline__ void ld_slot(const DictSlot* p, uint64_t& a, uint64_t& b, uint64_t& c, uint64_t& d) {
  ld_relaxed_b128(&p->hint, c, d);
  ld_relaxed_b128(&p->k0, a, b);
}
// ld_slot for a warp, by lane pairs: lanes 2j / 2j+1 load the two 16 B halves of ONE slot per instruction, first the slot of
// the even lane's row (the even lane its key words, the odd lane its {hint, len | state}), then the slot of the odd lane's row
// (the odd lane its key words, the even lane its {hint, len | state}).  Each lane then holds its own key words and the other
// half of its partner's slot, and one xor-shuffle of 16 B swaps those.  A warp's 32 probes cost two instructions of 16 sector
// requests each instead of two of 32.  The halves stay two unordered loads (by two lanes now), so the torn-read argument of
// ld_slot holds unchanged.  Every lane of the warp calls it with a valid slot index `idx` (the loads are not predicated per
// row: the caller skips the call when no row of the warp probes, and a row that does not probe ignores what it got).
__device__ __forceinline__ void ld_slot_paired(const DictSlot* slots, uint32_t idx, uint32_t odd, uint64_t& a, uint64_t& b,
                                               uint64_t& c, uint64_t& d) {
  const uint32_t idx2 = __shfl_xor_sync(0xffffffffu, idx, 1);
  const uint8_t* base = reinterpret_cast<const uint8_t*>(slots);
  uint64_t x0, x1, y0, y1;
  ld_relaxed_b128(base + (size_t)(odd ? idx2 : idx) * sizeof(DictSlot) + 16u * odd, x0, x1);
  ld_relaxed_b128(base + (size_t)(odd ? idx : idx2) * sizeof(DictSlot) + 16u * (odd ^ 1u), y0, y1);
  // x: the even lane's row, y: the odd lane's row
  a = odd ? y0 : x0; b = odd ? y1 : x1;
  c = __shfl_xor_sync(0xffffffffu, odd ? x0 : y0, 1); d = __shfl_xor_sync(0xffffffffu, odd ? x1 : y1, 1);
}
__device__ __forceinline__ void ld_slot_ordered(const DictSlot* p, uint64_t& a, uint64_t& b, uint64_t& c, uint64_t& d) {
  ld_acquire_b128(&p->hint, c, d);
  ld_relaxed_b128(&p->k0, a, b);
}
__device__ __forceinline__ bool slot_keys_unsettled(uint64_t a, uint64_t b) { return (a | b) == 0ull; }
__device__ __forceinline__ uint32_t ld_acquire_u32(const uint32_t* p) {
  uint32_t v; asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory"); return v;
}
__device__ __forceinline__ void st_release_u32(uint32_t* p, uint32_t v) {
  asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ void st_relaxed_u64(uint64_t* p, uint64_t v) {
  asm volatile("st.relaxed.gpu.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ void red_add_u64(unsigned long long* p, unsigned long long v) {
  asm volatile("red.global.add.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ void red_add_f64(double* p, double v) {
  asm volatile("red.global.add.f64 [%0], %1;" ::"l"(p), "d"(v) : "memory");
}
__device__ __forceinline__ void red_max_u64(unsigned long long* p, unsigned long long v) {
  asm volatile("red.global.max.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ void red_min_u64(unsigned long long* p, unsigned long long v) {
  asm volatile("red.global.min.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}

// ---------------------------------------------------------------- hashing
__host__ __device__ __forceinline__ uint64_t mix64(uint64_t x) {
  x ^= x >> 32; x *= 0xD6E8FEB86659FD93ull; x ^= x >> 32; x *= 0xD6E8FEB86659FD93ull; x ^= x >> 32; return x;
}
// inline keys (<= 16 B, four zero-padded 32-bit words): 32-bit multiply-xorshift chain -- the slot index needs < 30 bits and
// 64-bit multiplies cost 3-4 IMADs each on the hot path
__host__ __device__ __forceinline__ uint32_t hash_words(uint32_t w0, uint32_t w1, uint32_t w2, uint32_t w3, uint32_t len) {
  // four INDEPENDENT multiplies (they issue back to back), rotated so that the digits of "sensor_123"-style keys land in
  // different bit ranges, summed, then murmur3's 32-bit finaliser: a shorter dependent chain in front of the dictionary
  // probe than a word-by-word chain, same probe lengths in simulation (1.119 vs 1.117 average at 19 % load)
  uint32_t a = w1 * 0xC2B2AE35u, b = w2 * 0x27D4EB2Fu, c = w3 * 0x165667B1u;
  uint32_t h = w0 * 0x85EBCA6Bu + ((a << 13) | (a >> 19)) + ((b << 21) | (b >> 11)) + ((c << 5) | (c >> 27)) + len * 0x9E3779B1u;
  h ^= h >> 16; h *= 0x85EBCA6Bu; h ^= h >> 13; h *= 0xC2B2AE35u; h ^= h >> 16;
  return h;
}
__host__ __device__ __forceinline__ uint64_t hash_inline(uint64_t k0, uint64_t k1, uint32_t len) {
  return hash_words((uint32_t)k0, (uint32_t)(k0 >> 32), (uint32_t)k1, (uint32_t)(k1 >> 32), len);
}
// hash of a key as DictSlot / GidKey hold it (a long key's k0 already is the hash of all its bytes)
__host__ __device__ __forceinline__ uint64_t stored_key_hash(uint64_t k0, uint64_t k1, uint32_t len) {
  return len <= (uint32_t)INLINE_KEY ? hash_inline(k0, k1, len) : k0;
}
// multi-GPU owner of a group: the rank that merges its partial states and emits it (the NULL key belongs to rank 0)
__host__ __device__ __forceinline__ int key_owner(const GidKey& gk, int world) {
  return gk.len == 0xFFFFFFFFu ? 0 : (int)(stored_key_hash(gk.k0, gk.k1, gk.len) % (uint64_t)world);
}

// A key as the dictionary sees it.
struct KeyRef {
  uint64_t k0, k1;       // inline words (long keys: k0 = hash of all bytes)
  uint64_t hash;
  uint32_t len;
  const uint8_t* ptr;    // original bytes (needed only for long keys)
};

// Stored form of an integer key (Arrow Int64 / Int32 / UInt64 / UInt32) of `width` bytes (4 or 8): k0 = the value's bits,
// zero-extended; k1 = INT_KEY_TAG; len = width.  An ordinary inline key from then on (hash, owner, placement, checkpoint, the
// pack kernel's key bytes).  The tag keeps the key words non-zero: all-zero key words are the probe's torn-read marker
// (slot_keys_unsettled), and with k1 = 0 every row of the key 0 would take the ordered reload and the full lookup.
// Every builder of an integer key goes through int_key, so one value can never become two groups.
constexpr uint64_t INT_KEY_TAG = 0x494E544B45594B31ull;    // "1KYEKTNI": any non-zero constant
__host__ __device__ __forceinline__ KeyRef int_key(uint64_t bits, uint32_t width) {
  KeyRef k;
  k.k0 = width == 4u ? (uint64_t)(uint32_t)bits : bits; k.k1 = INT_KEY_TAG; k.len = width; k.ptr = nullptr;
  k.hash = hash_inline(k.k0, k.k1, width);
  return k;
}
// the integer key of row `row` of a values buffer (naturally aligned: the host copy is, device batches are checked)
template <int KW>
__device__ __forceinline__ KeyRef load_int_key(const uint8_t* values, int64_t row) {
  static_assert(KW == 4 || KW == 8, "integer key width");
  if (KW == 8) return int_key((uint64_t)__ldg(reinterpret_cast<const unsigned long long*>(values) + row), 8u);
  return int_key((uint64_t)__ldg(reinterpret_cast<const uint32_t*>(values) + row), 4u);
}

// Load up to 16 key bytes from an arbitrarily aligned address using aligned 32-bit loads.
// Reading the aligned words that contain the first / last key byte never leaves their 4 B word, so it is
// safe for both shared and global memory.
template <bool SHARED>
__device__ __forceinline__ uint32_t ld_word(const uint8_t* p) {
  if (SHARED) { uint32_t v; asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(smem_u32(p))); return v; }
  return __ldg(reinterpret_cast<const uint32_t*>(p));
}
template <bool SHARED>
__device__ __forceinline__ void load_key(const uint8_t* p, uint32_t len, KeyRef& k) {
  k.len = len; k.ptr = p;
  if (len <= (uint32_t)INLINE_KEY) {
    uint32_t mis = (uint32_t)(reinterpret_cast<uintptr_t>(p) & 3u);
    const uint8_t* q = p - mis;
    uint32_t nw = (mis + len + 3u) >> 2;            // aligned words holding the key (<= 5)
    uint32_t a[5];
#pragma unroll
    for (int i = 0; i < 5; i++) a[i] = (uint32_t)i < nw ? ld_word<SHARED>(q + 4 * i) : 0u;
    uint32_t w[4];
    uint32_t sh = mis * 8u;
#pragma unroll
    for (int i = 0; i < 4; i++) w[i] = __funnelshift_r(a[i], i < 4 ? a[i + 1] : 0u, sh);
#pragma unroll
    for (int i = 0; i < 4; i++) {                    // zero the bytes past len
      uint32_t lo = 4u * i;
      uint32_t keep = len <= lo ? 0u : (len - lo >= 4u ? 0xFFFFFFFFu : ((1u << ((len - lo) * 8u)) - 1u));
      w[i] &= keep;
    }
    k.k0 = (uint64_t)w[0] | ((uint64_t)w[1] << 32); k.k1 = (uint64_t)w[2] | ((uint64_t)w[3] << 32);
    k.hash = hash_inline(k.k0, k.k1, len);
  } else {
    // long key: two 32-bit multiply-xorshift lanes over its little-endian 32-bit words (aligned loads + funnel shifts; the
    // byte-at-a-time version cost ~250 instructions for a 36 B UUID and was the whole kernel for such streams)
    const uint32_t mis = (uint32_t)(reinterpret_cast<uintptr_t>(p) & 3u), sh = mis * 8u;
    const uint8_t* q = p - mis;
    const uint32_t nk = (len + 3u) >> 2, nw = (mis + len + 3u) >> 2;
    uint32_t h1 = 0x9E3779B1u * (len + 1u), h2 = 0x85EBCA77u ^ len;
    uint32_t prev = ld_word<SHARED>(q);
    for (uint32_t i = 0; i < nk; i++) {
      const uint32_t next = (i + 1u < nw) ? ld_word<SHARED>(q + 4u * (i + 1u)) : 0u;
      uint32_t w = __funnelshift_r(prev, next, sh);
      prev = next;
      if (i + 1u == nk && (len & 3u)) w &= (1u << ((len & 3u) * 8u)) - 1u;
      h1 = (h1 ^ w) * 0x85EBCA6Bu; h1 ^= h1 >> 15;
      h2 = (h2 + w) * 0xC2B2AE3Du; h2 = (h2 << 13) | (h2 >> 19);
    }
    h1 ^= h2 * 0x27D4EB2Fu; h1 ^= h1 >> 16; h1 *= 0x165667B1u; h1 ^= h1 >> 13;
    h2 ^= h1 * 0x9E3779B1u; h2 ^= h2 >> 15; h2 *= 0x85EBCA6Bu; h2 ^= h2 >> 16;
    const uint64_t h = ((uint64_t)h2 << 32) | h1;
    k.k0 = h; k.k1 = 0; k.hash = h;
  }
}

__device__ __forceinline__ uint8_t ld_key_byte(const uint8_t* p, bool shared) {
  if (shared) { uint32_t v; asm volatile("ld.shared.u8 %0, [%1];" : "=r"(v) : "r"(smem_u32(p))); return (uint8_t)v; }
  return __ldg(p);
}

// ---------------------------------------------------------------- dictionary
enum : uint32_t { GID_DEFER_GROUPS = 0xFFFFFFFEu, GID_DEFER_ARENA = 0xFFFFFFFDu };

// Publish a slot this thread has LOCKED: the key words with one 16 B store (what ld_slot's torn-read argument relies on), the
// length, then the state with a release store.
__device__ __forceinline__ void slot_publish(DictSlot* slot, uint64_t k0, uint64_t k1, uint32_t len, uint32_t state) {
  st_relaxed_b128(&slot->k0, k0, k1);
  slot->len = len;
  __threadfence();
  st_release_u32(&slot->state, state);
}

// Place a key that is not in the table yet (rehash, checkpoint restore): claim the first empty slot from `hash`, set its hint
// before the publish.  Keys are never compared, so no two threads may place the same key.
__device__ __forceinline__ void dict_place(const DictView& d, uint64_t hash, uint64_t k0, uint64_t k1, uint32_t len, uint64_t hint,
                                           uint32_t state) {
  uint32_t idx = (uint32_t)hash & d.mask;
  while (atomicCAS(&d.slots[idx].state, SLOT_EMPTY, SLOT_LOCKED) != SLOT_EMPTY) idx = (idx + 1) & d.mask;
  d.slots[idx].hint = hint;
  slot_publish(d.slots + idx, k0, k1, len, state);
}

// Try to claim `slot` for key k.  Returns gid, or GID_DEFER_* when a table is full, or 0xFFFFFFFF when the CAS was
// lost (caller re-examines the slot).
__device__ __forceinline__ uint32_t dict_try_insert(const DictView& d, DictSlot* slot, uint32_t slot_idx, const KeyRef& k,
                                                   bool key_shared) {
  unsigned long long arena_off = 0;
  if (k.len > (uint32_t)INLINE_KEY) {                // reserve arena space first (a lost race leaks a few bytes)
    unsigned long long need = (k.len + 7ull) & ~7ull;
    arena_off = atomicAdd(d.arena_used, need);
    if (arena_off + need > d.arena_cap) return GID_DEFER_ARENA;
  }
  uint32_t old = atomicCAS(&slot->state, SLOT_EMPTY, SLOT_LOCKED);
  if (old != SLOT_EMPTY) return 0xFFFFFFFFu;
  // group id: one atomicAdd (a CAS loop on this single counter serialises every inserter on the chip).  The counter may
  // run past gcap; ids >= gcap are never used (the rows are deferred) and the host clamps the counter before it grows.
  uint32_t g = atomicAdd(d.n_groups, 1u);
  if (g >= d.gcap) { st_release_u32(&slot->state, SLOT_EMPTY); return GID_DEFER_GROUPS; }
  // slot_publish's protocol, written out: k_aggregate's machine code is held as it is, with the gid_key store and the byte count
  // between the length store and the fence
  if (k.len > (uint32_t)INLINE_KEY) {
    for (uint32_t i = 0; i < k.len; i++) d.arena[arena_off + i] = ld_key_byte(k.ptr + i, key_shared);
    st_relaxed_b128(&slot->k0, k.k0, arena_off);
  } else {
    st_relaxed_b128(&slot->k0, k.k0, k.k1);         // one store: see ld_slot
  }                                                  // slot->hint stays 0 (= no hint) from the zero fill
  slot->len = k.len;
  d.gid_key[g] = GidKey{k.k0, k.len > (uint32_t)INLINE_KEY ? arena_off : k.k1, k.len, 0u};
  atomicAdd(d.key_bytes_total, (unsigned long long)k.len);
  __threadfence();
  st_release_u32(&slot->state, g + 1);
  return g;
}

__device__ __forceinline__ bool dict_long_equal(const DictView& d, uint64_t arena_off, const KeyRef& k, bool key_shared) {
  // word-wise; arena entries are 8 B aligned.  __ldcg: arena bytes of OTHER keys sharing an L1 sector may have been cached
  // before this key was written
  const uint32_t* aw = reinterpret_cast<const uint32_t*>(d.arena + arena_off);
  const uint32_t mis = (uint32_t)(reinterpret_cast<uintptr_t>(k.ptr) & 3u), sh = mis * 8u;
  const uint8_t* q = k.ptr - mis;
  const uint32_t nk = (k.len + 3u) >> 2, nw = (mis + k.len + 3u) >> 2;
  uint32_t prev = key_shared ? ld_word<true>(q) : ld_word<false>(q);
  for (uint32_t i = 0; i < nk; i++) {
    const uint32_t next = (i + 1u < nw) ? (key_shared ? ld_word<true>(q + 4u * (i + 1u)) : ld_word<false>(q + 4u * (i + 1u))) : 0u;
    uint32_t w = __funnelshift_r(prev, next, sh), a = __ldcg(aw + i);
    prev = next;
    if (i + 1u == nk && (k.len & 3u)) { const uint32_t m = (1u << ((k.len & 3u) * 8u)) - 1u; w &= m; a &= m; }
    if (w != a) return false;
  }
  return true;
}

// Examine one slot.  Returns: gid (found or inserted) / GID_DEFER_* / 0xFFFFFFFF = keep probing.
// `advance` is set when the probe must move to the next slot (occupied by a different key).
__device__ __forceinline__ uint32_t dict_step(const DictView& d, uint32_t idx, const KeyRef& k, bool key_shared, bool& advance) {
  DictSlot* slot = d.slots + idx;
  uint64_t a, b, hint, w3;
  ld_slot(slot, a, b, hint, w3);
  uint32_t state = (uint32_t)(w3 >> 32);
  if (state - 1u < 0xFFFFFFFEu && slot_keys_unsettled(a, b)) { ld_slot_ordered(slot, a, b, hint, w3); state = (uint32_t)(w3 >> 32); }
  const uint32_t len = (uint32_t)w3;
  advance = false;
  if (state == SLOT_EMPTY) {
    uint32_t g = dict_try_insert(d, slot, idx, k, key_shared);
    return g;                                  // 0xFFFFFFFF: lost the race -> re-read the same slot
  }
  if (state == SLOT_LOCKED) return 0xFFFFFFFFu;  // insert in flight -> re-read
  bool eq;
  if (k.len <= (uint32_t)INLINE_KEY) eq = (len == k.len) && a == k.k0 && b == k.k1;
  else eq = (len == k.len) && a == k.k0 && dict_long_equal(d, b, k, key_shared);
  if (eq) return state - 1;
  advance = true;
  return 0xFFFFFFFFu;
}

__device__ __forceinline__ uint32_t dict_lookup_null(const DictView& d) {
  for (;;) {
    uint32_t s = ld_acquire_u32(d.null_gid);
    if (s != 0 && s != SLOT_LOCKED) return s - 1;
    if (s == 0) {
      uint32_t old = atomicCAS(d.null_gid, 0u, SLOT_LOCKED);
      if (old != 0) continue;
      uint32_t g = atomicAdd(d.n_groups, 1u);
      if (g >= d.gcap) { st_release_u32(d.null_gid, 0u); return GID_DEFER_GROUPS; }
      d.gid_key[g] = GidKey{0ull, 0ull, 0xFFFFFFFFu, 0u};
      __threadfence();
      st_release_u32(d.null_gid, g + 1);
      return g;
    }
  }
}

// full lookup (used by the generic / deferred / merge paths and by the staged kernel's slow path)
__device__ __forceinline__ uint32_t dict_lookup(const DictView& d, const KeyRef& k, bool key_shared, uint32_t* slot_out = nullptr) {
  uint32_t idx = (uint32_t)k.hash & d.mask;
  for (;;) {
    bool adv;
    uint32_t g = dict_step(d, idx, k, key_shared, adv);
    if (g != 0xFFFFFFFFu) { if (slot_out) *slot_out = idx; return g; }
    if (adv) idx = (idx + 1) & d.mask;
    else __nanosleep(100);      // slot locked by an insert in flight (possibly by another lane of this warp): let it finish
  }
}

// ---------------------------------------------------------------- per-row accumulator update
// DataFusion-42 semantics (SURVEY.md §8a-5): count += 1 per non-null value; min: `if cur > v`, max: `if cur < v`
// from f64::MAX / f64::MIN (NaN never replaces, +inf never lowers min's start, -inf never raises max's start,
// the first +-0.0 wins); avg = sum / count.
__device__ __forceinline__ void state_update(GroupState* st, unsigned long long* fz, uint32_t gid, double v,
                                             unsigned long long rowseq) {
  GroupState* s = st + gid;
  unsigned long long bits = (unsigned long long)__double_as_longlong(v);
  if (v == 0.0) {                      // both zeros order as +0.0; remember which one came first
    red_min_u64(fz + gid, (rowseq << 1) | (bits >> 63));
    bits = 0ull;
  }
  red_add_f64(&s->cnt, 1.0);
  red_add_f64(&s->sum, v);
  unsigned long long o = ord_bits(bits);
  if (v <= 1.7976931348623157e308) red_max_u64(&s->minkey, ORD_F64_MAX - o);    // false for NaN and +inf
  if (v >= -1.7976931348623157e308) red_max_u64(&s->maxkey, o - ORD_F64_MIN);   // false for NaN and -inf
}

// Fold of partial states (per-CTA copies, warp partials, panes), added in the caller's order: counts add; the sum starts at the
// first partial with a non-zero count, so that an empty partial never adds +0.0 to a -0.0 sum; minkey / maxkey take the max.
// Count: double, or an exact integer where the caller keeps one.
template <typename Count>
struct StateFold {
  Count cnt = 0; double sum = 0.0; unsigned long long mnk = 0, mxk = 0; bool first = true;
  __device__ __forceinline__ void add(const GroupState& s) {
    if (s.cnt != 0.0) { sum = first ? s.sum : sum + s.sum; first = false; }
    cnt += (Count)s.cnt; mnk = max(mnk, s.minkey); mxk = max(mxk, s.maxkey);
  }
};

__device__ __forceinline__ void defer_row(const DeferList& dl, uint32_t tile, uint32_t row, uint32_t why) {
  atomicOr(dl.flags, why);
  unsigned long long i = atomicAdd(dl.count, 1ull);
  if (i < dl.cap) dl.entries[i] = DeferEntry{tile, row};
  else atomicOr(dl.flags, (uint32_t)DEFER_LIST_OVERFLOW);
}

__device__ __forceinline__ bool bit_at(const uint8_t* bm, int64_t i) { return (__ldg(bm + (i >> 3)) >> (i & 7)) & 1; }

}  // namespace dnz
