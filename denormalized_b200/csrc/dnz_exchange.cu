// dnz_exchange.cu -- multi-GPU pane exchange (SURVEY.md §8e): the all-to-all of per-pane partial aggregates that replaces
// RepartitionExec(Hash(group keys)) (physical_optimizer/coalesce_before_streaming_window_aggregate.rs:63-73) when the
// input is NOT key-partitioned: every GPU aggregates the batches it was dealt into its own panes; once a pane can no
// longer change, each GPU sends the states of the keys it does not own to their owners (owner = key hash % world), the
// owner merges them into its pane (count +, sum +, min / max over the ordered keys, null rows +, first-zero min) and
// emits the windows for its keys only (k_emit's owner filter).
#include "dnz_device.cuh"

namespace dnz {

// Positions in the per-owner output ranges.  One global atomic per thread on `world` addresses serialises in L2 (measured: 0.95 ms
// for 2 M cells on 2 owners); the block counts per owner in shared memory first and reserves each owner's block total with ONE
// global atomic.  A thread reserves `n` packets and `bytes` key bytes (one group id, all its non-empty panes of the launch); the
// result is (first row << 32 | first byte offset) relative to the owner's base.  Every thread of the block must call it (barriers).
__device__ __forceinline__ unsigned long long block_reserve(bool active, int owner, uint32_t n, uint32_t bytes, unsigned long long* owner_cursor, int world) {
  __shared__ uint32_t s_cnt[MAX_WORLD], s_bytes[MAX_WORLD];
  __shared__ unsigned long long s_base[MAX_WORLD];
  if (threadIdx.x < MAX_WORLD) { s_cnt[threadIdx.x] = 0u; s_bytes[threadIdx.x] = 0u; }
  __syncthreads();
  uint32_t lc = 0u, lb = 0u;
  if (active) { lc = atomicAdd(&s_cnt[owner], n); lb = atomicAdd(&s_bytes[owner], bytes); }
  __syncthreads();
  if ((int)threadIdx.x < world && s_cnt[threadIdx.x])
    s_base[threadIdx.x] = atomicAdd(owner_cursor + threadIdx.x, ((unsigned long long)s_cnt[threadIdx.x] << 32) | s_bytes[threadIdx.x]);
  __syncthreads();
  return active ? s_base[owner] + (((unsigned long long)lc << 32) | lb) : 0ull;
}

// ---- pack: thread per group id, up to PACK_PANES panes per launch; two passes (count, then write) over every pane sent ----
// One thread per group id: which of the launch's panes hold something for it (bit mask), its key, its owner.
struct PackCell { uint32_t amask; bool null_key; uint32_t klen, kpad; int owner; GidKey gk; };
__device__ __forceinline__ PackCell pack_cell(const PackParams& P, uint32_t g) {
  PackCell c{}; c.amask = 0u;
  if (g >= P.n_groups || g >= min(*P.dict.n_groups, P.dict.gcap)) return c;    // n_groups may be an upper bound (fused path)
  for (int j = 0; j < P.n_panes; j++) {
    const double cnt = P.st[j][g].cnt;
    const unsigned long long nr = P.nullrows[j] ? P.nullrows[j][g] : 0ull;
    if (!(cnt == 0.0 && nr == 0ull)) c.amask |= 1u << j;
  }
  if (!c.amask) return c;
  c.gk = P.dict.gid_key[g];
  c.null_key = c.gk.len == 0xFFFFFFFFu;
  c.klen = c.null_key ? 0u : c.gk.len;
  c.kpad = (c.klen + 7u) & ~7u;
  c.owner = key_owner(c.gk, P.world);
  if (c.owner == P.rank) c.amask = 0u;
  return c;
}
__device__ __forceinline__ PartialEntry pack_entry(const PackParams& P, int j, uint32_t g, uint32_t key_off, const PackCell& c) {
  const GroupState s = P.st[j][g];
  PartialEntry e;
  e.pane = P.pane[j]; e.cnt = (unsigned long long)s.cnt; e.sum = s.sum; e.minkey = s.minkey; e.maxkey = s.maxkey;
  e.nullrows = P.nullrows[j] ? P.nullrows[j][g] : 0ull; e.fz = P.fz[j] ? P.fz[j][g] : ~0ull;
  e.key_off = key_off; e.key_len = c.null_key ? 0xFFFFFFFFu : (c.klen | P.key_tag);
  return e;
}
// A 64 B packet leaves as four 128-bit stores, the widest store sm_90 has (a peer write travels NVLink per store instruction).
__device__ __forceinline__ void store_packet(PartialEntry* dst, const PartialEntry& e) {
  const unsigned long long* w = reinterpret_cast<const unsigned long long*>(&e);
#pragma unroll
  for (int i = 0; i < 4; i++)
    asm volatile("st.global.v2.b64 [%0], {%1, %2};" :: "l"(reinterpret_cast<char*>(dst) + 16 * i), "l"(w[2 * i]), "l"(w[2 * i + 1]) : "memory");
}

// Pass 0 counts every owner's packets and padded key bytes into owner_cursor.  Pass 1 reserves the same amounts again, from a
// zeroed cursor, inside every owner's destination and writes there: the packets, and each key as whole 8 B words (every key range
// is padded to 8 B and starts 8 B aligned; an arena entry is reserved in whole 8 B words, so reading kpad bytes stays inside it).
__global__ void __launch_bounds__(256) k_pack_partials(const __grid_constant__ PackParams P) {
  const uint32_t g = blockIdx.x * blockDim.x + threadIdx.x;
  const PackCell c = pack_cell(P, g);
  const uint32_t n = __popc(c.amask);
  const unsigned long long r = block_reserve(n != 0u, c.owner, n, n * c.kpad, P.owner_cursor, P.world);
  if (P.pass == 0 || !n) return;
  const PackDest d = P.dest[c.owner];
  if (!d.entries) return;                                                 // the owner's ring overflowed: nothing is written
  PartialEntry* out = d.entries + (r >> 32);
  uint32_t key_off = d.key_off0 + (uint32_t)(r & 0xFFFFFFFFull);
  for (uint32_t m = c.amask; m; m &= m - 1u, out++, key_off += c.kpad) {
    store_packet(out, pack_entry(P, __ffs(m) - 1, g, key_off, c));
    if (!c.null_key) {
      uint64_t* dst = reinterpret_cast<uint64_t*>(d.keys + key_off);
      if (c.klen <= (uint32_t)INLINE_KEY) {
        for (uint32_t i = 0; i < c.kpad / 8u; i++) dst[i] = i ? c.gk.k1 : c.gk.k0;
      } else {
        const uint64_t* src = reinterpret_cast<const uint64_t*>(P.dict.arena + c.gk.k1);
        for (uint32_t i = 0; i < c.kpad / 8u; i++) dst[i] = src[i];
      }
    }
  }
}
cudaError_t launch_pack_partials(const PackParams& p, cudaStream_t s) {
  if (!p.n_groups) return cudaSuccess;
  k_pack_partials<<<(p.n_groups + 255) / 256, 256, 0, s>>>(p);
  return cudaGetLastError();
}

// ---- merge: thread per received packet ---------------------------------------------------------------------------------
// Intern the packet's key (its bytes at `key`, 8 B aligned) and fold its partial state into the main pane it names.  Integer keys
// are rebuilt with int_key from the value the pack kernel wrote (the low key_width bytes of the stored k0).  A packet of another
// key type (its key_len carries the sender's type above KEY_TYPE_SHIFT) raises error bit 8 and is not merged.
__device__ __forceinline__ void merge_packet(const MergeParams& P, const PartialEntry& e, const uint8_t* key) {
  uint32_t gid;
  if (e.key_len == 0xFFFFFFFFu) gid = dict_lookup_null(P.dict);
  else if ((e.key_len >> KEY_TYPE_SHIFT) != (P.key_tag >> KEY_TYPE_SHIFT)) { atomicOr(P.error, 8u); return; }
  else if (P.key_width != 0) {
    if (e.key_len != (P.key_tag | (uint32_t)P.key_width)) { atomicOr(P.error, 8u); return; }
    gid = dict_lookup(P.dict, P.key_width == 8 ? load_int_key<8>(key, 0) : load_int_key<4>(key, 0), false);
  } else {
    KeyRef k; load_key<false>(key, e.key_len, k);
    gid = dict_lookup(P.dict, k, false);
  }
  const int64_t pi = e.pane - P.panes.pane0;
  if (gid >= GID_DEFER_ARENA || pi < 0 || pi >= P.panes.n_panes || P.panes.main[pi] == nullptr) { atomicOr(P.error, 1u); return; }
  GroupState* s = P.panes.main[pi] + gid;
  if (e.cnt) {
    red_add_f64(&s->cnt, (double)e.cnt); red_add_f64(&s->sum, e.sum);
    red_max_u64(&s->minkey, e.minkey); red_max_u64(&s->maxkey, e.maxkey);
  }
  if (e.nullrows) { if (P.panes.nullrows_main[pi]) red_add_u64(P.panes.nullrows_main[pi] + gid, e.nullrows); else atomicOr(P.error, 2u); }
  if (e.fz != ~0ull) { if (P.panes.fz_main[pi]) red_min_u64(P.panes.fz_main[pi] + gid, e.fz); else atomicOr(P.error, 4u); }
}

__global__ void __launch_bounds__(256) k_merge_partials(const __grid_constant__ MergeParams P) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= P.n_entries) return;
  const PartialEntry e = P.entries[i];
  int src = 0;
  while (src + 1 < P.world && i >= P.src_entry_end[src]) src++;
  merge_packet(P, e, P.key_bytes + P.src_key_base[src] + e.key_off);
}
cudaError_t launch_merge_partials(const MergeParams& p, cudaStream_t s) {
  if (p.n_entries <= 0) return cudaSuccess;
  k_merge_partials<<<(unsigned)((p.n_entries + 255) / 256), 256, 0, s>>>(p);
  return cudaGetLastError();
}


// =================================================================================================
// Fused pane exchange over peer memory (NVLink / NVSwitch): no host copy and no library collective in the data path.
//
// Every rank owns a RECEIVE region in its HBM (mapped into every peer with CUDA IPC): a cursor block, a ring of 64 B packets
// and a ring of key bytes, each split into two halves (step parity).  One exchange step of a rank, all on its own stream:
//
//   [wait: owners have merged step-2]      interprocess CUDA events, no spinning kernel
//   k_pack_partials (pass 0)   per-owner packet / key-byte counts of the panes that closed under the global watermark
//   k_xchg_reserve             one thread per owner: reserve the counted range in the OWNER'S ring with one remote atomicAdd
//   k_pack_partials (pass 1)   write the packets and their key bytes straight into the owners' rings with P2P stores
//   [record: my packets of this step are written]  /  [wait: every peer's packets are written]
//   k_merge_ring               intern unknown keys, merge the received partial states into the owner's panes
//   [reset the ring half; record: merged]
//   k_emit ...                 the owner emits the closed windows of ITS keys
// =================================================================================================
__global__ void k_xchg_reserve(XchgView X, unsigned long long* owner_cursor, PackDest* dest, unsigned long long* sent_total, uint32_t* err) {
  const int o = threadIdx.x;
  if (o >= X.world || o == X.rank) return;
  const unsigned long long c = owner_cursor[o];
  owner_cursor[o] = 0ull;
  atomicAdd(sent_total, c >> 32);
  dest[o].entries = nullptr;
  if (!c) return;
  const unsigned long long base = atomicAdd_system(&X.peer[o].ctl->cursor[X.step & 1], c);
  const uint64_t half = X.step & 1, row0 = base >> 32, byte0 = base & 0xFFFFFFFFull;
  if (row0 + (c >> 32) > X.ring_entries || byte0 + (c & 0xFFFFFFFFull) > X.ring_key_bytes) {
    atomicOr(&X.self.ctl->error, 1u); atomicOr(err, 0x100u);   // the owner's ring is too small for this step: nothing of it is written
    return;
  }
  dest[o] = PackDest{X.peer[o].entries + half * X.ring_entries + row0, X.peer[o].keys + half * X.ring_key_bytes, (uint32_t)byte0, 0u};
}
cudaError_t launch_xchg_reserve(const XchgView& X, unsigned long long* owner_cursor, PackDest* dest, unsigned long long* sent_total, uint32_t* err, cudaStream_t s) {
  k_xchg_reserve<<<1, MAX_WORLD, 0, s>>>(X, owner_cursor, dest, sent_total, err);
  return cudaGetLastError();
}

// merge everything the peers wrote into this rank's ring half of the step: grid-stride, the packet count is read on the device
__global__ void __launch_bounds__(256) k_merge_ring(const __grid_constant__ MergeParams P, const __grid_constant__ XchgView X, unsigned long long* merged_total) {
  const int half = (int)(X.step & 1);
  const unsigned long long cur = *reinterpret_cast<volatile unsigned long long*>(&X.self.ctl->cursor[half]);
  const uint64_t n = cur >> 32;
  const PartialEntry* ring = X.self.entries + (uint64_t)half * X.ring_entries;
  const uint8_t* keys = X.self.keys + (uint64_t)half * X.ring_key_bytes;
  if (blockIdx.x == 0 && threadIdx.x == 0) atomicAdd(merged_total, n);
  for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
    PartialEntry e;
    {   // packets were written by peers while this kernel may already have been resident: bypass L1
      const uint4* p4 = reinterpret_cast<const uint4*>(ring + i);
      uint4 a = __ldcg(p4), b = __ldcg(p4 + 1), c = __ldcg(p4 + 2), d = __ldcg(p4 + 3);
      memcpy(&e, &a, 16); memcpy(reinterpret_cast<char*>(&e) + 16, &b, 16); memcpy(reinterpret_cast<char*>(&e) + 32, &c, 16); memcpy(reinterpret_cast<char*>(&e) + 48, &d, 16);
    }
    merge_packet(P, e, keys + e.key_off);
  }
}
cudaError_t launch_merge_ring(const MergeParams& p, const XchgView& X, unsigned long long* merged_total, int sm_count, cudaStream_t s) {
  k_merge_ring<<<sm_count * 4, 256, 0, s>>>(p, X, merged_total);
  return cudaGetLastError();
}

}  // namespace dnz
