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

// ---- pack: thread per group id of one pane; two passes (count, then write) over every pane of the export ----------------
// pane j of the launch (a launch covers up to PACK_PANES panes; n_multi == 0: the single pane in st / nullrows / fz / pane)
struct PackPane { const GroupState* st; const unsigned long long* nu; const unsigned long long* fz; int64_t pane; };
__device__ __forceinline__ PackPane pack_pane(const PackParams& P, int j) {
  if (P.n_multi) return PackPane{P.mst[j], P.mnull[j], P.mfz[j], P.mpane[j]};
  return PackPane{P.st, P.nullrows, P.fz, P.pane};
}
// One thread per group id: which of the launch's panes hold something for it (bit mask), its key, its owner.
struct PackCell { uint32_t amask; bool null_key; uint32_t klen, kpad; int owner; GidKey gk; };
__device__ __forceinline__ PackCell pack_cell(const PackParams& P, uint32_t g) {
  PackCell c{}; c.amask = 0u;
  if (g >= P.n_groups || g >= min(*P.dict.n_groups, P.dict.gcap)) return c;    // n_groups may be an upper bound (fused path)
  const int np = P.n_multi ? P.n_multi : 1;
  for (int j = 0; j < np; j++) {
    const PackPane pp = pack_pane(P, j);
    const double cnt = pp.st[g].cnt;
    const unsigned long long nr = pp.nu ? pp.nu[g] : 0ull;
    if (!(cnt == 0.0 && nr == 0ull)) c.amask |= 1u << j;
  }
  if (!c.amask) return c;
  c.gk = P.dict.gid_key[g];
  c.null_key = c.gk.len == 0xFFFFFFFFu;
  c.klen = c.null_key ? 0u : c.gk.len;
  c.kpad = (c.klen + 7u) & ~7u;
  c.owner = c.null_key ? 0 : (int)((c.klen <= (uint32_t)INLINE_KEY ? hash_inline(c.gk.k0, c.gk.k1, c.klen) : c.gk.k0) % (uint64_t)P.world);
  if (c.owner == P.rank) c.amask = 0u;
  return c;
}
__device__ __forceinline__ PartialEntry pack_entry(const PackPane& pp, uint32_t g, uint32_t key_off, const PackCell& c) {
  const GroupState s = pp.st[g];
  PartialEntry e;
  e.pane = pp.pane; e.cnt = (unsigned long long)s.cnt; e.sum = s.sum; e.minkey = s.minkey; e.maxkey = s.maxkey;
  e.nullrows = pp.nu ? pp.nu[g] : 0ull; e.fz = pp.fz ? pp.fz[g] : ~0ull;
  e.key_off = key_off; e.key_len = c.null_key ? 0xFFFFFFFFu : c.klen;
  return e;
}

__global__ void __launch_bounds__(256) k_pack_partials(const __grid_constant__ PackParams P) {
  const uint32_t g = blockIdx.x * blockDim.x + threadIdx.x;
  const PackCell c = pack_cell(P, g);
  const uint32_t n = __popc(c.amask);
  const unsigned long long r = block_reserve(n != 0u, c.owner, n, n * c.kpad, P.owner_cursor, P.world);
  if (P.pass == 0 || !n) return;
  uint64_t row = (P.owner_base[c.owner] >> 32) + (r >> 32);
  uint32_t boff = (uint32_t)(r & 0xFFFFFFFFull);                          // inside this owner's key segment
  for (uint32_t m = c.amask; m; m &= m - 1u, row++, boff += c.kpad) {
    const PackPane pp = pack_pane(P, __ffs(m) - 1);
    P.entries[row] = pack_entry(pp, g, boff, c);
    if (!c.null_key) {
      uint8_t* dst = P.key_bytes + (P.owner_base[c.owner] & 0xFFFFFFFFull) + boff;
      if (c.klen <= (uint32_t)INLINE_KEY) {
        const uint64_t w[2] = {c.gk.k0, c.gk.k1};
        for (uint32_t i = 0; i < c.klen; i++) dst[i] = (uint8_t)(w[i >> 3] >> ((i & 7) * 8));
      } else {
        const uint8_t* src = P.dict.arena + c.gk.k1;
        for (uint32_t i = 0; i < c.klen; i++) dst[i] = src[i];
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
// Intern the packet's key (its bytes at `key`) and fold its partial state into the main pane it names.
__device__ __forceinline__ void merge_packet(const MergeParams& P, const PartialEntry& e, const uint8_t* key) {
  uint32_t gid;
  if (e.key_len == 0xFFFFFFFFu) gid = dict_lookup_null(P.dict);
  else {
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
//   k_pack_write_peer          write the packets and their key bytes straight into the owners' rings with P2P stores
//   [record: my packets of this step are written]  /  [wait: every peer's packets are written]
//   k_merge_ring               intern unknown keys, merge the received partial states into the owner's panes
//   [reset the ring half; record: merged]
//   k_emit ...                 the owner emits the closed windows of ITS keys
// =================================================================================================
__global__ void k_xchg_reserve(XchgView X, unsigned long long* owner_cursor, unsigned long long* owner_base, unsigned long long* sent_total, uint32_t* err) {
  const int o = threadIdx.x;
  if (o >= X.world || o == X.rank) return;
  const unsigned long long c = owner_cursor[o];
  unsigned long long base = 0;
  if (c) {
    base = atomicAdd_system(&X.peer[o].ctl->cursor[X.step & 1], c);
    if ((base >> 32) + (c >> 32) > X.ring_entries || (base & 0xFFFFFFFFull) + (c & 0xFFFFFFFFull) > X.ring_key_bytes) {
      atomicOr(&X.self.ctl->error, 1u); atomicOr(err, 0x100u);   // the owner's ring is too small for this step: nothing of it is written
      base = ~0ull;
    }
  }
  owner_base[o] = base;
  owner_cursor[o] = 0ull;
  atomicAdd(sent_total, c >> 32);
}
cudaError_t launch_xchg_reserve(const XchgView& X, unsigned long long* owner_cursor, unsigned long long* owner_base, unsigned long long* sent_total, uint32_t* err, cudaStream_t s) {
  k_xchg_reserve<<<1, MAX_WORLD, 0, s>>>(X, owner_cursor, owner_base, sent_total, err);
  return cudaGetLastError();
}

// pass 1 of the fused path: like k_pack_partials' write pass, but the destination is the owner's ring and key_off is absolute
// A 64 B packet leaves as four 128-bit stores, the widest store sm_90 has (a peer write travels NVLink per store instruction).
__device__ __forceinline__ void store_packet(PartialEntry* dst, const PartialEntry& e) {
  const unsigned long long* w = reinterpret_cast<const unsigned long long*>(&e);
#pragma unroll
  for (int i = 0; i < 4; i++)
    asm volatile("st.global.v2.b64 [%0], {%1, %2};" :: "l"(reinterpret_cast<char*>(dst) + 16 * i), "l"(w[2 * i]), "l"(w[2 * i + 1]) : "memory");
}
__global__ void __launch_bounds__(256) k_pack_write_peer(const __grid_constant__ PackParams P, const __grid_constant__ XchgView X, const unsigned long long* __restrict__ owner_base) {
  const uint32_t g = blockIdx.x * blockDim.x + threadIdx.x;
  PackCell c = pack_cell(P, g);
  unsigned long long base = 0ull;
  if (c.amask) { base = owner_base[c.owner]; if (base == ~0ull) c.amask = 0u; }      // the owner's ring overflowed: nothing is written
  const uint32_t n = __popc(c.amask);
  const unsigned long long r = block_reserve(n != 0u, c.owner, n, n * c.kpad, P.owner_cursor, P.world);
  if (!n) return;
  const int half = (int)(X.step & 1);
  uint64_t row = (base >> 32) + (r >> 32);
  uint64_t boff = (base & 0xFFFFFFFFull) + (r & 0xFFFFFFFFull);           // inside the owner's key half
  PartialEntry* ring = X.peer[c.owner].entries + (uint64_t)half * X.ring_entries;
  uint8_t* keys = X.peer[c.owner].keys + (uint64_t)half * X.ring_key_bytes;
  for (uint32_t m = c.amask; m; m &= m - 1u, row++, boff += c.kpad) {
    const PackPane pp = pack_pane(P, __ffs(m) - 1);
    store_packet(ring + row, pack_entry(pp, g, (uint32_t)boff, c));
    if (!c.null_key) {
      uint8_t* dst = keys + boff;
      if (c.klen <= (uint32_t)INLINE_KEY) {
        const uint64_t w[2] = {c.gk.k0, c.gk.k1};
        for (uint32_t i = 0; i < c.kpad; i += 8) *reinterpret_cast<uint64_t*>(dst + i) = w[i >> 3];   // 8 B aligned: key ranges are padded to 8
      } else {
        const uint8_t* src = P.dict.arena + c.gk.k1;                                                  // arena entries are 8 B aligned and padded
        for (uint32_t i = 0; i < c.kpad; i += 8) *reinterpret_cast<uint64_t*>(dst + i) = *reinterpret_cast<const uint64_t*>(src + i);
      }
    }
  }
}
cudaError_t launch_pack_write_peer(const PackParams& p, const XchgView& X, const unsigned long long* owner_base, cudaStream_t s) {
  if (!p.n_groups) return cudaSuccess;
  k_pack_write_peer<<<(p.n_groups + 255) / 256, 256, 0, s>>>(p, X, owner_base);
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
