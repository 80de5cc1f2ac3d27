// dnz_group.cu -- multi-GPU pane exchange: the host-driven export / import of partials and the dnz_group communicator.
#include "dnz_window.h"

#include <fcntl.h>
#include <sys/mman.h>
#include <unistd.h>

#include <atomic>

// ------------------------------------------------------------------------------------------------
// pane exchange (see include/dnz_gpu.h)
namespace {
// One pack launch per PACK_PANES panes of `send` (one thread per group id walks the panes of its launch).
template <class Launch> void for_pane_chunks(PackParams& P, const std::vector<Pane*>& send, Launch&& launch) {
  for (size_t i0 = 0; i0 < send.size(); i0 += PACK_PANES) {
    P.n_panes = (int32_t)std::min<size_t>(PACK_PANES, send.size() - i0);
    for (int j = 0; j < P.n_panes; j++) {
      const Pane* p = send[i0 + j];
      P.st[j] = p->st.as<GroupState>(); P.nullrows[j] = p->nullrows.as<unsigned long long>(); P.fz[j] = p->fz.as<unsigned long long>(); P.pane[j] = p->id;
    }
    launch();
  }
}
}  // namespace

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
  d_owner_cursor.reserve((size_t)world * 8); d_pack_dest.reserve((size_t)world * sizeof(PackDest));
  h_small.reserve((size_t)std::max<size_t>(256, world * sizeof(PackDest)));
  PackParams P; memset(&P, 0, sizeof P);
  P.n_groups = n_groups_host; P.rank = rank; P.world = world; P.dict = dict_view(); P.key_tag = key_tag();
  P.owner_cursor = d_owner_cursor.as<unsigned long long>(); P.dest = d_pack_dest.as<PackDest>();
  auto run_pass = [&](int pass) {
    CK(cudaMemsetAsync(d_owner_cursor.p, 0, (size_t)world * 8, stream));
    P.pass = pass;
    for_pane_chunks(P, send, [&] { CK(launch_pack_partials(P, stream)); stats.total_launches++; });
  };
  run_pass(0);
  CK(cudaMemcpyAsync(h_small.p, d_owner_cursor.p, (size_t)world * 8, cudaMemcpyDeviceToHost, stream));
  CK(cudaStreamSynchronize(stream));
  uint64_t n_total = 0, b_total = 0;
  for (int o = 0; o < world; o++) {
    uint64_t c = h_small.as<uint64_t>()[o];
    h_owner_counts[(size_t)o] = (int64_t)(c >> 32); h_owner_bytes[(size_t)o] = (int64_t)(c & 0xFFFFFFFFull);
    n_total += c >> 32; b_total += c & 0xFFFFFFFFull;
    if (n_total >= (1ull << 31) || b_total >= (1ull << 31)) fail(DNZ_ERR_UNSUPPORTED, "more than 2^31 packets or key bytes in one exchange step");
  }
  if (n_total == 0) return;
  d_part_entries.reserve((size_t)n_total * sizeof(PartialEntry)); d_part_keys.reserve((size_t)b_total + 64);
  PackDest* dest = h_small.as<PackDest>();                     // the owners' segments, in rank order
  int64_t n_seg = 0, b_seg = 0;
  for (int o = 0; o < world; o++) {
    dest[o] = PackDest{d_part_entries.as<PartialEntry>() + n_seg, d_part_keys.as<uint8_t>() + b_seg, 0u, 0u};
    n_seg += h_owner_counts[(size_t)o]; b_seg += h_owner_bytes[(size_t)o];
  }
  CK(cudaMemcpyAsync(d_pack_dest.p, dest, (size_t)world * sizeof(PackDest), cudaMemcpyHostToDevice, stream));
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
  for (int64_t p = pane_lo; p <= pane_hi; p++) ensure_side_arrays(get_pane(p, true));
  const size_t pb = (size_t)(pane_hi - pane_lo + 1) * sizeof(void*);
  h_xptrs.reserve(7 * pb); d_xptrs.reserve(7 * pb);
  M.panes = upload_pane_table(h_xptrs.as<void*>(), d_xptrs.as<char>(), pane_lo, pane_hi, [&](int64_t p) { return std::make_pair(get_pane(p, false), (Pane*)nullptr); });
  CK(cudaMemsetAsync(&ctl()->merge_err, 0, 4, stream));
  M.entries = reinterpret_cast<const PartialEntry*>(entries); M.n_entries = n; M.key_bytes = key_bytes; M.world = world; M.key_width = key_width; M.key_tag = key_tag();
  M.dict = dict_view(); M.error = &ctl()->merge_err;
  CK(launch_merge_partials(M, stream)); stats.total_launches++;
  fetch_ctl();
  uint32_t err = h_small.as<CtlBlock>()->merge_err;
  if (err & 8u) fail(DNZ_ERR_INVALID, "pane exchange: the packets hold keys of another type than this operator's group key (every rank must group by the same key type)");
  if (err) fail(DNZ_ERR_NOMEM, "pane merge failed (flags %u): table sizing error", err);
  stats.exchanged_in += n;
}

// =================================================================================================
// dnz_group: the library-owned communicator of the fused pane exchange (SURVEY.md §8b "dnz_group_create"; §8e).
// One rank per GPU.  Multi-process groups (one process per GPU, the production shape) map every rank's receive region into every
// peer with CUDA IPC, order the streams of different ranks with INTERPROCESS CUDA EVENTS (no kernel ever spins) and exchange the
// per-step host scalars (local watermark, first pane) through a POSIX shared-memory block; the rendezvous needs two all-gathers
// of a few hundred bytes at creation, which the host application supplies as a callback (the role the ncclUniqueId broadcast
// plays for NCCL).  Local groups put all ranks into one process (tests; several GPUs driven by one process): same kernels,
// same protocol, plain events.
// =================================================================================================
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
  DevBuf d_owner_cursor, d_pack_dest, d_totals;   // totals: [0] packets sent, [1] packets merged
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
  g->d_owner_cursor.alloc(MAX_WORLD * 8); g->d_pack_dest.alloc(MAX_WORLD * sizeof(PackDest)); g->d_totals.alloc(64);
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
  verify_completed();
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
  P.n_groups = gcap; P.rank = rank; P.world = world; P.dict = dict_view(); P.key_tag = key_tag();      // grid bound; the kernels clamp to the device counter
  P.owner_cursor = g->d_owner_cursor.as<unsigned long long>(); P.dest = g->d_pack_dest.as<PackDest>();
  auto pack = [&] { CK(launch_pack_partials(P, stream)); stats.total_launches++; };
  P.pass = 0;
  for_pane_chunks(P, send, pack);
  CK(launch_xchg_reserve(X, g->d_owner_cursor.as<unsigned long long>(), g->d_pack_dest.as<PackDest>(), g->d_totals.as<unsigned long long>(), &ctl()->merge_err, stream));
  stats.total_launches++;
  P.pass = 1;
  for_pane_chunks(P, send, pack);
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
      for (int64_t p = gfirst; p <= hi; p++) ensure_side_arrays(get_pane(p, true));
      // The pane table is staged in page-locked memory and copied by the stream when it gets there: the staging half may only be
      // rewritten once the copy issued two steps ago (same half) has executed -- its merge has been recorded in ev_merged[rank][mp].
      const size_t half_bytes = (size_t)7 * (1 << 16) * sizeof(void*);
      if (g->staged[mp]) CK(cudaEventSynchronize(g->ev_merged[rank][mp]));
      g->staged[mp] = true;
      g_tr.mark("x_sync_merged");
      MergeParams M; memset(&M, 0, sizeof M);
      M.panes = upload_pane_table(reinterpret_cast<void**>(h_xptrs.as<char>() + (size_t)mp * half_bytes), d_xptrs.as<char>() + (size_t)mp * half_bytes,
                                  gfirst, hi, [&](int64_t p) { return std::make_pair(get_pane(p, false), (Pane*)nullptr); });
      M.world = world; M.key_width = key_width; M.key_tag = key_tag(); M.dict = dict_view(); M.error = &ctl()->merge_err;
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
      emit_normal(R.gwm, nullptr);
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
  return create_guarded([&] {
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
  }, [&] { delete g; });
}

int32_t dnz_group_create_local(int32_t world, const int32_t* devices, int64_t ring_entries, int64_t ring_key_bytes, dnz_group** out) {
  if (!out || !devices) { g_last_error = "null argument"; return DNZ_ERR_INVALID; }
  std::vector<dnz_group*> gs;
  return create_guarded([&] {
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
  }, [&] { for (auto* g : gs) delete g; });
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
  InProcess scope(w);                                                               \
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
