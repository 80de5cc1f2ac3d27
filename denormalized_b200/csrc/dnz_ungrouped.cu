// dnz_ungrouped.cu -- ungrouped windows `.window([], aggs, ..)`: the Partial stage's emission schedule and the Final stage
// (streaming_window.rs:882-1051), run on the host over the per-window states the device reduces.
#include "dnz_window.h"

// ungrouped windows (include/dnz_gpu.h, DNZ_NO_KEY)
namespace {
// get_windows_for_watermark (streaming_window.rs:1053-1086), whole-second snap (:1088-1094): the frames a batch creates
void reference_windows(int64_t mn, int64_t mx, int64_t L, int64_t S, std::vector<int64_t>& out) {
  auto snap = [&](int64_t ts) { const int64_t wl = L / 1000, t = ts / 1000; return (t / wl) * wl * 1000; };
  if (S > 0) { for (int64_t cur = snap(mn - L); cur <= mx; cur += S) { const int64_t end = cur + L; if (mn > end || mx < cur) continue; out.push_back(cur); } }
  else for (int64_t cur = snap(mn); cur <= mx; cur += L) out.push_back(cur);
}
inline long long total_key_of(double d) { unsigned long long b; memcpy(&b, &d, 8); return total_key(b); }
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
    if (u_head + n > u_ring) { ungrouped_collect(true); u_head = 0; }              // staging full: take in what is on its way first
    if (n > u_ring) {                                  // a run may close up to MAX_RUN_PANES windows: grow the staging, now idle
      u_ring = std::max(n, 2 * u_ring);
      d_uwins.alloc(u_ring * sizeof(UWindow)); d_ustates.alloc(u_ring * sizeof(UState));
      h_uwins.reserve(u_ring * sizeof(UWindow)); h_ustates.reserve(u_ring * sizeof(UState));
    }
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
      else { if (total_key_of(x.mn) < total_key_of(f.mn)) f.mn = x.mn; if (total_key_of(x.mx) > total_key_of(f.mx)) f.mx = x.mx; }
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
        unsigned long long bmn = unord_bits(~u.mink), bmx = unord_bits(u.maxk);
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
  else verify_completed();
  ungrouped_collect(blocking);
  const size_t n = u_out.size();
  ArrowBatch b(n, 8 * round_up(n * 8 + 8, 64) + round_up((n + 7) / 8 + 8, 64) + 1024, aggs.size() + 2);
  int64_t* cnt = (int64_t*)b.take(n * 8); double* mn = (double*)b.take(n * 8); double* mx = (double*)b.take(n * 8); double* avg = (double*)b.take(n * 8);
  double* sum = (double*)b.take(n * 8); int64_t* ws = (int64_t*)b.take(n * 8); int64_t* we = (int64_t*)b.take(n * 8);
  uint8_t* bm = (uint8_t*)b.take((n + 7) / 8 + 8); memset(bm, 0, (n + 7) / 8 + 8);
  int64_t nulls = 0;
  for (size_t i = 0; i < n; i++) {
    const URow& x = u_out[i];
    cnt[i] = x.cnt; mn[i] = x.mn; mx[i] = x.mx; avg[i] = x.avg; sum[i] = x.valid ? x.sum : 0.0; ws[i] = x.ws; we[i] = x.we;
    if (x.valid) bm[i >> 3] |= (uint8_t)(1u << (i & 7)); else nulls++;
  }
  hand_out(b, ExportColumns{nulls ? bm : nullptr, nulls, cnt, mn, mx, avg, sum, ws, we}, out, schema, has_output);
  u_out.clear();
}

