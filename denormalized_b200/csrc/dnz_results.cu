// dnz_results.cu -- emitted rows: the two device result sets and their snapshots, and the hand-over to the consumer as Arrow
// C-Data (host) or as device columns.
#include "dnz_window.h"

namespace {

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
  CK(cudaMemsetAsync(&ctl()->result[i], 0, sizeof(ResultCursor), stream));
  r.rows = 0; r.bytes = 0; r.exp_rows = 0; r.exp_bytes = 0; r.snap_issued = false;
  for (Slot& s : slot) if (s.emit_set == i) { s.add_rows_bound = 0; s.add_bytes_bound = 0; }
}
void dnz_window::reset_results() { reset_set(wr); res_consumed = false; }

// cursor of the current set -> pinned memory, in stream order behind the emit launches
void dnz_window::snapshot_results() {
  ResultSet& r = R();
  CK(cudaMemcpyAsync(r.snap.p, &ctl()->result[wr], sizeof(ResultCursor), cudaMemcpyDeviceToHost, stream));
  CK(cudaEventRecord(r.snap_ev, stream));
  r.snap_issued = true;
}
// every row of the set has been handed out and nothing is in flight for it
bool dnz_window::set_drained(ResultSet& r) {
  if (!r.snap_issued) return r.exp_rows == r.rows;
  if (cudaEventQuery(r.snap_ev) != cudaSuccess) { cudaGetLastError(); return false; }
  uint64_t c = reinterpret_cast<volatile ResultCursor*>(r.snap.p)->cursor;
  return (c >> 32) == r.exp_rows;
}
// The rows of a set that are COMPLETE on the device: those below its newest snapshot, once that snapshot's event has fired
// (false: no such snapshot).
bool dnz_window::ready_rows(ResultSet& r, uint64_t& rows, uint64_t& bytes) {
  if (!r.snap_issued) return false;
  if (cudaEventQuery(r.snap_ev) != cudaSuccess) { cudaGetLastError(); return false; }
  const volatile ResultCursor* sp = reinterpret_cast<volatile ResultCursor*>(r.snap.p);
  const uint64_t c = sp->cursor;
  if (sp->overflow) fail(DNZ_ERR_NOMEM, "result buffer overflow (internal sizing error)");
  rows = c >> 32; bytes = c & 0xFFFFFFFFull;
  return true;
}
// Called before a superbatch's emits are enqueued (only matters when the consumer uses the non-blocking poll): reuse the
// current set in place when it is drained, else switch to the other one if that is drained, else keep appending.
void dnz_window::rotate_result_sets() {
  if (!async_polls) return;
  if (set_drained(rs[wr])) { if (rs[wr].exp_rows) reset_set(wr); return; }
  if (set_drained(rs[wr ^ 1])) { if (rs[wr ^ 1].exp_rows || rs[wr ^ 1].rows) reset_set(wr ^ 1); wr ^= 1; }
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
  // the input's key type (a literal: the schema outlives the operator); integer keys keep the input field's nullability
  if (!ungrouped) add(key_name, KEY_TYPES[key_type].format, (key_width == 0 || key_nullable) ? ARROW_FLAG_NULLABLE : 0);
  for (size_t i = 0; i < aggs.size(); i++) add(aliases[i], agg_format(aggs[i].kind), aggs[i].kind == DNZ_AGG_COUNT ? 0 : ARROW_FLAG_NULLABLE);
  add("window_start_time", "tsm:", 0);     // continuous/mod.rs:42-62: Timestamp(ms, None), non-null
  add("window_end_time", "tsm:", 0);
  for (size_t i = 0; i < nc; i++) { sp->children[i]->name = sp->names[i].c_str(); sp->child_ptrs.push_back(sp->children[i].get()); }
  memset(schema, 0, sizeof(*schema));
  schema->format = "+s"; schema->name = ""; schema->n_children = (int64_t)nc; schema->children = sp->child_ptrs.data();
  schema->release = release_schema; schema->private_data = sp;
}

// Completes an export whose key column (grouped windows) has been added: one column per aggregate, the window bounds, the
// struct array in `out` and the schema; the rows count as handed out.
void dnz_window::hand_out(ArrowBatch& b, const ExportColumns& c, ArrowArray* out, ArrowSchema* schema, int32_t* has_output) {
  for (auto& a : aggs) {
    switch (a.kind) {
      case DNZ_AGG_COUNT: b.add_child({nullptr, c.count}, 0); break;
      case DNZ_AGG_MIN: b.add_child({c.validity, c.mn}, c.nulls); break;
      case DNZ_AGG_MAX: b.add_child({c.validity, c.mx}, c.nulls); break;
      case DNZ_AGG_AVG: b.add_child({c.validity, c.avg}, c.nulls); break;
      default: b.add_child({c.validity, c.sum}, c.nulls); break;
    }
  }
  b.add_child({nullptr, c.ws}, 0);
  b.add_child({nullptr, c.we}, 0);
  ExportPrivate* ep = b.ep.get();
  for (auto& ch : ep->children) ep->child_ptrs.push_back(ch.get());
  ep->buffers.push_back({nullptr});
  memset(out, 0, sizeof(*out));
  out->length = b.n; out->null_count = 0; out->n_buffers = 1; out->buffers = ep->buffers.back().data();
  out->n_children = (int64_t)ep->children.size(); out->children = ep->child_ptrs.data(); out->release = release_array;
  out->private_data = b.ep.release();
  if (schema) fill_schema(schema);
  if (has_output) *has_output = b.n > 0;
  stats.rows_out += b.n;
}


// Hands out every emitted row that is COMPLETE on the device: per result set, the rows between what was exported before and
// the newest snapshot whose event has fired (older set first).  `blocking` callers have synchronised the stream, so every
// snapshot has fired; the non-blocking poll simply leaves rows of still-running emits for the next call.  The device->host
// copies run on their own stream, never behind queued input.
void dnz_window::export_arrow(ArrowArray* out, ArrowSchema* schema, int32_t* has_output, bool blocking) {
  if (ungrouped) { export_ungrouped(out, schema, has_output, blocking); return; }
  if (blocking) { CK(cudaStreamSynchronize(stream)); }
  else verify_completed();
  struct Range { ResultSet* r; uint64_t r0, r1, b0, b1; };
  std::vector<Range> ranges;
  for (int k = 0; k < 2; k++) {
    ResultSet& r = rs[k == 0 ? (wr ^ 1) : wr];
    uint64_t rows = 0, bytes = 0;
    if (!ready_rows(r, rows, bytes)) continue;
    if (rows > r.exp_rows) ranges.push_back(Range{&r, r.exp_rows, rows, r.exp_bytes, bytes});
  }
  uint64_t n = 0, nbytes = 0;
  for (auto& g : ranges) { n += g.r1 - g.r0; nbytes += g.b1 - g.b0; }
  if (nbytes >= (1ull << 31)) fail(DNZ_ERR_UNSUPPORTED, "more than 2 GiB of key bytes in one poll (Utf8 offsets are 32-bit); poll more often");
  ArrowBatch b(n, round_up((n + 1) * 4, 64) + round_up(nbytes, 64) + 2 * round_up(n, 64) + 7 * round_up(n * 8, 64) +
                    2 * round_up((n + 7) / 8 + 8, 64) + 1024, 1 + aggs.size() + 2);
  // one column of every range, back to back
  auto fetch = [&](DevBuf ResultSet::*col, size_t elem, bool by_bytes, size_t extra) -> void* {
    char* h = (char*)b.take((by_bytes ? nbytes : n) * elem + extra);
    size_t at = 0;
    for (auto& g : ranges) {
      const uint64_t lo = by_bytes ? g.b0 : g.r0, hi = by_bytes ? g.b1 : g.r1;
      const size_t bytes = (size_t)(hi - lo) * elem;
      if (bytes) { CK(cudaMemcpyAsync(h + at, (g.r->*col).template as<char>() + lo * elem, bytes, cudaMemcpyDeviceToHost, d2h_stream)); stats.d2h_bytes += (int64_t)bytes; }
      at += bytes;
    }
    return h;
  };
  // integer keys: key_bytes holds key_width bytes per row, the Arrow values buffer itself (no offsets)
  int32_t* koff = key_width ? nullptr : (int32_t*)fetch(&ResultSet::key_off, 4, false, 4);
  uint8_t* kbytes = (uint8_t*)fetch(&ResultSet::key_bytes, 1, true, 0);
  uint8_t* kvalid = (uint8_t*)fetch(&ResultSet::key_valid, 1, false, 0);
  int64_t* count = (int64_t*)fetch(&ResultSet::count, 8, false, 0);
  double* mn = (double*)fetch(&ResultSet::mn, 8, false, 0); double* mx = (double*)fetch(&ResultSet::mx, 8, false, 0);
  double* avg = (double*)fetch(&ResultSet::avg, 8, false, 0); double* sum = (double*)fetch(&ResultSet::sum, 8, false, 0);
  uint8_t* avalid = (uint8_t*)fetch(&ResultSet::agg_valid, 1, false, 0);
  int64_t* ws = (int64_t*)fetch(&ResultSet::wstart, 8, false, 0); int64_t* we = (int64_t*)fetch(&ResultSet::wend, 8, false, 0);
  CK(cudaStreamSynchronize(d2h_stream));
  if (koff) {   // key offsets are relative to each set's byte buffer: rebase them onto the concatenated export
    uint64_t row_at = 0, byte_at = 0;
    for (auto& g : ranges) {
      const int64_t delta = (int64_t)byte_at - (int64_t)g.b0;
      if (delta != 0) for (uint64_t i = row_at; i < row_at + (g.r1 - g.r0); i++) koff[i] = (int32_t)(koff[i] + delta);
      row_at += g.r1 - g.r0; byte_at += g.b1 - g.b0;
    }
  }
  if (koff) koff[n] = (int32_t)nbytes;
  // byte-per-row validity -> Arrow bitmaps
  auto pack = [&](const uint8_t* v, int64_t& nulls) -> uint8_t* {
    nulls = 0;
    for (uint64_t i = 0; i < n; i++) nulls += !v[i];
    if (!nulls) return nullptr;
    uint8_t* bm = (uint8_t*)b.take((n + 7) / 8 + 8);
    memset(bm, 0, (n + 7) / 8 + 8);
    for (uint64_t i = 0; i < n; i++) if (v[i]) bm[i >> 3] |= (uint8_t)(1u << (i & 7));
    return bm;
  };
  int64_t key_nulls = 0, agg_nulls = 0;
  uint8_t* kbm = pack(kvalid, key_nulls);
  uint8_t* abm = pack(avalid, agg_nulls);
  if (key_width) b.add_child({kbm, kbytes}, key_nulls);
  else b.add_child({kbm, koff, kbytes}, key_nulls);
  hand_out(b, ExportColumns{abm, agg_nulls, count, mn, mx, avg, sum, ws, we}, out, schema, has_output);
  for (auto& g : ranges) { g.r->exp_rows = g.r1; g.r->exp_bytes = g.b1; }
  if (blocking) {         // stream idle: drained sets can be recycled right away
    for (int i = 0; i < 2; i++) if (rs[i].exp_rows && set_drained(rs[i])) reset_set(i);
  }
}

// Device-resident hand-over: the oldest range of emitted rows that has not been handed out yet, one result set per call (call
// again until n_rows == 0 when both sets may hold rows).  blocking: everything has been aggregated and the stream is idle, so
// every emitted row is eligible.  Non-blocking: only rows whose emission is COMPLETE on the device; nothing queued is forced.
// key_off entries are offsets into `key_bytes` (the set's byte buffer); key_bytes_len is the offset at which the last returned
// key ends.  Integer keys: key_off = NULL, key_bytes = the values of the returned rows (key_width bytes each, the NULL key's
// zero-filled), key_bytes_len = n_rows * key_width.
void dnz_window::export_device(dnz_device_result* out, bool blocking) {
  if (ungrouped) fail(DNZ_ERR_UNSUPPORTED, "ungrouped windows finish on the host (Final stage): use dnz_window_poll / dnz_window_poll_ready");
  memset(out, 0, sizeof *out);
  ResultSet* r = nullptr; uint64_t r0 = 0, r1 = 0, b0 = 0, b1 = 0;
  if (blocking) fetch_ctl();
  else verify_completed();          // release the input of launches that have completed (never waits)
  for (int k = 0; k < 2 && !r; k++) {
    ResultSet& c = rs[k == 0 ? (wr ^ 1) : wr];
    uint64_t rows = c.rows, bytes = c.bytes;
    if (!blocking && !ready_rows(c, rows, bytes)) continue;
    if (rows > c.exp_rows) { r = &c; r0 = c.exp_rows; r1 = rows; b0 = c.exp_bytes; b1 = bytes; }
  }
  if (!r) return;
  r->exp_rows = r1; r->exp_bytes = b1;
  if (blocking) {          // stream idle: a set that has been handed out completely restarts at row 0 with the next emission
    for (int i = 0; i < 2; i++) if (rs[i].exp_rows && rs[i].exp_rows == rs[i].rows) reset_set(i);
  }
  out->n_rows = (int64_t)(r1 - r0); out->key_bytes_len = (int64_t)b1;
  out->key_off = r->key_off.as<int32_t>() + r0; out->key_bytes = r->key_bytes.as<uint8_t>(); out->key_valid = r->key_valid.as<uint8_t>() + r0;
  if (key_width) { out->key_off = nullptr; out->key_bytes += b0; out->key_bytes_len = (int64_t)(b1 - b0); }
  out->count = r->count.as<int64_t>() + r0; out->min = r->mn.as<double>() + r0; out->max = r->mx.as<double>() + r0;
  out->avg = r->avg.as<double>() + r0; out->sum = r->sum.as<double>() + r0; out->agg_valid = r->agg_valid.as<uint8_t>() + r0;
  out->window_start_ms = r->wstart.as<int64_t>() + r0; out->window_end_ms = r->wend.as<int64_t>() + r0;
  stats.rows_out += (int64_t)(r1 - r0);
}

