/*
 * dnz_oracle.c -- CPU restatement of Denormalized's grouped streaming-window aggregate.
 * TEST INFRASTRUCTURE ONLY (see dnz_oracle.h).  PARITY UNPINNED (see dnz_oracle.h).
 *
 * The code deliberately performs the same passes over the data as the reference does
 * (two materialised filter copies per overlapping window, key interning, then one pass per
 * accumulator), so that the same routine serves as ground truth and as the timed CPU baseline.
 */
#define _GNU_SOURCE
#include "dnz_oracle.h"
#include <math.h>
#include <pthread.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

/* ------------------------------------------------------------------------------------------ */
/* small helpers                                                                               */

static inline int bit_get(const uint8_t* bm, int64_t i) { return bm == NULL || ((bm[i >> 3] >> (i & 7)) & 1); }
static inline void bit_set(uint8_t* bm, int64_t i) { bm[i >> 3] |= (uint8_t)(1u << (i & 7)); }

static void* xrealloc(void* p, size_t n) {
  void* q = realloc(p, n ? n : 1);
  if (!q) { fprintf(stderr, "dnz_oracle: out of memory (%zu)\n", n); abort(); }
  return q;
}
static void* xcalloc(size_t n, size_t s) {
  void* q = calloc(n ? n : 1, s ? s : 1);
  if (!q) { fprintf(stderr, "dnz_oracle: out of memory\n"); abort(); }
  return q;
}

static inline uint64_t hash_bytes(const uint8_t* p, int64_t n) {
  /* any good hash will do: results do not depend on it (the reference uses ahash). */
  uint64_t h = 0x9E3779B97F4A7C15ull ^ ((uint64_t)n * 0xff51afd7ed558ccdull);
  while (n >= 8) { uint64_t w; memcpy(&w, p, 8); h = (h ^ w) * 0x9FB21C651E98DF25ull; h ^= h >> 32; p += 8; n -= 8; }
  uint64_t w = 0; if (n > 0) memcpy(&w, p, (size_t)n);
  h = (h ^ w) * 0x9FB21C651E98DF25ull; h ^= h >> 29; h *= 0xBF58476D1CE4E5B9ull; h ^= h >> 32;
  return h;
}

/* IEEE-754 totalOrder, as f64::total_cmp (arrow-ord 53 cmp kernels for floats). */
static inline int64_t total_order_key(double d) {
  int64_t b; memcpy(&b, &d, 8);
  b ^= (int64_t)(((uint64_t)(b >> 63)) >> 1);
  return b;
}
static int total_cmp(double a, double b) {
  int64_t x = total_order_key(a), y = total_order_key(b);
  return (x > y) - (x < y);
}

/* ------------------------------------------------------------------------------------------ */
/* a materialised (filtered) batch: what filter_record_batch produces                          */

typedef struct {
  int64_t n, cap, bytes_cap, bar_bytes_cap;
  int64_t* ts; uint8_t* ts_valid;
  double* val; uint8_t* val_valid;
  int32_t* key_off; uint8_t* key_bytes; uint8_t* key_valid;
  int64_t* occurred_at;
  int32_t* barrier_off; uint8_t* barrier_bytes;
  int has_ts_valid, has_val_valid, has_key_valid, has_occ, has_bar;
} own_batch;

static void own_batch_free(own_batch* o) {
  free(o->ts); free(o->ts_valid); free(o->val); free(o->val_valid); free(o->key_off); free(o->key_bytes);
  free(o->key_valid); free(o->occurred_at); free(o->barrier_off); free(o->barrier_bytes);
  memset(o, 0, sizeof(*o));
}

static void own_batch_reserve(own_batch* o, int64_t n, int64_t key_bytes, int64_t bar_bytes) {
  if (n + 1 > o->cap) {
    int64_t c = n + 1;
    o->ts = xrealloc(o->ts, c * 8); o->val = xrealloc(o->val, c * 8);
    o->key_off = xrealloc(o->key_off, c * 4); o->barrier_off = xrealloc(o->barrier_off, c * 4);
    o->occurred_at = xrealloc(o->occurred_at, c * 8);
    o->ts_valid = xrealloc(o->ts_valid, (c + 7) / 8 + 1); o->val_valid = xrealloc(o->val_valid, (c + 7) / 8 + 1);
    o->key_valid = xrealloc(o->key_valid, (c + 7) / 8 + 1);
    o->cap = c;
  }
  if (key_bytes > o->bytes_cap) { o->key_bytes = xrealloc(o->key_bytes, key_bytes); o->bytes_cap = key_bytes; }
  if (bar_bytes > o->bar_bytes_cap) { o->barrier_bytes = xrealloc(o->barrier_bytes, bar_bytes); o->bar_bytes_cap = bar_bytes; }
}

static orc_batch own_as_view(const own_batch* o) {
  orc_batch v;
  v.n = o->n; v.ts = o->ts; v.ts_valid = o->has_ts_valid ? o->ts_valid : NULL;
  v.val = o->val; v.val_valid = o->has_val_valid ? o->val_valid : NULL;
  v.key_off = o->key_off; v.key_bytes = o->key_bytes; v.key_valid = o->has_key_valid ? o->key_valid : NULL;
  v.occurred_at = o->has_occ ? o->occurred_at : NULL;
  v.barrier_off = o->has_bar ? o->barrier_off : NULL; v.barrier_bytes = o->has_bar ? o->barrier_bytes : NULL;
  return v;
}

/* filter_record_batch(batch, mask): copies EVERY column (grouped_window_agg_stream.rs:573,600).
 * mask semantics: null timestamp -> comparison is null -> row dropped. */
static void filter_copy(const orc_batch* in, int cmp_ge, int64_t bound, own_batch* out) {
  int64_t n = in->n;
  int64_t kb = n > 0 ? (int64_t)in->key_off[n] - in->key_off[0] : 0;
  int64_t bb = (in->barrier_off && n > 0) ? (int64_t)in->barrier_off[n] - in->barrier_off[0] : 0;
  own_batch_reserve(out, n, kb, bb);
  out->has_ts_valid = in->ts_valid != NULL; out->has_val_valid = in->val_valid != NULL;
  out->has_key_valid = in->key_valid != NULL; out->has_occ = in->occurred_at != NULL;
  out->has_bar = in->barrier_off != NULL;
  if (out->has_ts_valid) memset(out->ts_valid, 0, (size_t)((n + 7) / 8 + 1));
  if (out->has_val_valid) memset(out->val_valid, 0, (size_t)((n + 7) / 8 + 1));
  if (out->has_key_valid) memset(out->key_valid, 0, (size_t)((n + 7) / 8 + 1));
  int64_t m = 0; int32_t ko = 0, bo = 0;
  out->key_off[0] = 0; out->barrier_off[0] = 0;
  for (int64_t i = 0; i < n; i++) {
    if (!bit_get(in->ts_valid, i)) continue;
    int64_t t = in->ts[i];
    int keep = cmp_ge ? (t >= bound) : (t < bound);
    if (!keep) continue;
    out->ts[m] = t; if (out->has_ts_valid) bit_set(out->ts_valid, m);
    out->val[m] = in->val[i]; if (out->has_val_valid && bit_get(in->val_valid, i)) bit_set(out->val_valid, m);
    int32_t a = in->key_off[i], b = in->key_off[i + 1];
    memcpy(out->key_bytes + ko, in->key_bytes + a, (size_t)(b - a)); ko += b - a; out->key_off[m + 1] = ko;
    if (out->has_key_valid && bit_get(in->key_valid, i)) bit_set(out->key_valid, m);
    if (out->has_occ) out->occurred_at[m] = in->occurred_at[i];
    if (out->has_bar) {
      int32_t c = in->barrier_off[i], d = in->barrier_off[i + 1];
      memcpy(out->barrier_bytes + bo, in->barrier_bytes + c, (size_t)(d - c)); bo += d - c; out->barrier_off[m + 1] = bo;
    }
    m++;
  }
  out->n = m;
}

/* ------------------------------------------------------------------------------------------ */
/* GroupedAggWindowFrame                                                                       */

typedef struct {
  int64_t start_ms, end_ms;
  /* GroupValues: open-addressing map key bytes -> dense group id (first-seen order) */
  int64_t tab_cap;           /* power of two */
  int32_t* tab_gid;          /* -1 empty */
  uint64_t* tab_hash;
  int64_t n_groups, g_cap;
  int32_t* g_off; int64_t g_bytes_cap; uint8_t* g_bytes;  /* key arena; g_off[n_groups+1] */
  int32_t null_gid;          /* -1 until a NULL key is seen */
  /* accumulators, indexed by group id */
  int64_t* cnt;              /* CountGroupsAccumulator */
  double* mn; double* mx;    /* PrimitiveGroupsAccumulator<Float64> */
  uint8_t* mn_seen; uint8_t* mx_seen;   /* NullState */
  double* sum; uint64_t* avg_cnt;       /* AvgGroupsAccumulator */
  /* scratch */
  int64_t* gids; int64_t gids_cap;
  own_batch f1, f2;
} frame_t;

static frame_t* frame_new(int64_t start_ms, int64_t end_ms) {
  frame_t* f = xcalloc(1, sizeof(frame_t));
  f->start_ms = start_ms; f->end_ms = end_ms; f->null_gid = -1;
  f->tab_cap = 64; f->tab_gid = xrealloc(NULL, f->tab_cap * 4); f->tab_hash = xrealloc(NULL, f->tab_cap * 8);
  for (int64_t i = 0; i < f->tab_cap; i++) f->tab_gid[i] = -1;
  f->g_off = xcalloc(1, 4);
  return f;
}
static void frame_free(frame_t* f) {
  free(f->tab_gid); free(f->tab_hash); free(f->g_off); free(f->g_bytes); free(f->cnt); free(f->mn); free(f->mx);
  free(f->mn_seen); free(f->mx_seen); free(f->sum); free(f->avg_cnt); free(f->gids);
  own_batch_free(&f->f1); own_batch_free(&f->f2); free(f);
}

static void frame_grow_groups(frame_t* f, int64_t need) {
  if (need <= f->g_cap) return;
  int64_t c = f->g_cap ? f->g_cap * 2 : 64; while (c < need) c *= 2;
  f->g_off = xrealloc(f->g_off, (c + 1) * 4);
  f->cnt = xrealloc(f->cnt, c * 8); f->mn = xrealloc(f->mn, c * 8); f->mx = xrealloc(f->mx, c * 8);
  f->mn_seen = xrealloc(f->mn_seen, c); f->mx_seen = xrealloc(f->mx_seen, c);
  f->sum = xrealloc(f->sum, c * 8); f->avg_cnt = xrealloc(f->avg_cnt, c * 8);
  f->g_cap = c;
}
static int32_t frame_new_group(frame_t* f, const uint8_t* p, int32_t len) {
  frame_grow_groups(f, f->n_groups + 1);
  int32_t g = (int32_t)f->n_groups++;
  int32_t o = f->g_off[g];
  if (o + len > f->g_bytes_cap) { int64_t c = f->g_bytes_cap ? f->g_bytes_cap * 2 : 1024; while (c < o + len) c *= 2; f->g_bytes = xrealloc(f->g_bytes, c); f->g_bytes_cap = c; }
  if (len) memcpy(f->g_bytes + o, p, (size_t)len);
  f->g_off[g + 1] = o + len;
  /* accumulator starting values */
  f->cnt[g] = 0; f->mn[g] = 1.7976931348623157e308 /* f64::MAX */; f->mx[g] = -1.7976931348623157e308 /* f64::MIN */;
  f->mn_seen[g] = 0; f->mx_seen[g] = 0; f->sum[g] = 0.0; f->avg_cnt[g] = 0;
  return g;
}
static void frame_rehash(frame_t* f) {
  int64_t nc = f->tab_cap * 2;
  int32_t* ng = xrealloc(NULL, nc * 4); uint64_t* nh = xrealloc(NULL, nc * 8);
  for (int64_t i = 0; i < nc; i++) ng[i] = -1;
  for (int64_t i = 0; i < f->tab_cap; i++) if (f->tab_gid[i] >= 0) {
    int64_t s = (int64_t)(f->tab_hash[i] & (uint64_t)(nc - 1));
    while (ng[s] >= 0) s = (s + 1) & (nc - 1);
    ng[s] = f->tab_gid[i]; nh[s] = f->tab_hash[i];
  }
  free(f->tab_gid); free(f->tab_hash); f->tab_gid = ng; f->tab_hash = nh; f->tab_cap = nc;
}
/* GroupValues::intern for one Utf8 key column */
static void frame_intern(frame_t* f, const orc_batch* b) {
  if (b->n > f->gids_cap) { f->gids = xrealloc(f->gids, b->n * 8); f->gids_cap = b->n; }
  for (int64_t i = 0; i < b->n; i++) {
    if (!bit_get(b->key_valid, i)) {
      if (f->null_gid < 0) f->null_gid = frame_new_group(f, NULL, 0);
      f->gids[i] = f->null_gid; continue;
    }
    const uint8_t* p = b->key_bytes + b->key_off[i]; int32_t len = b->key_off[i + 1] - b->key_off[i];
    uint64_t h = hash_bytes(p, len);
    int64_t s = (int64_t)(h & (uint64_t)(f->tab_cap - 1));
    for (;;) {
      int32_t g = f->tab_gid[s];
      if (g < 0) {
        g = frame_new_group(f, p, len);
        f->tab_gid[s] = g; f->tab_hash[s] = h; f->gids[i] = g;
        if ((f->n_groups + 1) * 2 > f->tab_cap) frame_rehash(f);
        break;
      }
      if (f->tab_hash[s] == h && g != f->null_gid && f->g_off[g + 1] - f->g_off[g] == len &&
          memcmp(f->g_bytes + f->g_off[g], p, (size_t)len) == 0) { f->gids[i] = g; break; }
      s = (s + 1) & (f->tab_cap - 1);
    }
  }
}

/* group_aggregate_batch (:501-537): intern, then one update_batch pass per accumulator */
static void frame_aggregate(frame_t* f, const orc_batch* b) {
  frame_intern(f, b);
  const int64_t* g = f->gids; int64_t n = b->n;
  /* count(reading) */
  for (int64_t i = 0; i < n; i++) if (bit_get(b->val_valid, i)) f->cnt[g[i]] += 1;
  /* min(reading): if *cur > new { *cur = new } */
  for (int64_t i = 0; i < n; i++) if (bit_get(b->val_valid, i)) { double v = b->val[i]; f->mn_seen[g[i]] = 1; if (f->mn[g[i]] > v) f->mn[g[i]] = v; }
  /* max(reading): if *cur < new { *cur = new } */
  for (int64_t i = 0; i < n; i++) if (bit_get(b->val_valid, i)) { double v = b->val[i]; f->mx_seen[g[i]] = 1; if (f->mx[g[i]] < v) f->mx[g[i]] = v; }
  /* avg(reading): sums[g] += v in row order; counts[g] += 1 */
  for (int64_t i = 0; i < n; i++) if (bit_get(b->val_valid, i)) { f->sum[g[i]] += b->val[i]; f->avg_cnt[g[i]] += 1; }
}

/* GroupedAggWindowFrame::push (:548-605) */
static void frame_push(frame_t* f, const orc_batch* b) {
  filter_copy(b, 1, f->start_ms, &f->f1);              /* cmp::gt_eq(ts, window_start) + filter_record_batch */
  orc_batch v1 = own_as_view(&f->f1);
  filter_copy(&v1, 0, f->end_ms, &f->f2);              /* cmp::lt(ts, window_end) + filter_record_batch */
  orc_batch v2 = own_as_view(&f->f2);
  frame_aggregate(f, &v2);
}

/* ------------------------------------------------------------------------------------------ */
/* result set                                                                                  */

typedef struct {
  int64_t n, cap, bytes, bytes_cap;
  int32_t* key_off; uint8_t* key_bytes; uint8_t* key_isnull;
  int64_t* count; double* mn; double* mx; double* avg; double* sum; uint8_t* agg_isnull;
  int64_t* ws; int64_t* we; int64_t* seq;
} results_t;

static void results_free(results_t* r) {
  free(r->key_off); free(r->key_bytes); free(r->key_isnull); free(r->count); free(r->mn); free(r->mx); free(r->avg); free(r->sum);
  free(r->agg_isnull); free(r->ws); free(r->we); free(r->seq); memset(r, 0, sizeof(*r));
}
static void results_push(results_t* r, const uint8_t* key, int32_t len, int key_isnull, int64_t count, double mn, double mx,
                         double avg, double sum, int agg_isnull, int64_t ws, int64_t we, int64_t seq) {
  if (r->n + 1 > r->cap) {
    int64_t c = r->cap ? r->cap * 2 : 1024;
    r->key_off = xrealloc(r->key_off, (c + 1) * 4); r->key_isnull = xrealloc(r->key_isnull, c);
    r->count = xrealloc(r->count, c * 8); r->mn = xrealloc(r->mn, c * 8); r->mx = xrealloc(r->mx, c * 8);
    r->avg = xrealloc(r->avg, c * 8); r->sum = xrealloc(r->sum, c * 8); r->agg_isnull = xrealloc(r->agg_isnull, c);
    r->ws = xrealloc(r->ws, c * 8); r->we = xrealloc(r->we, c * 8); r->seq = xrealloc(r->seq, c * 8);
    if (r->cap == 0) r->key_off[0] = 0;
    r->cap = c;
  }
  if (r->bytes + len > r->bytes_cap) { int64_t c = r->bytes_cap ? r->bytes_cap * 2 : 4096; while (c < r->bytes + len) c *= 2; r->key_bytes = xrealloc(r->key_bytes, c); r->bytes_cap = c; }
  if (len) memcpy(r->key_bytes + r->bytes, key, (size_t)len);
  r->bytes += len;
  int64_t i = r->n++;
  r->key_off[i + 1] = (int32_t)r->bytes; r->key_isnull[i] = (uint8_t)key_isnull;
  r->count[i] = count; r->mn[i] = mn; r->mx[i] = mx; r->avg[i] = avg; r->sum[i] = sum; r->agg_isnull[i] = (uint8_t)agg_isnull;
  r->ws[i] = ws; r->we[i] = we; r->seq[i] = seq;
}

/* ------------------------------------------------------------------------------------------ */
/* GroupedWindowAggStream                                                                      */

struct orc_window {
  orc_config cfg;
  frame_t** frames; int64_t n_frames, frames_cap;   /* BTreeMap<SystemTime, frame>: kept sorted by start */
  int has_wm; int64_t wm_ms;
  int64_t seq;
  results_t res;
  char err[256];
};

orc_window* orc_create(const orc_config* cfg) {
  orc_window* w = xcalloc(1, sizeof(orc_window));
  w->cfg = *cfg;
  return w;
}
void orc_destroy(orc_window* w) {
  if (!w) return;
  for (int64_t i = 0; i < w->n_frames; i++) frame_free(w->frames[i]);
  free(w->frames); results_free(&w->res); free(w);
}
const char* orc_last_error(const orc_window* w) { return w->err; }
int64_t orc_open_frames(const orc_window* w) { return w->n_frames; }
int64_t orc_watermark(const orc_window* w) { return w->has_wm ? w->wm_ms : INT64_MIN; }
void orc_clear_results(orc_window* w) { w->res.n = 0; w->res.bytes = 0; }
void orc_get_results(orc_window* w, orc_result* o) {
  static const int32_t zero_off[1] = {0};
  o->n = w->res.n; o->key_off = w->res.key_off ? w->res.key_off : zero_off; o->key_bytes = w->res.key_bytes;
  o->key_isnull = w->res.key_isnull; o->count = w->res.count; o->min = w->res.mn; o->max = w->res.mx; o->avg = w->res.avg;
  o->agg_isnull = w->res.agg_isnull; o->window_start_ms = w->res.ws; o->window_end_ms = w->res.we; o->emit_seq = w->res.seq;
  o->sum = w->res.sum;
}

/* snap_to_window_start (streaming_window.rs:1088-1094): whole-second arithmetic */
static int64_t snap_to_window_start(int64_t ts_ms, int64_t window_ms) {
  int64_t wl_s = window_ms / 1000, t_s = ts_ms / 1000;
  return (t_s / wl_s) * wl_s * 1000;
}

static frame_t* find_or_insert_frame(orc_window* w, int64_t start, int64_t end) {
  int64_t lo = 0, hi = w->n_frames;
  while (lo < hi) { int64_t mid = (lo + hi) / 2; if (w->frames[mid]->start_ms < start) lo = mid + 1; else hi = mid; }
  if (lo < w->n_frames && w->frames[lo]->start_ms == start) return w->frames[lo];
  if (w->n_frames + 1 > w->frames_cap) { w->frames_cap = w->frames_cap ? w->frames_cap * 2 : 16; w->frames = xrealloc(w->frames, w->frames_cap * sizeof(frame_t*)); }
  memmove(w->frames + lo + 1, w->frames + lo, (size_t)(w->n_frames - lo) * sizeof(frame_t*));
  w->frames[lo] = frame_new(start, end); w->n_frames++;
  return w->frames[lo];
}

static int filter_pass(const orc_config* c, int64_t count, double mn, double mx, double avg, double sum, int agg_isnull) {
  if (!c->has_filter) return 1;
  int cmp;
  if (c->filter_col == ORC_COL_COUNT) {
    /* Int64 column against a literal: DataFusion coerces both sides to a common type; with a Float64
     * literal the count is cast to Float64. */
    cmp = total_cmp((double)count, c->filter_lit);
  } else {
    if (agg_isnull) return 0;      /* null predicate -> row dropped */
    double v = c->filter_col == ORC_COL_MIN ? mn : c->filter_col == ORC_COL_MAX ? mx : c->filter_col == ORC_COL_SUM ? sum : avg;
    cmp = total_cmp(v, c->filter_lit);
  }
  switch (c->filter_op) {
    case ORC_OP_GT: return cmp > 0; case ORC_OP_GTE: return cmp >= 0; case ORC_OP_LT: return cmp < 0;
    case ORC_OP_LTE: return cmp <= 0; case ORC_OP_EQ: return cmp == 0; default: return cmp != 0;
  }
}

/* frame.evaluate() + add_window_columns_to_record_batch + FilterExec */
static int64_t emit_frame(orc_window* w, frame_t* f) {
  int64_t emitted = 0;
  for (int64_t g = 0; g < f->n_groups; g++) {
    int isnull = !f->mn_seen[g];                  /* NullState: null until first non-null value */
    double avg = isnull ? 0.0 : f->sum[g] / (double)f->avg_cnt[g];
    double mn = isnull ? 0.0 : f->mn[g], mx = isnull ? 0.0 : f->mx[g];
    double sum = isnull ? 0.0 : f->sum[g];        /* sum(reading): PrimitiveGroupsAccumulator, +0.0 then += v in row order */
    if (!filter_pass(&w->cfg, f->cnt[g], mn, mx, avg, sum, isnull)) continue;
    results_push(&w->res, f->g_bytes + f->g_off[g], f->g_off[g + 1] - f->g_off[g], (int32_t)g == f->null_gid,
                 f->cnt[g], mn, mx, avg, sum, isnull, f->start_ms, f->end_ms, w->seq);
    emitted++;
  }
  return emitted;
}

static int batch_watermark(const orc_batch* b, int64_t* mn, int64_t* mx) {
  int any = 0; int64_t lo = INT64_MAX, hi = INT64_MIN;
  for (int64_t i = 0; i < b->n; i++) if (bit_get(b->ts_valid, i)) { int64_t t = b->ts[i]; any = 1; if (t < lo) lo = t; if (t > hi) hi = t; }
  *mn = lo; *mx = hi; return any;
}

/* shared by the single- and multi-partition streams: everything poll_next_inner does for one
 * non-empty batch EXCEPT that the batch watermark may be supplied by the caller (multi-partition mode). */
static int64_t stream_push(orc_window* w, const orc_batch* b, int use_given_wm, int64_t given_min, int64_t given_max, int aggregate) {
  int64_t L = w->cfg.window_ms, S = w->cfg.slide_ms;
  int64_t mn, mx;
  if (use_given_wm) { mn = given_min; mx = given_max; }
  else if (!batch_watermark(b, &mn, &mx)) { snprintf(w->err, sizeof w->err, "all-null canonical_timestamp (reference: unwrap on None panics)"); return -1; }
  if (L / 1000 == 0) { snprintf(w->err, sizeof w->err, "window length < 1 s: snap_to_window_start divides by zero"); return -2; }
  if (mn < 0 || (S > 0 && mn - L < 0)) { snprintf(w->err, sizeof w->err, "timestamp before epoch(+window): duration_since(UNIX_EPOCH) panics"); return -3; }
  if (aggregate) {
    /* get_windows_for_watermark (streaming_window.rs:1053-1086) */
    if (S > 0) {
      int64_t cur = snap_to_window_start(mn - L, L);
      while (cur <= mx) {
        int64_t end = cur + L;
        if (mn > end || mx < cur) { cur += S; continue; }
        frame_push(find_or_insert_frame(w, cur, end), b);
        cur += S;
      }
    } else {
      int64_t cur = snap_to_window_start(mn, L);
      while (cur <= mx) { int64_t end = cur + L; frame_push(find_or_insert_frame(w, cur, end), b); cur = end; }
    }
  }
  /* process_watermark (:255-266) */
  if (!w->has_wm || w->wm_ms <= mn) { w->wm_ms = mn; w->has_wm = 1; }
  /* trigger_windows (:220-253) */
  int64_t emitted = 0, keep = 0;
  for (int64_t i = 0; i < w->n_frames; i++) {
    frame_t* f = w->frames[i];
    if (w->wm_ms >= f->end_ms) { emitted += emit_frame(w, f); frame_free(f); }
    else w->frames[keep++] = f;
  }
  w->n_frames = keep;
  return emitted;
}

int64_t orc_push(orc_window* w, const orc_batch* b) {
  int64_t r = 0;
  if (b->n > 0) r = stream_push(w, b, 0, 0, 0, 1);   /* empty batch: returns an empty batch, no trigger (:331,:343-345) */
  w->seq++;
  return r;
}

/* ------------------------------------------------------------------------------------------ */
/* multi-threaded hash-partition mode (timed CPU baseline)                                     */

struct orc_mt {
  orc_config cfg; int P; int64_t CH;
  orc_window** parts;
  /* persistent worker pool + scratch: [CH][P] sub-batches produced by the partitioning phase of the current chunk */
  pthread_t* th; struct mt_arg* args;
  pthread_barrier_t bar_start, bar_mid, bar_end;
  own_batch* subs; int64_t* wm_min; int64_t* wm_max; int* wm_any;
  const orc_batch* batches; int64_t c0, c1; int stop;
  char err[256];
};

typedef struct mt_arg { orc_mt* m; int tid; int64_t emitted; int err; } mt_arg;

static void* mt_worker(void* vp);

orc_mt* orc_mt_create(const orc_config* cfg, int partitions) {
  orc_mt* m = xcalloc(1, sizeof(orc_mt));
  m->cfg = *cfg; m->P = partitions < 1 ? 1 : partitions;
  int P = m->P;
  m->CH = P * 2 > 16 ? P * 2 : 16;                 /* batches per chunk: bounds the partition scratch */
  m->parts = xcalloc(P, sizeof(orc_window*));
  for (int p = 0; p < P; p++) m->parts[p] = orc_create(cfg);
  m->subs = xcalloc((size_t)(m->CH * P), sizeof(own_batch));
  m->wm_min = xcalloc(m->CH, 8); m->wm_max = xcalloc(m->CH, 8); m->wm_any = xcalloc(m->CH, sizeof(int));
  pthread_barrier_init(&m->bar_start, NULL, (unsigned)P + 1);
  pthread_barrier_init(&m->bar_mid, NULL, (unsigned)P);
  pthread_barrier_init(&m->bar_end, NULL, (unsigned)P + 1);
  m->th = xcalloc(P, sizeof(pthread_t)); m->args = xcalloc(P, sizeof(mt_arg));
  for (int t = 0; t < P; t++) { m->args[t].m = m; m->args[t].tid = t; pthread_create(&m->th[t], NULL, mt_worker, &m->args[t]); }
  return m;
}
void orc_mt_destroy(orc_mt* m) {
  if (!m) return;
  m->stop = 1;
  pthread_barrier_wait(&m->bar_start);
  for (int t = 0; t < m->P; t++) pthread_join(m->th[t], NULL);
  pthread_barrier_destroy(&m->bar_start); pthread_barrier_destroy(&m->bar_mid); pthread_barrier_destroy(&m->bar_end);
  for (int64_t i = 0; i < m->CH * m->P; i++) own_batch_free(&m->subs[i]);
  free(m->subs); free(m->wm_min); free(m->wm_max); free(m->wm_any); free(m->th); free(m->args);
  for (int p = 0; p < m->P; p++) orc_destroy(m->parts[p]);
  free(m->parts); free(m);
}

/* RepartitionExec(Hash): hash the key of every row (create_hashes), build the row-index list of each output
 * partition, then `take` the rows of each partition (all columns are copied once more). */
static void partition_batch(const orc_batch* b, int P, own_batch* subs /* [P] */) {
  int64_t n = b->n;
  uint16_t* part = xrealloc(NULL, (size_t)(n ? n : 1) * 2);
  int64_t* cnt = xcalloc((size_t)P, 8); int64_t* kbytes = xcalloc((size_t)P, 8); int64_t* bbytes = xcalloc((size_t)P, 8);
  for (int64_t i = 0; i < n; i++) {
    int32_t a = b->key_off[i], e = b->key_off[i + 1];
    uint64_t h = bit_get(b->key_valid, i) ? hash_bytes(b->key_bytes + a, e - a) : 0;
    int p = (int)((h >> 17) % (uint64_t)P);
    part[i] = (uint16_t)p; cnt[p]++; kbytes[p] += e - a;
    if (b->barrier_off) bbytes[p] += b->barrier_off[i + 1] - b->barrier_off[i];
  }
  for (int p = 0; p < P; p++) {
    own_batch* o = &subs[p];
    own_batch_reserve(o, cnt[p], kbytes[p], bbytes[p]);
    o->n = 0; o->key_off[0] = 0; o->barrier_off[0] = 0;
    o->has_ts_valid = b->ts_valid != NULL; o->has_val_valid = b->val_valid != NULL; o->has_key_valid = b->key_valid != NULL;
    o->has_occ = b->occurred_at != NULL; o->has_bar = b->barrier_off != NULL;
    if (o->has_ts_valid) memset(o->ts_valid, 0, (size_t)((cnt[p] + 7) / 8 + 1));
    if (o->has_val_valid) memset(o->val_valid, 0, (size_t)((cnt[p] + 7) / 8 + 1));
    if (o->has_key_valid) memset(o->key_valid, 0, (size_t)((cnt[p] + 7) / 8 + 1));
  }
  for (int64_t i = 0; i < n; i++) {
    int32_t a = b->key_off[i], e = b->key_off[i + 1];
    own_batch* o = &subs[part[i]];
    int64_t m = o->n++;
    o->ts[m] = b->ts[i]; if (o->has_ts_valid && bit_get(b->ts_valid, i)) bit_set(o->ts_valid, m);
    o->val[m] = b->val[i]; if (o->has_val_valid && bit_get(b->val_valid, i)) bit_set(o->val_valid, m);
    int32_t ko = o->key_off[m]; memcpy(o->key_bytes + ko, b->key_bytes + a, (size_t)(e - a)); o->key_off[m + 1] = ko + (e - a);
    if (o->has_key_valid && bit_get(b->key_valid, i)) bit_set(o->key_valid, m);
    if (o->has_occ) o->occurred_at[m] = b->occurred_at[i];
    if (o->has_bar) { int32_t c = b->barrier_off[i], d = b->barrier_off[i + 1]; int32_t bo = o->barrier_off[m]; memcpy(o->barrier_bytes + bo, b->barrier_bytes + c, (size_t)(d - c)); o->barrier_off[m + 1] = bo + (d - c); }
  }
  free(part); free(cnt); free(kbytes); free(bbytes);
}

static void* mt_worker(void* vp) {
  mt_arg* a = (mt_arg*)vp; orc_mt* m = a->m; int P = m->P;
  for (;;) {
    pthread_barrier_wait(&m->bar_start);
    if (m->stop) return NULL;
    /* phase 1: threads split the chunk's batches and hash-partition them */
    for (int64_t i = m->c0 + a->tid; i < m->c1; i += P) {
      const orc_batch* b = &m->batches[i];
      m->wm_any[i - m->c0] = batch_watermark(b, &m->wm_min[i - m->c0], &m->wm_max[i - m->c0]);
      partition_batch(b, P, m->subs + (i - m->c0) * P);
    }
    pthread_barrier_wait(&m->bar_mid);
    /* phase 2: thread p runs partition p's stream over its sub-batches in batch order */
    orc_window* w = m->parts[a->tid];
    for (int64_t i = m->c0; i < m->c1 && !a->err; i++) {
      if (m->batches[i].n == 0) { w->seq++; continue; }
      if (!m->wm_any[i - m->c0]) { a->err = -1; break; }
      orc_batch v = own_as_view(&m->subs[(i - m->c0) * P + a->tid]);
      int64_t r = stream_push(w, &v, 1, m->wm_min[i - m->c0], m->wm_max[i - m->c0], v.n > 0);
      w->seq++;
      if (r < 0) { a->err = (int)r; break; }
      a->emitted += r;
    }
    pthread_barrier_wait(&m->bar_end);
  }
}

int64_t orc_mt_push_many(orc_mt* m, const orc_batch* batches, int64_t nb) {
  int P = m->P; int64_t total = 0; int err = 0;
  for (int t = 0; t < P; t++) { m->args[t].emitted = 0; m->args[t].err = 0; }
  m->batches = batches;
  for (int64_t c0 = 0; c0 < nb && !err; c0 += m->CH) {
    m->c0 = c0; m->c1 = c0 + m->CH < nb ? c0 + m->CH : nb;
    pthread_barrier_wait(&m->bar_start);
    pthread_barrier_wait(&m->bar_end);
    for (int t = 0; t < P; t++) if (m->args[t].err) err = m->args[t].err;
  }
  for (int t = 0; t < P; t++) total += m->args[t].emitted;
  return err ? err : total;
}
int64_t orc_mt_num_results(const orc_mt* m) { int64_t n = 0; for (int p = 0; p < m->P; p++) n += m->parts[p]->res.n; return n; }
void orc_mt_get_results(orc_mt* m, int partition, orc_result* out) { orc_get_results(m->parts[partition], out); }
void orc_mt_clear_results(orc_mt* m) { for (int p = 0; p < m->P; p++) orc_clear_results(m->parts[p]); }

/* ------------------------------------------------------------------------------------------ */
/* synthetic sensor stream (SURVEY.md §8d; emit_measurements.rs:30-33,45)                      */

static inline uint64_t splitmix64(uint64_t x) {
  x += 0x9E3779B97F4A7C15ull;
  uint64_t z = x;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}

int64_t orc_synth_fill(int64_t row0, int64_t n, uint64_t seed, int64_t groups, int64_t rows_per_ms, int64_t t0_ms,
                       int32_t uuid_keys, int64_t key_mul, int64_t key_add, int64_t* ts, double* val, int32_t* key_off, uint8_t* key_bytes) {
  static const char hex[] = "0123456789abcdef";
  int32_t o = 0; key_off[0] = 0;
  for (int64_t k = 0; k < n; k++) {
    uint64_t i = (uint64_t)(row0 + k);
    uint64_t r = splitmix64(seed ^ i), r2 = splitmix64(r);
    uint64_t key_id = ((r >> 11) % (uint64_t)groups) * (uint64_t)key_mul + (uint64_t)key_add;
    ts[k] = t0_ms + (int64_t)(i / (uint64_t)rows_per_ms);
    val[k] = ((double)(r2 >> 11) * 0x1.0p-53) * 115.0;
    uint8_t* p = key_bytes + o;
    if (uuid_keys) {
      uint64_t h1 = splitmix64(key_id), h2 = splitmix64(h1);
      int q = 0;
      for (int d = 0; d < 32; d++) {
        uint64_t src = d < 16 ? h1 : h2; int sh = 60 - 4 * (d & 15);
        if (d == 8 || d == 12 || d == 16 || d == 20) p[q++] = '-';
        p[q++] = (uint8_t)hex[(src >> sh) & 15];
      }
      o += 36;
    } else {
      memcpy(p, "sensor_", 7);
      char tmp[24]; int nd = 0; uint64_t v = key_id;
      do { tmp[nd++] = (char)('0' + v % 10); v /= 10; } while (v);
      for (int d = 0; d < nd; d++) p[7 + d] = (uint8_t)tmp[nd - 1 - d];
      o += 7 + nd;
    }
    key_off[k + 1] = o;
  }
  return o;
}

/* ------------------------------------------------------------------------------------------ */
/* Input-contract producer (SURVEY.md §8 f1): canonical event time from a raw column.            */
/* Restates array_to_timestamp_array (crates/core/src/physical_plan/utils/time.rs:59-94):        */
/*   Int64Millis   values as they are (the validity bitmap is not consulted)                     */
/*   Int64Seconds  ts * 1000                                                                     */
/*   StringIso8601 chrono 0.4 NaiveDateTime::parse_from_str(s, fmt).unwrap().and_utc()           */
/*                 .timestamp_millis()  (chrono is a crates.io dependency, not under              */
/*                 /root/reference: published strftime semantics restated for the specifiers      */
/*                 %Y %m %d %H %M %S %f %.f %3f %6f %9f %.3f %.6f %.9f %% and literals)           */
/* Returns 0, or the 1-based index of the first row that does not parse (the reference panics).   */
static int ts_digits_c(const uint8_t* s, int* i, int n, int min_d, int max_d, long long* out) {
  int d = 0; long long v = 0;
  while (d < max_d && *i < n && s[*i] >= '0' && s[*i] <= '9') { v = v * 10 + (s[*i] - '0'); (*i)++; d++; }
  *out = v;
  return d >= min_d;
}
static int ts_parse_c(const uint8_t* s, int n, const char* fmt, long long* out_ms) {
  long long Y = 1970, mo = 1, D = 1, H = 0, Mi = 0, S = 0, nanos = 0, v;
  int i = 0;
  for (const char* f = fmt; *f; f++) {
    char c = *f;
    if (c == ' ' || c == '\t' || c == '\n') { while (i < n && (s[i] == ' ' || s[i] == '\t' || s[i] == '\n')) i++; continue; }
    if (c != '%') { if (i >= n || s[i] != (uint8_t)c) return 0; i++; continue; }
    char sp = *++f; int dot = 0, fixed = 0;
    if (sp == '.') { dot = 1; sp = *++f; }
    if (sp == '3' || sp == '6' || sp == '9') { fixed = sp - '0'; sp = *++f; }
    switch (sp) {
      case 'Y': { int neg = 0; if (i < n && (s[i] == '-' || s[i] == '+')) { neg = s[i] == '-'; i++; } int sg = neg || (i > 0 && s[i - 1] == '+'); if (!ts_digits_c(s, &i, n, 1, sg ? 6 : 4, &v)) return 0; Y = neg ? -v : v; break; }   /* chrono: more than 4 year digits need a sign */
      case 'm': if (!ts_digits_c(s, &i, n, 1, 2, &v) || v < 1 || v > 12) return 0; mo = v; break;
      case 'd': if (!ts_digits_c(s, &i, n, 1, 2, &v) || v < 1 || v > 31) return 0; D = v; break;
      case 'H': if (!ts_digits_c(s, &i, n, 1, 2, &v) || v > 23) return 0; H = v; break;
      case 'M': if (!ts_digits_c(s, &i, n, 1, 2, &v) || v > 59) return 0; Mi = v; break;
      case 'S': if (!ts_digits_c(s, &i, n, 1, 2, &v) || v > 60) return 0; S = v; break;
      case 'f':
        if (dot) {
          if (i < n && s[i] == '.') {
            i++; int d0 = i;
            if (!ts_digits_c(s, &i, n, fixed ? fixed : 1, fixed ? fixed : 9, &v)) return 0;
            for (int k = i - d0; k < 9; k++) v *= 10;
            while (!fixed && i < n && s[i] >= '0' && s[i] <= '9') i++;
            nanos = v;
          } else if (fixed) return 0;
        } else if (fixed) {
          if (!ts_digits_c(s, &i, n, fixed, fixed, &v)) return 0;
          for (int k = fixed; k < 9; k++) v *= 10;
          nanos = v;
        } else { if (!ts_digits_c(s, &i, n, 1, 9, &v)) return 0; nanos = v; }
        break;
      case '%': if (i >= n || s[i] != '%') return 0; i++; break;
      default: return 0;
    }
  }
  if (i != n) return 0;
  {
    int leap = (Y % 4 == 0 && Y % 100 != 0) || Y % 400 == 0;
    int mdays[12] = {31, leap ? 29 : 28, 31, 30, 31, 30, 31, 31, 30, 31, 30, 31};
    if (D > mdays[mo - 1]) return 0;
  }
  long long y = mo <= 2 ? Y - 1 : Y;
  long long era = (y >= 0 ? y : y - 399) / 400, yoe = y - era * 400;
  long long doy = (153 * (mo + (mo > 2 ? -3 : 9)) + 2) / 5 + D - 1;
  long long doe = yoe * 365 + yoe / 4 - yoe / 100 + doy;
  long long days = era * 146097 + doe - 719468;
  long long secs = days * 86400 + H * 3600 + Mi * 60 + (S == 60 ? 59 : S);
  if (S == 60) nanos += 1000000000ll;
  *out_ms = secs * 1000 + nanos / 1000000;
  return 1;
}
int64_t orc_ts_convert(int32_t unit, int64_t n, const int64_t* ints, const int32_t* off, const uint8_t* bytes, const char* fmt, int64_t* out) {
  for (int64_t i = 0; i < n; i++) {
    if (unit == 1) out[i] = ints[i];
    else if (unit == 2) out[i] = ints[i] * 1000;
    else {
      long long ms = 0;
      if (!ts_parse_c(bytes + off[i], off[i + 1] - off[i], fmt, &ms)) return i + 1;
      out[i] = ms;
    }
  }
  return 0;
}

/* ------------------------------------------------------------------------------------------ */
/* Ungrouped windows: `.window([], aggs, len, slide)` (SURVEY.md §8 f2).                          */
/* planner/streaming_window.rs:133-153 builds StreamingWindowExec(Partial) -> StreamingWindowExec */
/* (Final); one partition of that chain is restated here:                                        */
/*   WindowAggStream::poll_next_inner   streaming_window.rs:791-828  (Partial: per-batch windows,  */
/*                                       PartialWindowAggFrame::push = two filters + aggregate_batch)*/
/*   FullWindowAggStream::poll_next_inner :934-1032 (Final: frame keyed by the MAX window start of  */
/*                                       the incoming batch, seen_windows late drop, finalize when  */
/*                                       watermark > window end, watermark = max window START seen) */
/* Row accumulators of DataFusion 42 (not the grouped ones): CountAccumulator; Min/MaxAccumulator   */
/* = arrow compute::min/max + ScalarValue total_cmp (IEEE totalOrder); AvgAccumulator state         */
/* [count u64, sum f64], merged by addition in Final, evaluated as sum / count.                     */
typedef struct { int64_t start, end; uint64_t cnt; double sum; int has; double mn, mx; int used; } uframe_t;
struct orc_uwindow {
  orc_config cfg; int has_wm; int64_t wm;
  uframe_t* pf; int64_t n_pf, cap_pf;          /* Partial frames, ascending start */
  uframe_t* ff; int64_t n_ff, cap_ff;          /* Final frames (cached_frames), ascending start */
  int64_t* seen; int64_t n_seen, cap_seen;     /* seen_windows */
  int has_fwm; int64_t fwm;                    /* Final watermark (a window START) */
  results_t res; int64_t seq; char err[160];
};
static uframe_t* uf_find_or_insert(uframe_t** arr, int64_t* n, int64_t* cap, int64_t start, int64_t end, int* created) {
  int64_t lo = 0, hi = *n;
  while (lo < hi) { int64_t mid = (lo + hi) / 2; if ((*arr)[mid].start < start) lo = mid + 1; else hi = mid; }
  if (created) *created = 0;
  if (lo < *n && (*arr)[lo].start == start) return &(*arr)[lo];
  if (*n + 1 > *cap) { *cap = *cap ? *cap * 2 : 16; *arr = xrealloc(*arr, (size_t)*cap * sizeof(uframe_t)); }
  memmove(*arr + lo + 1, *arr + lo, (size_t)(*n - lo) * sizeof(uframe_t));
  uframe_t f; memset(&f, 0, sizeof f); f.start = start; f.end = end;
  (*arr)[lo] = f; (*n)++;
  if (created) *created = 1;
  return &(*arr)[lo];
}
orc_uwindow* orc_u_create(const orc_config* cfg) {
  orc_uwindow* w = calloc(1, sizeof *w);
  w->cfg = *cfg;
  return w;
}
void orc_u_destroy(orc_uwindow* w) { if (!w) return; free(w->pf); free(w->ff); free(w->seen); results_free(&w->res); free(w); }
const char* orc_u_last_error(const orc_uwindow* w) { return w->err; }
void orc_u_clear_results(orc_uwindow* w) { w->res.n = 0; w->res.bytes = 0; }
void orc_u_get_results(orc_uwindow* w, orc_result* o) {
  static const int32_t zero_off[1] = {0};
  o->n = w->res.n; o->key_off = w->res.key_off ? w->res.key_off : zero_off; o->key_bytes = w->res.key_bytes;
  o->key_isnull = w->res.key_isnull; o->count = w->res.count; o->min = w->res.mn; o->max = w->res.mx; o->avg = w->res.avg;
  o->agg_isnull = w->res.agg_isnull; o->window_start_ms = w->res.ws; o->window_end_ms = w->res.we; o->emit_seq = w->res.seq;
  o->sum = w->res.sum;
}
/* PartialWindowAggFrame::push: rows with start <= ts < end; accumulators updated with the filtered batch */
static void uframe_push(uframe_t* f, const orc_batch* b) {
  for (int64_t i = 0; i < b->n; i++) {
    if (!bit_get(b->ts_valid, i)) continue;
    int64_t t = b->ts[i];
    if (t < f->start || t >= f->end) continue;
    if (!bit_get(b->val_valid, i)) continue;
    double v = b->val[i];
    f->cnt++; f->sum += v;
    if (!f->has) { f->mn = f->mx = v; f->has = 1; }
    else { if (total_cmp(v, f->mn) < 0) f->mn = v; if (total_cmp(v, f->mx) > 0) f->mx = v; }
  }
}
int64_t orc_u_push(orc_uwindow* w, const orc_batch* b) {
  int64_t emitted = 0;
  if (b->n > 0) {
    int64_t L = w->cfg.window_ms, S = w->cfg.slide_ms, mn, mx;
    if (!batch_watermark(b, &mn, &mx)) { snprintf(w->err, sizeof w->err, "all-null canonical_timestamp"); return -1; }
    if (L / 1000 == 0) { snprintf(w->err, sizeof w->err, "window length < 1 s"); return -2; }
    if (mn < 0 || (S > 0 && mn - L < 0)) { snprintf(w->err, sizeof w->err, "timestamp before epoch(+window)"); return -3; }
    /* ---- Partial: get_windows_for_watermark, ensure frames, push */
    if (S > 0) {
      for (int64_t cur = snap_to_window_start(mn - L, L); cur <= mx; cur += S) {
        int64_t end = cur + L;
        if (mn > end || mx < cur) continue;
        uframe_push(uf_find_or_insert(&w->pf, &w->n_pf, &w->cap_pf, cur, end, NULL), b);
      }
    } else {
      for (int64_t cur = snap_to_window_start(mn, L); cur <= mx; cur += L)
        uframe_push(uf_find_or_insert(&w->pf, &w->n_pf, &w->cap_pf, cur, cur + L, NULL), b);
    }
    if (!w->has_wm || w->wm <= mn) { w->wm = mn; w->has_wm = 1; }
    /* trigger_windows: ONE batch with a row per closed frame, ascending start */
    int64_t keep = 0, n_closed = 0;
    uframe_t* closed = NULL;
    for (int64_t i = 0; i < w->n_pf; i++) {
      if (w->wm >= w->pf[i].end) { closed = xrealloc(closed, (size_t)(n_closed + 1) * sizeof(uframe_t)); closed[n_closed++] = w->pf[i]; }
      else w->pf[keep++] = w->pf[i];
    }
    w->n_pf = keep;
    /* ---- Final: the partial batch (if it has rows) */
    if (n_closed > 0) {
      int64_t start = closed[0].start, end = closed[0].end;
      for (int64_t i = 1; i < n_closed; i++) { if (closed[i].start > start) start = closed[i].start; if (closed[i].end > end) end = closed[i].end; }
      int was_seen = 0, cached = 0;
      for (int64_t i = 0; i < w->n_seen; i++) if (w->seen[i] == start) was_seen = 1;
      for (int64_t i = 0; i < w->n_ff; i++) if (w->ff[i].start == start) cached = 1;
      if (!(was_seen && !cached)) {                     /* else: late data for a finalized window, dropped */
        uframe_t* f = uf_find_or_insert(&w->ff, &w->n_ff, &w->cap_ff, start, end, NULL);
        if (!was_seen) { if (w->n_seen + 1 > w->cap_seen) { w->cap_seen = w->cap_seen ? w->cap_seen * 2 : 64; w->seen = xrealloc(w->seen, (size_t)w->cap_seen * sizeof(int64_t)); } w->seen[w->n_seen++] = start; }
        for (int64_t i = 0; i < n_closed; i++) {          /* merge_batch over EVERY row of the batch (the reference assumes one row) */
          f->cnt += closed[i].cnt;
          if (closed[i].has) {
            f->sum += closed[i].sum;
            if (!f->has) { f->mn = closed[i].mn; f->mx = closed[i].mx; f->has = 1; }
            else { if (total_cmp(closed[i].mn, f->mn) < 0) f->mn = closed[i].mn; if (total_cmp(closed[i].mx, f->mx) > 0) f->mx = closed[i].mx; }
          }
        }
        if (!w->has_fwm || start > w->fwm) { w->fwm = start; w->has_fwm = 1; }
        /* finalize_windows: watermark > window_end_time */
        int64_t k2 = 0;
        for (int64_t i = 0; i < w->n_ff; i++) {
          uframe_t* g = &w->ff[i];
          if (w->fwm > g->end) {
            int isnull = !g->has;
            results_push(&w->res, NULL, 0, 1, (int64_t)g->cnt, isnull ? 0.0 : g->mn, isnull ? 0.0 : g->mx, isnull ? 0.0 : g->sum / (double)g->cnt, isnull ? 0.0 : g->sum, isnull, g->start, g->end, w->seq);
            emitted++;
          } else w->ff[k2++] = *g;
        }
        w->n_ff = k2;
      }
    }
    free(closed);
  }
  w->seq++;
  return emitted;
}
