/*
 * TEST-ONLY.  Occupancy checkers on the C oracle (oracle/dcsim_oracle.c, compiled here unchanged into its own library),
 * for tests/test_occupancy.py:
 *   - oracleocc_occupancy steps the oracle one event at a time and applies the definition of include/dcsim_b200.h
 *     (dcsim_enable_occupancy) to each DC's queue lengths, running count and busy GPUs as they stand before each step;
 *   - oracleocc_reached lists every job that reached its DC, with its xfer_done, start and finish instants (Little's law).
 * Nothing here is part of, linked into, or reachable from the product library.
 */
#include "../../oracle/dcsim_oracle.c"

void oracleocc_set_test_time_quantum(double q) { g_test_time_quantum = q; }

/* One function's open level (include/dcsim_b200.h, dcsim_enable_occupancy): start (-1: none yet) and value. */
typedef struct { double s, v; } occ_level_t;

/* DC d's function `fn` (0 Qi, 1 Qt, 2 N, 3 Q, 4 B) closes level [s, e] at value v into `row`, laid out as the library's
 * column of one replica: [1 + 8 * n_dc + 2 * 128 * n_dc]. */
static void occ_close(const dcsim_spec_t* sp, double* row, int d, int fn, double s, double e, double v) {
  const int nd = sp->n_dc;
  double* f = row + 1;
  const double len = e - s;
  switch (fn) {
    case 0: f[0 * nd + d] += v * len; if (v > f[3 * nd + d]) f[3 * nd + d] = v; break;
    case 1: f[1 * nd + d] += v * len; if (v > f[4 * nd + d]) f[4 * nd + d] = v; break;
    case 2: f[2 * nd + d] += v * len; break;
    case 3:
      if (v > 0) f[5 * nd + d] += len;
      f[8 * nd + d * 128 + (v < 127 ? (int)v : 127)] += len;
      break;
    default: {
      const int total = sp->dc[d].total_gpus, w = (total + 1 + 127) / 128;
      if ((int)v == total) f[6 * nd + d] += len;
      if ((int)v == 0) f[7 * nd + d] += len;
      f[8 * nd + (nd + d) * 128 + (int)v / w] += len;
    }
  }
}

/* The interval (a, b] of DC d held `vals`: positive length only; a changed value closes the open level at a. */
static void occ_interval(const dcsim_spec_t* sp, double* row, occ_level_t lv[][5], int d, double a, double b, const double* vals) {
  if (!(b > a)) return;
  for (int fn = 0; fn < 5; ++fn) {
    occ_level_t* l = &lv[d][fn];
    if (l->s < 0) { l->s = a; l->v = vals[fn]; }
    else if (l->v != vals[fn]) { occ_close(sp, row, d, fn, l->s, a, l->v); l->s = a; l->v = vals[fn]; }
  }
}

static void occ_values(const sim_t* s, int d, double* vals) {
  const dcstate_t* dc = &s->dc[d];
  vals[0] = (double)fifo_len(&dc->q_inf); vals[1] = (double)fifo_len(&dc->q_trn); vals[2] = (double)dc->n_running;
  vals[3] = vals[0] + vals[1]; vals[4] = (double)dc->busy;
}

/* One replica to the end, stepping the oracle one event at a time and reading every DC's queue lengths, running count
 * and busy GPUs before each step: the interval from the previous event to this one held them.  Then the tail
 * (last event, end_time] with the final state, and every open level closes at end_time.  `row` (zeroed by the caller)
 * gets the occupancy columns of include/dcsim_b200.h.  Returns the events processed, -1 on a malformed spec. */
long long oracleocc_occupancy(const void* spec_blob, size_t spec_bytes, uint64_t seed, int rng_kind, double* row) {
  if (!spec_ok(spec_blob, spec_bytes)) return -1;
  dcsim_spec_t spec;
  memcpy(&spec, spec_blob, sizeof(spec));
  sim_t* s = (sim_t*)calloc(1, sizeof(sim_t));
  sim_init(s, &spec, rng_kind, seed);
  occ_level_t lv[DCSIM_MAX_DC][5];
  for (int d = 0; d < DCSIM_MAX_DC; ++d)
    for (int fn = 0; fn < 5; ++fn) lv[d][fn].s = -1.0;
  double prev = -1.0, t0 = -1.0, vals[5];
  while (!s->done) {
    const int have = s->heap_n > 0;
    const double t = have ? s->heap[0].t : INFINITY;
    if (have && t <= spec.end_time) {
      if (prev >= 0)
        for (int d = 0; d < spec.n_dc; ++d) { occ_values(s, d, vals); occ_interval(&spec, row, lv, d, prev, t, vals); }
      else t0 = t;
      prev = t;
    }
    sim_run(s, 1);
  }
  if (prev >= 0) {
    for (int d = 0; d < spec.n_dc; ++d) {
      occ_values(s, d, vals);
      occ_interval(&spec, row, lv, d, prev, spec.end_time, vals);
      const double end = spec.end_time > prev ? spec.end_time : prev;
      for (int fn = 0; fn < 5; ++fn)
        if (lv[d][fn].s >= 0) occ_close(&spec, row, d, fn, lv[d][fn].s, end, lv[d][fn].v);
    }
    row[0] = spec.end_time - t0;
  }
  const long long n = (long long)s->n_events;
  sim_free(s);
  free(s);
  return n;
}

typedef struct {
  uint32_t jid;
  int32_t dc, jtype;
  double xfer_done, start, finish; /* start / finish: +inf when it did not happen by end_time */
} oracle_reached_row_t;

/* Every job whose xfer_done event was processed (it reached its DC), in xfer_done order, with its start and finish
 * instants (+inf when still queued / running at the end).  Writes up to `cap` rows; returns their number (> cap: a
 * prefix), -1 on a malformed spec. */
long long oracleocc_reached(const void* spec_blob, size_t spec_bytes, uint64_t seed, int rng_kind, oracle_reached_row_t* out,
                             uint32_t cap) {
  if (!spec_ok(spec_blob, spec_bytes)) return -1;
  dcsim_spec_t spec;
  memcpy(&spec, spec_blob, sizeof(spec));
  sim_t* s = (sim_t*)calloc(1, sizeof(sim_t));
  sim_init(s, &spec, rng_kind, seed);
  size_t n_cap = 1024, n = 0;
  uint32_t* jids = (uint32_t*)malloc(n_cap * sizeof(uint32_t));
  double* tx = (double*)malloc(n_cap * sizeof(double));
  double* fin = NULL;
  size_t fin_cap = 0;
  while (!s->done) {
    const int have = s->heap_n > 0;
    const event_t ev = have ? s->heap[0] : (event_t){0};
    const uint64_t fin_before = s->n_fin;
    sim_run(s, 1);
    if (!have || s->n_events == 0 || s->now != ev.t) continue; /* the run ended instead */
    if (ev.kind == EV_XFER) {
      if (n == n_cap) {
        n_cap *= 2;
        jids = (uint32_t*)realloc(jids, n_cap * sizeof(uint32_t));
        tx = (double*)realloc(tx, n_cap * sizeof(double));
      }
      jids[n] = ev.jid; tx[n] = ev.t; ++n;
    } else if (ev.kind == EV_FINISH && s->n_fin > fin_before) {
      if (ev.jid >= fin_cap) {
        const size_t nc = 2 * (size_t)ev.jid + 1024;
        fin = (double*)realloc(fin, nc * sizeof(double));
        for (size_t i = fin_cap; i < nc; ++i) fin[i] = INFINITY;
        fin_cap = nc;
      }
      fin[ev.jid] = ev.t;
    }
  }
  for (size_t i = 0; i < n && i < cap; ++i) {
    const job_t* j = &s->jobs[jids[i]];
    oracle_reached_row_t* r = &out[i];
    r->jid = jids[i]; r->dc = j->dc; r->jtype = j->jtype; r->xfer_done = tx[i];
    r->start = j->start_time != 0.0 ? j->start_time : INFINITY;
    r->finish = jids[i] < fin_cap ? fin[jids[i]] : INFINITY;
  }
  free(jids); free(tx); free(fin);
  sim_free(s);
  free(s);
  return (long long)n;
}
