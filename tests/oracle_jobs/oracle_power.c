/*
 * TEST-ONLY.  The power profile on the C oracle (oracle/dcsim_oracle.c, compiled unchanged into oracle_probes.c), for
 * tests/test_recorder_corpus*.py: oraclepower_profile steps the oracle one event at a time, records the power every
 * energy accrual is about to integrate, and applies the definition of include/dcsim_b200.h (DCSIM_STAT_POWER_PROFILE)
 * to those intervals.  tests/golden/make_golden_power.py does the same from the reference; this is its C twin, so a
 * random scenario has a bit-exact reference too.  Nothing here is part of, linked into, or reachable from the product
 * library.
 */

typedef struct {
  const dcsim_spec_t* sp;
  double* row;           /* [DCSIM_PP_FIELDS + n_dc + DCSIM_PP_BINS] */
  double hi, thr;
  int have_lv, n_lv, any;
  double lv_s, lv_e, lv_p; /* the open level */
  int in_run;
  double run_s;
  double first_a;          /* start of the first accrued interval: the first event's instant */
} pp_acc_t;

/* One level, in level order: bin, peak, threshold fields (make_golden_power.expected). */
static void pp_close_level(pp_acc_t* a) {
  double* f = a->row;
  const double s = a->lv_s, e = a->lv_e, p = a->lv_p, L = e - s;
  const double k = floor(p / (a->hi / DCSIM_PP_BINS));
  const int b = k < 0.0 ? 0 : (k > DCSIM_PP_BINS - 1 ? DCSIM_PP_BINS - 1 : (int)k);
  if (!(0.0 <= p && p <= a->hi)) f[DCSIM_PP_OUT_OF_RANGE] += 1.0;
  f[DCSIM_PP_FIELDS + a->sp->n_dc + b] += L;
  if (a->n_lv == 0 || p > f[DCSIM_PP_PEAK_W]) { f[DCSIM_PP_PEAK_W] = p; f[DCSIM_PP_T_PEAK_S] = s; }
  if (p > a->thr) {
    f[DCSIM_PP_OVER_S] += L;
    f[DCSIM_PP_OVER_J] += (p - a->thr) * L;
    if (!a->in_run) { a->in_run = 1; a->run_s = s; f[DCSIM_PP_EXCURSIONS] += 1.0; }
  } else if (a->in_run) {
    if (s - a->run_s > f[DCSIM_PP_LONGEST_OVER_S]) f[DCSIM_PP_LONGEST_OVER_S] = s - a->run_s;
    a->in_run = 0;
  }
  ++a->n_lv;
}

/* One accrual (a, b] of every DC at powers ps[d]: the cluster power sums them in DC order from 0.0; bitwise-equal
 * consecutive powers extend the open level; zero-length intervals are ignored. */
static void pp_interval(pp_acc_t* a, double ta, double tb, const double* ps) {
  if (!a->any) { a->any = 1; a->first_a = ta; }
  if (!(tb > ta)) return;
  const int nd = a->sp->n_dc;
  double p = 0.0;
  for (int d = 0; d < nd; ++d) p += ps[d];
  double* dc_peak = a->row + DCSIM_PP_FIELDS;
  for (int d = 0; d < nd; ++d)
    if (!a->have_lv || ps[d] > dc_peak[d]) dc_peak[d] = ps[d];
  if (a->have_lv && memcmp(&a->lv_p, &p, sizeof(double)) == 0) { a->lv_e = tb; return; }
  if (a->have_lv) pp_close_level(a);
  a->have_lv = 1; a->lv_s = ta; a->lv_e = tb; a->lv_p = p;
}

/* One replica to the end.  Before each step whose event is at or before end_time, every DC's interval
 * (last_energy_time, t] at estimate_dc_power (what accrue_energy is about to integrate; nothing while last_energy_time
 * is 0.0, its first-touch rule); before the step that ends the run, the tail (last_energy_time, end_time] at
 * instantaneous_power_w.  `row` (zeroed by the caller) gets the power-profile column of include/dcsim_b200.h over
 * threshold `thr` (+inf: none) and histogram range `hi` (the library's dcsim_power_profile_range).  Returns the events
 * processed, -1 on a malformed spec, -2 when the DCs' accrual instants ever disagree (the rule above assumes one). */
long long oraclepower_profile(const void* spec_blob, size_t spec_bytes, uint64_t seed, int rng_kind, double* row, double thr,
                              double hi) {
  if (!spec_ok(spec_blob, spec_bytes)) return -1;
  dcsim_spec_t spec;
  memcpy(&spec, spec_blob, sizeof(spec));
  sim_t* s = (sim_t*)calloc(1, sizeof(sim_t));
  sim_init(s, &spec, rng_kind, seed);
  pp_acc_t a;
  memset(&a, 0, sizeof(a));
  a.sp = &spec; a.row = row; a.hi = hi; a.thr = thr;
  double ps[DCSIM_MAX_DC];
  int n_bad = 0;
  while (!s->done) {
    const int have = s->heap_n > 0;
    const double t = have ? s->heap[0].t : INFINITY;
    const int tail = !(have && t <= spec.end_time);
    const double b = tail ? spec.end_time : t;
    for (int d = 1; d < spec.n_dc; ++d)
      if (s->dc[d].last_energy_time != s->dc[0].last_energy_time) { n_bad = 1; break; } /* one accrual per event */
    if (s->dc[0].last_energy_time != 0.0) {
      for (int d = 0; d < spec.n_dc; ++d) ps[d] = tail ? instantaneous_power_w(s, d) : estimate_dc_power(s, d);
      pp_interval(&a, s->dc[0].last_energy_time, b, ps);
    }
    sim_run(s, 1);
  }
  if (a.have_lv) pp_close_level(&a);
  if (a.in_run && a.lv_e - a.run_s > row[DCSIM_PP_LONGEST_OVER_S]) row[DCSIM_PP_LONGEST_OVER_S] = a.lv_e - a.run_s;
  if (a.any) row[DCSIM_PP_PROFILE_S] = spec.end_time - a.first_a;
  const long long n = n_bad ? -2 : (long long)s->n_events;
  sim_free(s);
  free(s);
  return n;
}
