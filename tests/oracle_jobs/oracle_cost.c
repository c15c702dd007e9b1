/*
 * TEST-ONLY.  The energy cost on the C oracle (oracle/dcsim_oracle.c, compiled unchanged into oracle_probes.c), for
 * tests/test_energy_cost*.py: oraclecost_run steps the oracle one event at a time, records the power every energy accrual
 * of every DC is about to integrate, and applies the definition of include/dcsim_b200.h (DCSIM_STAT_ENERGY_COST) to
 * those intervals.  tests/golden/make_golden_cost.py does the same from the reference; this is its C twin, so a random
 * scenario has a bit-exact reference too.  Nothing here is part of, linked into, or reachable from the product library.
 */

typedef struct {
  int have_lv;
  double lv_s, lv_e, lv_p; /* DC d's open level */
} cost_dc_t;

/* Level [s, e] of DC d at power p: cut at every hour boundary 3600 k strictly inside it; each piece [a, b] adds
 * p * (b - a) to hour (k mod 24) of its window k, 3600 k <= a < 3600 (k + 1). */
static void cost_close_level(double* row, int d, double s, double e, double p) {
  double k = floor(s / 3600.0);
  if (3600.0 * k > s) k -= 1.0;
  else if (3600.0 * (k + 1.0) <= s) k += 1.0;
  double a = s;
  for (;;) {
    const double b = 3600.0 * (k + 1.0);
    const int cut = b < e;
    row[DCSIM_COST_HOUR_J(0, d, (int)fmod(k, (double)DCSIM_HOURS))] += p * ((cut ? b : e) - a);
    if (!cut) break;
    a = b;
    k += 1.0;
  }
}

/* One accrual (ta, tb] of DC d at power p: bitwise-equal consecutive powers extend the open level; zero-length
 * intervals are ignored. */
static void cost_interval(double* row, cost_dc_t* c, int d, double ta, double tb, double p) {
  if (!(tb > ta)) return;
  if (c->have_lv && memcmp(&c->lv_p, &p, sizeof(double)) == 0) { c->lv_e = tb; return; }
  if (c->have_lv) cost_close_level(row, d, c->lv_s, c->lv_e, c->lv_p);
  c->have_lv = 1; c->lv_s = ta; c->lv_e = tb; c->lv_p = p;
}

/* One replica to the end.  Before each step whose event is at or before end_time, every DC's interval
 * (last_energy_time, t] at estimate_dc_power (nothing while last_energy_time is 0.0, its first-touch rule); before the
 * step that ends the run, the tail (last_energy_time, end_time] at instantaneous_power_w.  `row` (zeroed by the caller,
 * DCSIM_COST_COLS(n_dc) doubles) gets the energy-cost column of include/dcsim_b200.h; it stays 0 when nothing accrued.
 * Returns the events processed, -1 on a malformed spec. */
long long oraclecost_run(const void* spec_blob, size_t spec_bytes, uint64_t seed, int rng_kind, double* row) {
  if (!spec_ok(spec_blob, spec_bytes)) return -1;
  dcsim_spec_t spec;
  memcpy(&spec, spec_blob, sizeof(spec));
  const int nd = spec.n_dc;
  sim_t* s = (sim_t*)calloc(1, sizeof(sim_t));
  sim_init(s, &spec, rng_kind, seed);
  cost_dc_t c[DCSIM_MAX_DC];
  memset(c, 0, sizeof(c));
  int any = 0;
  while (!s->done) {
    const int have = s->heap_n > 0;
    const double t = have ? s->heap[0].t : INFINITY;
    const int tail = !(have && t <= spec.end_time);
    const double b = tail ? spec.end_time : t;
    for (int d = 0; d < nd; ++d) {
      const double a = s->dc[d].last_energy_time;
      if (a == 0.0) continue;
      any = 1;
      cost_interval(row, &c[d], d, a, b, tail ? instantaneous_power_w(s, d) : estimate_dc_power(s, d));
    }
    sim_run(s, 1);
  }
  if (any) {
    double tot_j = 0.0, tot_usd = 0.0, tot_g = 0.0;
    for (int d = 0; d < nd; ++d) {
      if (c[d].have_lv) cost_close_level(row, d, c[d].lv_s, c[d].lv_e, c[d].lv_p);
      double ej = 0.0, usd = 0.0;
      for (int h = 0; h < DCSIM_HOURS; ++h) {
        const double e = row[DCSIM_COST_HOUR_J(nd, d, h)];
        ej += e;
        usd += (e / 3.6e6) * spec.dc[d].price_kwh[h];
      }
      const double g = (ej / 3.6e6) * spec.dc[d].carbon_intensity;
      row[DCSIM_COST_ENERGY_J(nd, d)] = ej;
      row[DCSIM_COST_USD(nd, d)] = usd;
      row[DCSIM_COST_CARBON_G(nd, d)] = g;
      tot_j += ej; tot_usd += usd; tot_g += g;
    }
    row[DCSIM_COST_TOTAL_J(nd)] = tot_j;
    row[DCSIM_COST_TOTAL_USD(nd)] = tot_usd;
    row[DCSIM_COST_TOTAL_G(nd)] = tot_g;
  }
  const long long n = (long long)s->n_events;
  sim_free(s);
  free(s);
  return n;
}
