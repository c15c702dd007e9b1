/*
 * TEST-ONLY.  The arrivals of one replica as the C oracle (oracle/dcsim_oracle.c, compiled unchanged into
 * oracle_probes.c) processes them: the independent reference of the arrival pre-pass (dcsim_generate_arrivals) and of what the
 * list merge derives from it.  The oracle is stepped one event at a time; before each step the event about to fire is
 * the heap's top, and every event pushed during the step has a seq at or above the counter's value before it.  For each
 * arrival event (SIM:537-592):
 *   - its instant, stream (2 * ingress + job type), job size and chosen DC (the DC is read off the xfer_done push, so it
 *     is -1 when that push was not schedulable);
 *   - the instant of the xfer_done it pushed, +inf when none was pushed (+inf or later than end_time + 1e-9, SIM:161);
 *   - pred: the arrival whose processing pushed this one, 0xffffffff for the constructor's pushes (SIM:154-156);
 *   - whether it pushed its stream's next arrival.
 * Per replica also the RNG words the whole run consumed and first_mask (bit s: stream s's first arrival was pushed).
 * Nothing here is part of, linked into, or reachable from the product library.
 */

typedef struct {
  double t, size, tx;
  uint32_t stream;
  int32_t dc;
  uint32_t pred, next;
} oracle_arr_row_t;

/* One replica (key `seed`) to the end.  Writes up to `cap` rows; info[0] = first_mask, info[1] = RNG words.  Returns
 * the number of arrivals processed (> cap: the rows are a prefix), -1 on a malformed spec. */
long long oraclelists_run(const void* spec_blob, size_t spec_bytes, uint64_t seed, int rng_kind, oracle_arr_row_t* out,
                          uint32_t cap, uint64_t* info) {
  if (!spec_ok(spec_blob, spec_bytes)) return -1;
  dcsim_spec_t spec;
  memcpy(&spec, spec_blob, sizeof(spec));
  sim_t* s = (sim_t*)calloc(1, sizeof(sim_t));
  sim_init(s, &spec, rng_kind, seed);
  uint32_t first_mask = 0u, pending_pred[2 * DCSIM_MAX_ING];
  for (size_t i = 0; i < s->heap_n; ++i)
    if (s->heap[i].kind == EV_ARR_INF || s->heap[i].kind == EV_ARR_TRN) first_mask |= 1u << (2 * s->heap[i].ing + s->heap[i].kind);
  for (int q = 0; q < 2 * DCSIM_MAX_ING; ++q) pending_pred[q] = 0xffffffffu;
  long long n = 0;
  while (!s->done) {
    const int have = s->heap_n > 0;
    const event_t ev = have ? s->heap[0] : (event_t){0};
    const uint32_t seq_before = s->seq;
    const uint64_t events_before = s->n_events;
    sim_run(s, 1);
    if (!have || s->n_events == events_before) continue; /* the run ended instead */
    if (ev.kind != EV_ARR_INF && ev.kind != EV_ARR_TRN) continue;
    const uint32_t stream = 2u * (uint32_t)ev.ing + (uint32_t)ev.kind;
    oracle_arr_row_t row = {s->now, s->jobs[s->jid_counter].size, INFINITY, stream, -1, pending_pred[stream], 0u};
    for (size_t i = 0; i < s->heap_n; ++i) {
      const event_t* e = &s->heap[i];
      if (e->seq < seq_before) continue;
      if (e->kind == EV_XFER) { row.tx = e->t; row.dc = e->dc; }
      else if (e->kind == EV_ARR_INF || e->kind == EV_ARR_TRN) { row.next = 1u; pending_pred[stream] = (uint32_t)n; }
    }
    if (n < (long long)cap) out[n] = row;
    ++n;
  }
  info[0] = first_mask;
  info[1] = s->rng.words;
  sim_free(s);
  free(s);
  return n;
}
