/*
 * TEST-ONLY.  Every job the C oracle (oracle/dcsim_oracle.c, compiled here unchanged through oracle_jobs.c) creates in
 * one replica, finished or not: its job type, the DC it was routed to, its arrival and xfer_done instants and, when it
 * finished, its start and finish.  The per-run tail-latency tests need the jobs that did not finish (UNFINISHED per type
 * and DC), which the per-job rows of oracle_jobs.c leave out.  The oracle is stepped one event at a time as in
 * oracle_jobs.c.  A job's routed DC is that of its xfer_done event; when the arrival pushed none (the instant lies past
 * the end, or the DC is unreachable) the routing draw is replayed from the RNG state before the arrival (the draws of
 * simulator_paper_multi.py:537-577: the size, then the DC).  Nothing here is part of, linked into, or reachable from the
 * product library.
 */
#include "oracle_jobs.c"

typedef struct {
  uint32_t jid;
  int32_t jtype, dc;
  int32_t finished; /* 1: finished by end_time */
  double arrival, xfer_done, start, finish;
} oracle_tail_row_t;

/* One replica (key `seed`) to the end.  Row jid - 1 for every created job; writes up to `cap` rows; returns the number
 * of created jobs (> cap: the rows are a prefix), -1 on a malformed spec. */
long long oracletail_run(const void* spec_blob, size_t spec_bytes, uint64_t seed, int rng_kind, oracle_tail_row_t* out,
                         uint32_t cap) {
  if (!spec_ok(spec_blob, spec_bytes)) return -1;
  dcsim_spec_t spec;
  memcpy(&spec, spec_blob, sizeof(spec));
  sim_t* s = (sim_t*)calloc(1, sizeof(sim_t));
  sim_init(s, &spec, rng_kind, seed);
  while (!s->done) {
    const int have = s->heap_n > 0;
    const event_t ev = have ? s->heap[0] : (event_t){0};
    const uint64_t fin_before = s->n_fin;
    const rng_t rng_before = s->rng;
    sim_run(s, 1);
    if (!have || s->n_events == 0 || s->now != ev.t) continue; /* the run ended instead */
    if (ev.kind == EV_ARR_INF || ev.kind == EV_ARR_TRN) {
      const uint32_t jid = s->jid_counter;
      if (jid > cap) continue;
      oracle_tail_row_t* r = &out[jid - 1];
      memset(r, 0, sizeof(*r));
      r->jid = jid;
      r->jtype = ev.kind == EV_ARR_INF ? DCSIM_JT_INFERENCE : DCSIM_JT_TRAINING;
      r->arrival = s->now;
      r->xfer_done = INFINITY;
      r->dc = -1;
      r->start = r->finish = NAN;
      for (size_t i = 0; i < s->heap_n; ++i)
        if (s->heap[i].kind == EV_XFER && s->heap[i].jid == jid) { r->xfer_done = s->heap[i].t; r->dc = s->heap[i].dc; }
      if (r->dc < 0) { /* no xfer_done pushed: replay the draws of the arrival */
        const rng_t rng_after = s->rng;
        s->rng = rng_before;
        (void)sample_job_size(s, r->jtype);
        if (spec.algo == DCSIM_ALGO_ECO_ROUTE) {
          double best = 0.0;
          for (int d = 0; d < spec.n_dc; ++d) {
            const double score = score_dc_for_job(s, d, &s->jobs[jid]);
            if (d == 0 || score < best) { best = score; r->dc = d; }
          }
        } else {
          r->dc = rng_randbelow(&s->rng, spec.n_dc);
        }
        s->rng = rng_after;
      }
    } else if (ev.kind == EV_FINISH && s->n_fin > fin_before && ev.jid <= cap) {
      const job_t* j = &s->jobs[ev.jid];
      oracle_tail_row_t* r = &out[ev.jid - 1];
      r->finished = 1; r->start = j->start_time; r->finish = j->finish_time;
    }
  }
  const long long n = s->jid_counter;
  sim_free(s);
  free(s);
  return n;
}
