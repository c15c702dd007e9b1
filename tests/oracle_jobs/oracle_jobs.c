/*
 * TEST-ONLY.  Per-job instants of the C oracle (oracle/dcsim_oracle.c, compiled here unchanged into its own library):
 * for every job that finished, its arrival instant (simulator_paper_multi.py:539-540), its xfer_done instant
 * (SIM:580-588), its start and finish, and whether it started in the handler of its own xfer_done event (SIM:603-676)
 * rather than in a dequeue loop (SIM:840-927).  The oracle is stepped one event at a time; before each step the event
 * about to fire is the heap's top, and after it the oracle's own state shows what the event did:
 *   - an arrival took job id jid_counter at `now`, and pushed that job's xfer_done event (found in the heap; absent when
 *     the instant lies past the end);
 *   - an xfer_done event started its job when the job is running afterwards;
 *   - a job_finish finished its job when the finish count went up.
 * Rows come out in finish order.  Nothing here is part of, linked into, or reachable from the product library.
 */
#include "../../oracle/dcsim_oracle.c"

typedef struct {
  uint32_t jid;
  int32_t dc, jtype;
  int32_t at_xfer; /* 1: started by its own xfer_done event */
  double arrival, xfer_done, start, finish;
} oracle_job_row_t;

void oraclejobs_set_test_time_quantum(double q) { g_test_time_quantum = q; }

/* One replica (key `seed`) to the end.  Writes up to `cap` rows; returns the number of finished jobs (> cap: the rows
 * are a prefix), -1 on a malformed spec. */
long long oraclejobs_run(const void* spec_blob, size_t spec_bytes, uint64_t seed, int rng_kind, oracle_job_row_t* out,
                         uint32_t cap) {
  if (!spec_ok(spec_blob, spec_bytes)) return -1;
  dcsim_spec_t spec;
  memcpy(&spec, spec_blob, sizeof(spec));
  sim_t* s = (sim_t*)calloc(1, sizeof(sim_t));
  sim_init(s, &spec, rng_kind, seed);
  size_t n_cap = 1024;
  double* arr = (double*)malloc(n_cap * sizeof(double));
  double* tx = (double*)malloc(n_cap * sizeof(double));
  int32_t* at_xfer = (int32_t*)calloc(n_cap, sizeof(int32_t));
  long long n_rows = 0;
  while (!s->done) {
    const int have = s->heap_n > 0;
    const event_t ev = have ? s->heap[0] : (event_t){0};
    const uint64_t fin_before = s->n_fin;
    sim_run(s, 1);
    if (!have || s->n_events == 0 || s->now != ev.t) continue; /* the run ended instead */
    if (ev.kind == EV_ARR_INF || ev.kind == EV_ARR_TRN) {
      const uint32_t jid = s->jid_counter;
      if (jid >= n_cap) {
        const size_t nc = 2 * (size_t)jid;
        arr = (double*)realloc(arr, nc * sizeof(double));
        tx = (double*)realloc(tx, nc * sizeof(double));
        at_xfer = (int32_t*)realloc(at_xfer, nc * sizeof(int32_t));
        memset(at_xfer + n_cap, 0, (nc - n_cap) * sizeof(int32_t));
        n_cap = nc;
      }
      arr[jid] = s->now;
      tx[jid] = INFINITY;
      for (size_t i = 0; i < s->heap_n; ++i)
        if (s->heap[i].kind == EV_XFER && s->heap[i].jid == jid) tx[jid] = s->heap[i].t;
    } else if (ev.kind == EV_XFER) {
      at_xfer[ev.jid] = s->jobs[ev.jid].running;
    } else if (ev.kind == EV_FINISH && s->n_fin > fin_before) {
      const job_t* j = &s->jobs[ev.jid];
      if (n_rows < (long long)cap) {
        oracle_job_row_t* r = &out[n_rows];
        r->jid = ev.jid; r->dc = ev.dc; r->jtype = j->jtype; r->at_xfer = at_xfer[ev.jid];
        r->arrival = arr[ev.jid]; r->xfer_done = tx[ev.jid]; r->start = j->start_time; r->finish = j->finish_time;
      }
      ++n_rows;
    }
  }
  free(arr); free(tx); free(at_xfer);
  sim_free(s);
  free(s);
  return n_rows;
}
