/*
 * TEST-ONLY.  The single-lane host build of the device core (tests/hostemu/hostemu.cpp, compiled unchanged into this
 * file) with the energy-cost recorder on.  hostemu_run_batch allocates the launch parameters itself and knows nothing of
 * this recorder, so the build arms its output before the call: the parameters' calloc is routed through
 * hostemu_cost_calloc, which sets P->cost and P->cost_work on the one block it allocates while armed.  Everything else
 * (pre-pass, merge, chunked launches, head staging, every other recorder, the library's launch-parameter rules) is
 * hostemu_run_batch's own.  Built twice by build.sh: plain and DCSIM_HOST_UNIFORM_LOOP.  Not part of, linked into, or
 * reachable from the product library.
 */
#include <stdlib.h>
#include <string.h>

static void* hostemu_cost_calloc(size_t n, size_t size);
#define calloc hostemu_cost_calloc
#include "../hostemu/hostemu.cpp"
#undef calloc

namespace {
double* g_cost = NULL;       /* [DCSIM_COST_COLS(n_dc)][n] output of the next run, NULL: disarmed */
double* g_cost_work = NULL;  /* its working rows, [n][n_dc][DCSIM_COSTW_N] */
}

static void* hostemu_cost_calloc(size_t n, size_t size) {
  void* p = calloc(n, size);
  if (p && g_cost && n == 1 && size == sizeof(dcsim_kparams_t)) {
    dcsim_kparams_t* P = (dcsim_kparams_t*)p;
    P->cost = g_cost;
    P->cost_work = g_cost_work;
    g_cost = NULL;
  }
  return p;
}

extern "C" {

/* hostemu_run_batch with the energy-cost recorder writing `cost` ([DCSIM_COST_COLS(n_dc)][n_replicas], zeroed here). */
long long hostemu_cost_run_batch(const void* spec_lists, const void* spec_run, size_t spec_bytes, uint64_t n_replicas,
                                 uint64_t seed0, uint64_t chunk_events, int rng_kind, const hostemu_out_t* o, double* cost) {
  if (!spec_ok(spec_run, spec_bytes) || !cost) return -1;
  const int n_dc = ((const dcsim_spec_t*)spec_run)->n_dc;
  memset(cost, 0, (size_t)DCSIM_COST_COLS(n_dc) * n_replicas * sizeof(double));
  g_cost_work = (double*)calloc(n_replicas * (size_t)n_dc * DCSIM_COSTW_N, sizeof(double));
  g_cost = cost;
  const long long r = hostemu_run_batch(spec_lists, spec_run, spec_bytes, n_replicas, seed0, chunk_events, rng_kind, o);
  g_cost = NULL;
  free(g_cost_work);
  g_cost_work = NULL;
  return r;
}

/* the recorder's hour window of an instant (dcsim_cost_window), and the hour the handlers use (dcsim_current_hour) */
double hostemu_cost_window(double t) { return dcsim_cost_window(t); }
int hostemu_current_hour(double t) { return dcsim_current_hour(t); }

} /* extern "C" */
