/*
 * TEST-ONLY.  Single-lane host build of distributed_cluster_gpus_b200/csrc/dcsim_core.cuh for the rule that lets
 * handles share one arrival pre-pass (dcsim_create_shared): dump the merged {arrival, xfer_done} lists a spec gives,
 * and run the event loop of one spec on the lists drawn under another.  It is not part of, linked into, or reachable
 * from the product library.  Built twice by build.sh: plain, and with DCSIM_HOST_UNIFORM_LOOP (the warp-uniform
 * event-loop skeleton of the lane-group GPU builds).
 */
#define DCSIM_HOST_EMU 1
#include "../../distributed_cluster_gpus_b200/csrc/dcsim_core.cuh"

#include <stdio.h>
#include <stdlib.h>

namespace {

bool spec_ok(const void* blob, size_t bytes) {
  if (!blob || bytes != sizeof(dcsim_spec_t)) return false;
  const dcsim_spec_t* sp = (const dcsim_spec_t*)blob;
  return sp->magic == DCSIM_SPEC_MAGIC && sp->n_dc >= 1 && sp->n_dc <= DCSIM_MAX_DC && sp->n_ing >= 1 && sp->n_ing <= DCSIM_MAX_ING;
}

/* Launch parameters of a batch of `spec` (the library's fill_kparams for the fields the host build uses) with the
 * arrival buffers allocated. */
dcsim_kparams_t* make_params(const void* spec_blob, uint64_t n_replicas, uint64_t seed0, uint64_t chunk_events, int rng_kind) {
  dcsim_kparams_t* P = (dcsim_kparams_t*)calloc(1, sizeof(dcsim_kparams_t));
  memcpy(&P->spec, spec_blob, sizeof(dcsim_spec_t));
  dcsim_make_layout(&P->spec, &P->L, /*job_log=*/0);
  P->cap_arr = (uint32_t)(P->spec.cap_arrivals > 0 ? P->spec.cap_arrivals : 16384);
  P->rec.trace_replica = -1; P->rec.log_replica = -1;
  P->n_replicas = n_replicas; P->seed0 = seed0; P->max_events = chunk_events;
  P->budget32 = (chunk_events == 0ull || chunk_events > 0xfffffffeull) ? 0xffffffffu : (uint32_t)chunk_events;
  P->end_eps = P->spec.end_time + 1e-9;
  for (int i = 0; i < P->spec.n_ing; ++i)
    for (int d = 0; d < P->spec.n_dc; ++d)
      for (int jt = 0; jt < 2; ++jt) {
        const double v = P->spec.transfer_s[i][d][jt];
        if (v == v && v < 1e300 && v > P->max_transfer) P->max_transfer = v;
      }
  const size_t ne = n_replicas * (size_t)P->cap_arr;
  P->arr_t = (double*)calloc(ne, sizeof(double));
  P->arr_raw = (double*)calloc(ne, sizeof(double));
  P->arr_meta = (uint32_t*)calloc(ne, sizeof(uint32_t));
  P->arr_pred = (uint32_t*)calloc(ne, sizeof(uint32_t));
  P->arr_tx = (double*)calloc(ne, sizeof(double));
  P->arr_fin = (uint32_t*)calloc(ne, sizeof(uint32_t));
  P->ml_t = (double*)calloc(2 * ne, sizeof(double));
  P->ml_aux = (double*)calloc(2 * ne, sizeof(double));
  P->ml_meta = (uint32_t*)calloc(2 * ne, sizeof(uint32_t));
  P->arr_hdr = (dcsim_arrhdr_t*)calloc(n_replicas, sizeof(dcsim_arrhdr_t));
  if (rng_kind == 1) P->mt_state = (uint32_t*)calloc(n_replicas * (size_t)DCSIM_MT_N, sizeof(uint32_t));
  return P;
}

void free_params(dcsim_kparams_t* P) {
  free(P->arr_t); free(P->arr_raw); free(P->arr_meta); free(P->arr_pred); free(P->arr_tx); free(P->arr_fin);
  free(P->ml_t); free(P->ml_aux); free(P->ml_meta); free(P->arr_hdr); free(P->mt_state); free(P);
}

/* The pre-pass and the list merge, replica by replica. */
void draw_lists(dcsim_kparams_t* P, int rng_kind) {
  double clocks[2 * DCSIM_MAX_ING];
  uint32_t last[2 * DCSIM_MAX_ING];
  uint32_t ring[DCSIM_TRNG_RING];
  static dcsim_merge_ring_t merge_ring;
  for (uint64_t r = 0; r < P->n_replicas; ++r) {
    if (rng_kind == 1) dcsim_generate_arrivals<true>(P, r, clocks, last, ring, 1); else dcsim_generate_arrivals<false>(P, r, clocks, last, ring, 1);
    dcsim_merge_arrivals(P, r, 0, &merge_ring);
  }
}

}  // namespace

extern "C" {

size_t hostemu_pair_sizeof_spec(void) { return sizeof(dcsim_spec_t); }
size_t hostemu_pair_sizeof_arrhdr(void) { return sizeof(dcsim_arrhdr_t); }

/* dcsim_arrival_inputs_equal: 1 equal, 0 not (the first differing field's name into `field`, `field_bytes` long), -1 on
 * a malformed blob. */
int hostemu_pair_compatible(const void* a, size_t a_bytes, const void* b, size_t b_bytes, char* field, size_t field_bytes) {
  if (!spec_ok(a, a_bytes) || !spec_ok(b, b_bytes)) return -1;
  const char* diff = NULL;
  const bool eq = dcsim_arrival_inputs_equal((const dcsim_spec_t*)a, (const dcsim_spec_t*)b, &diff);
  if (field && field_bytes) snprintf(field, field_bytes, "%s", diff ? diff : "");
  return eq ? 1 : 0;
}

/* The merged lists of n replicas from keys seed0, seed0 + 1, ...: ml_t / ml_aux / ml_meta [n][2 * cap_arr] (the first
 * hdr[r].ml_count entries of row r are the list) and the headers [n] (dcsim_arrhdr_t).  -1 on a bad blob. */
int hostemu_pair_lists(const void* spec_blob, size_t spec_bytes, uint64_t n_replicas, uint64_t seed0, int rng_kind,
                       double* ml_t, double* ml_aux, uint32_t* ml_meta, void* hdr) {
  if (!spec_ok(spec_blob, spec_bytes)) return -1;
  dcsim_kparams_t* P = make_params(spec_blob, n_replicas, seed0, 0, rng_kind);
  draw_lists(P, rng_kind);
  const size_t ne2 = 2 * n_replicas * (size_t)P->cap_arr;
  memcpy(ml_t, P->ml_t, ne2 * sizeof(double));
  memcpy(ml_aux, P->ml_aux, ne2 * sizeof(double));
  memcpy(ml_meta, P->ml_meta, ne2 * sizeof(uint32_t));
  memcpy(hdr, P->arr_hdr, n_replicas * sizeof(dcsim_arrhdr_t));
  free_params(P);
  return 0;
}

/* The pre-pass and the merge under `spec_src`, then the event loop of `spec_run` on those lists (what a member of
 * spec_src's group runs): n replicas from keys seed0, seed0 + 1, ...; each launch processes `chunk_events` events per
 * replica (0 = to the end).  Returns the events processed, -1 on a bad blob or specs whose arrival inputs differ. */
long long hostemu_pair_run(const void* spec_src, const void* spec_run, size_t spec_bytes, uint64_t n_replicas, uint64_t seed0,
                           uint64_t chunk_events, int rng_kind, double* out_summaries) {
  if (!spec_ok(spec_src, spec_bytes) || !spec_ok(spec_run, spec_bytes)) return -1;
  if (!dcsim_arrival_inputs_equal((const dcsim_spec_t*)spec_src, (const dcsim_spec_t*)spec_run)) return -1;
  dcsim_kparams_t* P = make_params(spec_src, n_replicas, seed0, chunk_events, rng_kind);
  uint32_t counts[4] = {0, 0, 0, 0};
  P->rec.counts = counts;
  draw_lists(P, rng_kind);
  memcpy(&P->spec, spec_run, sizeof(dcsim_spec_t)); /* the member's own spec and layout from here on */
  dcsim_make_layout(&P->spec, &P->L, /*job_log=*/0);
  P->state = (char*)calloc(n_replicas, (size_t)P->L.total_bytes);
  P->queues = (char*)calloc(n_replicas, (size_t)P->L.queue_bytes + 16);
  P->summary = out_summaries;
  char* work = (char*)malloc((size_t)P->L.total_bytes);
  long long total = 0;
  for (uint64_t r = 0; r < n_replicas; ++r) {
    char* home = P->state + r * (uint64_t)P->L.total_bytes;
    for (int guard = 0; guard < 100000000; ++guard) {
      const bool fresh = ((dcsim_hdr_t*)home)->initialized == 0u;
      if (!fresh) memcpy(work, home, (size_t)P->L.total_bytes); /* stage in */
      total += P->L.cap_stale ? dcsim_replica_step<true, false>(P, r, work, work, fresh) : dcsim_replica_step<false, false>(P, r, work, work, fresh);
      memcpy(home, work, (size_t)P->L.total_bytes);             /* stage out */
      const dcsim_hdr_t* H = (const dcsim_hdr_t*)home;
      if (H->done || H->status || chunk_events == 0) break;
    }
  }
  free(work); free(P->state); free(P->queues);
  free_params(P);
  return total;
}

} /* extern "C" */
