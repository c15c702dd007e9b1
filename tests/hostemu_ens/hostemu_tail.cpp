/*
 * TEST-ONLY.  Single-lane host build of distributed_cluster_gpus_b200/csrc/dcsim_core.cuh with the per-run tail-latency
 * recorder (P->tail) and its selection pass (dcsim_tail_select, one thread per "CTA") wired in, so that both can be
 * pinned against the oracle's per-job instants and numpy's order statistics where no GPU exists.  Exports the
 * time-quantum test hook of tests/hostemu.  The batch driver is the one of hostemu_jwait.cpp next to it (pre-pass and
 * list merge replica by replica, then every replica's state block round-tripping through "HBM" between launches of
 * `chunk_events` events); it is not part of, linked into, or reachable from the product library.  Built twice by
 * build_tail.sh: plain, and with DCSIM_HOST_UNIFORM_LOOP (the warp-uniform event-loop skeleton of the lane-group GPU
 * builds).
 */
#define DCSIM_HOST_EMU 1
#include "../../distributed_cluster_gpus_b200/csrc/dcsim_core.cuh"

#include <stdio.h>
#include <stdlib.h>

extern "C" {

void hostemu_tail_set_test_time_quantum(double q) { dcsim_test_time_quantum = q; } /* see dcsim_core.cuh dcsim_test_quantize */

uint32_t hostemu_tail_cap_arr(const void* spec_blob) {
  const int32_t c = ((const dcsim_spec_t*)spec_blob)->cap_arrivals;
  return (uint32_t)(c > 0 ? c : 16384);
}

/* Runs n replicas from keys seed0, seed0 + 1, ...; each launch processes `chunk_events` events per replica (0 = to the
 * end).  `slots` (NULL: recorder off; the running records then stay lean, as in the library) [n_replicas][cap_arr][2]
 * doubles, set to NaN here; `cols` [DCSIM_TAIL_COLS(n_dc)][n_replicas] doubles, the selection pass's output (with
 * slots).  `arr_t`, `arr_tx` (each [n_replicas][cap_arr] doubles) and `arr_meta` ([n_replicas][cap_arr] u32), when not
 * NULL, receive the pre-pass's and the merge's buffers.  DCSIM_RECORDS=global: head-staged mode.  Returns the events
 * processed, -1 on a bad spec blob. */
long long hostemu_tail_run_batch(const void* spec_blob, size_t spec_bytes, uint64_t n_replicas, uint64_t seed0,
                                 uint64_t chunk_events, double* out_summaries, int rng_kind, double sla_s, double* slots,
                                 double* cols, double* arr_t_out, double* arr_tx_out, uint32_t* arr_meta_out) {
  if (!spec_blob || spec_bytes != sizeof(dcsim_spec_t)) return -1;
  dcsim_kparams_t* P = (dcsim_kparams_t*)calloc(1, sizeof(dcsim_kparams_t));
  memcpy(&P->spec, spec_blob, sizeof(dcsim_spec_t));
  if (P->spec.magic != DCSIM_SPEC_MAGIC) { free(P); return -1; }
  dcsim_make_layout(&P->spec, &P->L, /*job_log=*/slots != NULL); /* the library's relayout rule */
  P->cap_arr = hostemu_tail_cap_arr(spec_blob);
  uint32_t counts[4] = {0, 0, 0, 0};
  P->rec.counts = counts;
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
  P->max_transfer += dcsim_test_time_quantum; /* test hook: a rounded-up xfer_done instant may exceed t + transfer_s */
  P->state = (char*)calloc(n_replicas, (size_t)P->L.total_bytes);
  P->queues = (char*)calloc(n_replicas, (size_t)P->L.queue_bytes + 16);
  P->summary = out_summaries;
  const size_t ne = n_replicas * (size_t)P->cap_arr;
  P->tail = slots; P->tail_cols = cols; P->tail_sla = sla_s;
  if (slots) memset(slots, 0xff, 2 * ne * sizeof(double)); /* NaN: not finished (dcsim_enable_tail_latency) */
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
  {
    double clocks[2 * DCSIM_MAX_ING];
    uint32_t last[2 * DCSIM_MAX_ING];
    uint32_t ring[DCSIM_TRNG_RING];
    static dcsim_merge_ring_t merge_ring;
    for (uint64_t r = 0; r < n_replicas; ++r) {
      if (rng_kind == 1) dcsim_generate_arrivals<true>(P, r, clocks, last, ring, 1); else dcsim_generate_arrivals<false>(P, r, clocks, last, ring, 1);
      dcsim_merge_arrivals(P, r, 0, &merge_ring);
    }
  }
  char* work = (char*)malloc((size_t)P->L.total_bytes);
  const char* rm = getenv("DCSIM_RECORDS");
  const bool head_only = rm && rm[0] == 'g';
  const size_t staged = head_only ? (size_t)P->L.rec_off : (size_t)P->L.total_bytes;
  long long total = 0;
  for (uint64_t r = 0; r < n_replicas; ++r) {
    char* home = P->state + r * (uint64_t)P->L.total_bytes;
    char* rec = head_only ? home : work;
    for (int guard = 0; guard < 100000000; ++guard) {
      const bool fresh = ((dcsim_hdr_t*)home)->initialized == 0u;
      if (!fresh) memcpy(work, home, staged); /* stage in */
      /* the profile instantiation (PP), the one the library launches with the recorder on */
      total += P->L.cap_stale ? (head_only ? dcsim_replica_step<true, true, true>(P, r, work, rec, fresh) : dcsim_replica_step<true, false, true>(P, r, work, rec, fresh))
                               : (head_only ? dcsim_replica_step<false, true, true>(P, r, work, rec, fresh) : dcsim_replica_step<false, false, true>(P, r, work, rec, fresh));
      memcpy(home, work, staged);             /* stage out */
      const dcsim_hdr_t* H = (const dcsim_hdr_t*)home;
      if (H->done || H->status || chunk_events == 0) break;
    }
  }
  if (slots && cols) {
    dcsim_tail_smem_t* S = (dcsim_tail_smem_t*)malloc(sizeof(dcsim_tail_smem_t));
    for (uint64_t r = 0; r < n_replicas; ++r) dcsim_tail_select(P, r, 0, 1, S);
    free(S);
  }
  if (arr_t_out) memcpy(arr_t_out, P->arr_t, ne * sizeof(double));
  if (arr_tx_out) memcpy(arr_tx_out, P->arr_tx, ne * sizeof(double));
  if (arr_meta_out) memcpy(arr_meta_out, P->arr_meta, ne * sizeof(uint32_t));
  free(work); free(P->state); free(P->queues); free(P->arr_t); free(P->arr_raw); free(P->arr_meta); free(P->arr_pred); free(P->arr_tx); free(P->arr_fin);
  free(P->ml_t); free(P->ml_aux); free(P->ml_meta); free(P->arr_hdr); free(P->mt_state); free(P);
  return total;
}

/* The selection pass alone on synthetic jobs: one replica of a 1-DC spec whose `n` created slots hold arrival 0,
 * xfer_done `tx[k]`, start `start[k]` and finish `finish[k]` (NaN: unfinished), job type `jtype[k]`.  `summary_status`
 * is the replica's status word.  `cols`: [DCSIM_TAIL_COLS(1)] doubles. */
void hostemu_tail_select_synthetic(uint32_t n, const double* tx, const double* start, const double* finish,
                                   const int32_t* jtype, double sla_s, double summary_status, double* cols) {
  dcsim_kparams_t* P = (dcsim_kparams_t*)calloc(1, sizeof(dcsim_kparams_t));
  P->spec.n_dc = 1;
  P->n_replicas = 1;
  P->cap_arr = n ? n : 1;
  double summary[DCSIM_SUMMARY_K] = {0};
  summary[DCSIM_S_STATUS] = summary_status;
  summary[DCSIM_S_JOBS_CREATED] = (double)n;
  P->summary = summary;
  P->arr_t = (double*)calloc(P->cap_arr, sizeof(double));
  P->arr_tx = (double*)calloc(P->cap_arr, sizeof(double));
  P->arr_meta = (uint32_t*)calloc(P->cap_arr, sizeof(uint32_t));
  P->tail = (double*)calloc(2 * (size_t)P->cap_arr, sizeof(double));
  for (uint32_t k = 0; k < n; ++k) {
    P->arr_tx[k] = tx[k];
    P->arr_meta[k] = (uint32_t)(jtype[k] & 1); /* stream jt of ingress 0, routed to DC 0 */
    P->tail[2 * k] = start[k];
    P->tail[2 * k + 1] = finish[k];
  }
  P->tail_cols = cols;
  P->tail_sla = sla_s;
  dcsim_tail_smem_t* S = (dcsim_tail_smem_t*)malloc(sizeof(dcsim_tail_smem_t));
  dcsim_tail_select(P, 0, 0, 1, S);
  free(S); free(P->arr_t); free(P->arr_tx); free(P->arr_meta); free(P->tail); free(P);
}

} /* extern "C" */
