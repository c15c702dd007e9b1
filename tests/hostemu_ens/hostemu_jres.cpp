/*
 * TEST-ONLY.  Single-lane host build of distributed_cluster_gpus_b200/csrc/dcsim_core.cuh with the job-log ensemble
 * recorder (P->jens, P->jens_hist) and the job-resources recorder on top of it (P->jres, P->jres_mix, P->jres_hist)
 * wired in, so that the recorder of the device source can be pinned against the oracle's job records where no GPU
 * exists.  The batch driver is the one of hostemu_jwait.cpp next to it (pre-pass and list merge replica by replica, then
 * every replica's state block round-tripping through "HBM" between launches of `chunk_events` events), running the
 * profile instantiation the library launches with the recorder on; it is not part of, linked into, or reachable from
 * the product library.  Built twice by build_jres.sh: plain, and with DCSIM_HOST_UNIFORM_LOOP (the warp-uniform
 * event-loop skeleton of the lane-group GPU builds).
 */
#define DCSIM_HOST_EMU 1
#include "../../distributed_cluster_gpus_b200/csrc/dcsim_core.cuh"

#include <stdio.h>
#include <stdlib.h>

extern "C" {

/* the library's window count of the job-log ensemble for a resolved bin width (dcsim_enable_job_ensemble) */
uint64_t hostemu_jres_windows(const void* spec_blob, double bin_s) {
  return dcsim_jens_windows(((const dcsim_spec_t*)spec_blob)->end_time, bin_s);
}

/* Runs n replicas from keys seed0, seed0 + 1, ...; each launch processes `chunk_events` events per replica (0 = to the
 * end).  `jens`: [W + 1][DCSIM_JENS_STORED][n_dc][2][n_replicas] doubles and `jens_hist`
 * [n_replicas][n_dc][2][DCSIM_LAT_BINS] u32, zeroed by the caller, W = hostemu_jres_windows(spec, bin_s).  `jres`
 * (NULL: recorder off; the running records then stay as lean as the spec allows, as in the library)
 * [W + 1][DCSIM_JRES_STORED][n_dc][2][n_replicas] doubles, `mix` [n_dc][2][DCSIM_JRES_MIX_COLS(G)][n_replicas] and
 * `ehist` [n_dc][2][DCSIM_JRES_EBINS][n_replicas] u32, zeroed by the caller.
 * DCSIM_RECORDS=global: head-staged mode (the running-job records are used where they live).  Returns the events
 * processed, -1 on a bad spec blob. */
long long hostemu_jres_run_batch(const void* spec_blob, size_t spec_bytes, uint64_t n_replicas, uint64_t seed0,
                                 uint64_t chunk_events, double* out_summaries, int rng_kind, double bin_s, double* jens,
                                 uint32_t* jens_hist, double* jres, uint32_t* mix, uint32_t* ehist) {
  if (!spec_blob || spec_bytes != sizeof(dcsim_spec_t)) return -1;
  dcsim_kparams_t* P = (dcsim_kparams_t*)calloc(1, sizeof(dcsim_kparams_t));
  memcpy(&P->spec, spec_blob, sizeof(dcsim_spec_t));
  if (P->spec.magic != DCSIM_SPEC_MAGIC) { free(P); return -1; }
  dcsim_make_layout(&P->spec, &P->L, /*job_log=*/jres != NULL); /* the library's relayout rule */
  P->cap_arr = (uint32_t)(P->spec.cap_arrivals > 0 ? P->spec.cap_arrivals : 16384);
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
  P->jens = jens; P->jens_hist = jens_hist; P->jens_bin = bin_s;
  P->jens_windows = dcsim_jens_windows(P->spec.end_time, bin_s);
  P->jres = jres; P->jres_mix = mix; P->jres_hist = ehist;
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
  free(work); free(P->state); free(P->queues); free(P->arr_t); free(P->arr_raw); free(P->arr_meta); free(P->arr_pred); free(P->arr_tx); free(P->arr_fin);
  free(P->ml_t); free(P->ml_aux); free(P->ml_meta); free(P->arr_hdr); free(P->mt_state); free(P);
  return total;
}

} /* extern "C" */
