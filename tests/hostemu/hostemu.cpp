/*
 * TEST-ONLY.  Single-lane host build of distributed_cluster_gpus_b200/csrc/dcsim_core.cuh
 * (DCSIM_LANES = 1; warp collectives are identities, atomics plain read-modify-writes).  Lets the CPU test-suite run the
 * *device source's* pre-pass, list merge, handler logic, state-block layout, Philox window, FIFO rings, resume path and
 * recorders against the oracle where no GPU exists.  It is not part of, linked into, or reachable from the product
 * library — the product fails loudly without CUDA.  What it cannot show (lane mapping, __syncwarp placement, REDUX) is
 * what the `-m gpu` parity tests are for.
 *
 * Launch parameters come from the library's own rules (dcsim_cap_arr, dcsim_max_transfer, dcsim_job_fields,
 * dcsim_derive_kparams, dcsim_profile_recorders).  Built four times by build.sh: plain, DCSIM_HOST_UNIFORM_LOOP (the
 * warp-uniform event-loop skeleton of the lane-group GPU builds), DCSIM_HOSTEMU_PERTURB (below) and DCSIM_MERGE_RING=32u
 * (a merge ring of one chunk: every scan that reaches back or ahead takes the HBM fall-back path).
 */
#define DCSIM_HOST_EMU 1
#ifdef DCSIM_HOSTEMU_PERTURB
/* Conditioning probe (libdcsim_hostemu_perturbed.so): every 5th pow() result is moved by ONE ulp — the
 * kind of difference two correct libm implementations (glibc here, CUDA's on the device) have.  How far a scenario's
 * results move under it is that scenario's sensitivity to last-bit differences: ~1e-15 for ordinary scenarios, orders
 * of magnitude more where the power-cap controller keeps re-timing back-to-back jobs (each re-timing multiplies a
 * start-time error by rate_old/rate_new).  tools/fuzz_gpu.py uses it to tell ill-conditioned scenarios from bugs. */
#include <math.h>
static inline double dcsim_hostemu_perturbed_pow(double a, double b) {
  static unsigned long calls = 0;
  const double r = pow(a, b);
  return (++calls % 5ul == 0ul) ? nextafter(r, INFINITY) : r;
}
#define pow dcsim_hostemu_perturbed_pow
#endif
#include "../../distributed_cluster_gpus_b200/csrc/dcsim_core.cuh"

#include <stdio.h>
#include <stdlib.h>

/* The outputs of one run, each NULL (0) when off; the recorders mirror the library's dcsim_enable_* calls. */
struct hostemu_out_t {
  double* summary;                   /* [n][DCSIM_SUMMARY_K] */
  int64_t rec_replica;               /* the replica trace / jobs / cluster record, -1: none */
  dcsim_trace_rec_t* trace;
  dcsim_job_rec_t* jobs;
  dcsim_cluster_rec_t* cluster;
  uint32_t trace_cap, jobs_cap, cluster_cap, ens_cap;
  uint32_t* counts;                  /* [4]: the rows trace, jobs and cluster would have written */
  int32_t* layout;                   /* [6]: total_bytes, cap_xfer, cap_run, cap_q_inf, cap_q_trn, rec_off */
  uint32_t* lat_hist;                /* [n][2][DCSIM_LAT_BINS] */
  double* ens;                       /* [ens_cap][DCSIM_ENS_FIELDS][n_dc][n] */
  double* jens;                      /* [W + 1][DCSIM_JENS_STORED][n_dc][2][n], W = dcsim_jens_windows(end_time, jens_bin) */
  uint32_t* jens_hist;               /* [n][n_dc][2][DCSIM_LAT_BINS] */
  double jens_bin;
  double* jwait;                     /* [W + 1][DCSIM_JWAIT_STORED][n_dc][2][n] (with jens) */
  uint32_t* jwait_hist;              /* [n][n_dc][2][2][DCSIM_LAT_BINS] */
  double* jres;                      /* [W + 1][DCSIM_JRES_STORED][n_dc][2][n] (with jens) */
  uint32_t* jres_mix;                /* [n_dc][2][DCSIM_JRES_MIX_COLS(G)][n] */
  uint32_t* jres_hist;               /* [n_dc][2][DCSIM_JRES_EBINS][n] */
  double* pp;                        /* [DCSIM_PP_FIELDS + n_dc + DCSIM_PP_BINS][n] */
  double pp_threshold;
  double* occ;                       /* [1 + DCSIM_OCC_FIELDS * n_dc + 2 * DCSIM_OCC_BINS * n_dc][n] */
  double* tail;                      /* [n][cap_arr][2], set to NaN here */
  double* tail_cols;                 /* [DCSIM_TAIL_COLS(n_dc)][n] (with tail) */
  double tail_sla;
  double* cost;                      /* [DCSIM_COST_COLS(n_dc)][n] */
  /* what the pre-pass and the merge leave: arr_* [n][cap_arr], ml_* [n][2 * cap_arr], arr_hdr [n]; entries they did not
   * write hold 0xee bytes */
  double* arr_t;
  double* arr_raw;
  uint32_t* arr_meta;
  uint32_t* arr_pred;
  double* arr_tx;
  double* ml_t;
  double* ml_aux;
  uint32_t* ml_meta;
  dcsim_arrhdr_t* arr_hdr;
  int32_t lists_only;                /* stop after the pre-pass and the merge */
};

namespace {

bool spec_ok(const void* blob, size_t bytes) {
  if (!blob || bytes != sizeof(dcsim_spec_t)) return false;
  const dcsim_spec_t* sp = (const dcsim_spec_t*)blob;
  return sp->magic == DCSIM_SPEC_MAGIC && sp->n_dc >= 1 && sp->n_dc <= DCSIM_MAX_DC && sp->n_ing >= 1 && sp->n_ing <= DCSIM_MAX_ING;
}

template <bool CAP, bool RECG>
uint32_t step(const dcsim_kparams_t* P, uint64_t r, char* work, char* rec, bool fresh) {
  return dcsim_profile_recorders(P) ? dcsim_replica_step<CAP, RECG, true>(P, r, work, rec, fresh)
                                    : dcsim_replica_step<CAP, RECG, false>(P, r, work, rec, fresh);
}

}  // namespace

extern "C" {

size_t hostemu_sizeof_spec(void) { return sizeof(dcsim_spec_t); }
size_t hostemu_sizeof_arrhdr(void) { return sizeof(dcsim_arrhdr_t); }
size_t hostemu_sizeof_out(void) { return sizeof(hostemu_out_t); }
uint32_t hostemu_merge_ring(void) { return DCSIM_MERGE_RING; }
void hostemu_set_test_time_quantum(double q) { dcsim_test_time_quantum = q; } /* see dcsim_core.cuh dcsim_test_quantize */
uint32_t hostemu_cap_arr(const void* spec_blob) { return dcsim_cap_arr((const dcsim_spec_t*)spec_blob); }
/* the library's default tick capacity (dcsim_recorder_enable of DCSIM_STAT_CLUSTER_ENSEMBLE with max_ticks = 0) */
uint32_t hostemu_ens_ticks(const void* spec_blob) { return dcsim_ens_ticks((const dcsim_spec_t*)spec_blob); }
/* the library's window count of the job-log ensemble for a resolved bin width (dcsim_recorder_enable of DCSIM_STAT_JOB_ENSEMBLE) */
uint64_t hostemu_jens_windows(const void* spec_blob, double bin_s) {
  return dcsim_jens_windows(((const dcsim_spec_t*)spec_blob)->end_time, bin_s);
}
/* the library's histogram range for a spec (dcsim_power_profile_range) */
double hostemu_pp_range(const void* spec_blob) { return dcsim_pp_range((const dcsim_spec_t*)spec_blob); }
/* the GPU-count rows of the job-resources mix (the last one takes g >= G) */
uint32_t hostemu_jres_g(const void* spec_blob) { return (uint32_t)DCSIM_JRES_G(((const dcsim_spec_t*)spec_blob)->max_gpus_per_job); }
/* the energy-cost recorder's hour window of an instant (dcsim_cost_window), and the hour the handlers use
 * (dcsim_current_hour) */
double hostemu_energy_cost_window(double t) { return dcsim_cost_window(t); }
int hostemu_current_hour(double t) { return dcsim_current_hour(t); }

/* dcsim_arrival_inputs_equal: 1 equal, 0 not (the first differing field's name into `field`, `field_bytes` long), -1 on
 * a malformed blob. */
int hostemu_compatible(const void* a, size_t a_bytes, const void* b, size_t b_bytes, char* field, size_t field_bytes) {
  if (!spec_ok(a, a_bytes) || !spec_ok(b, b_bytes)) return -1;
  const char* diff = NULL;
  const bool eq = dcsim_arrival_inputs_equal((const dcsim_spec_t*)a, (const dcsim_spec_t*)b, &diff);
  if (field && field_bytes) snprintf(field, field_bytes, "%s", diff ? diff : "");
  return eq ? 1 : 0;
}

/* n replicas from keys seed0, seed0 + 1, ...: the pre-pass and the list merge under `spec_lists`, replica by replica,
 * then the event loop of `spec_run` on those lists (what a member of spec_lists's group runs; the two are the same blob
 * outside that case).  Each launch processes `chunk_events` events per replica (0 = to the end) and the state block
 * round-trips through "HBM" between launches exactly as the kernel's stage-in/stage-out does; DCSIM_RECORDS=global:
 * the kernel's head-staged mode (only [0, rec_off) is staged, the running-job records are used where they live).
 * rng_kind: 0 Philox, 1 MT19937.  Returns the events processed, -1 on a bad blob or specs whose arrival inputs differ. */
long long hostemu_run_batch(const void* spec_lists, const void* spec_run, size_t spec_bytes, uint64_t n_replicas,
                            uint64_t seed0, uint64_t chunk_events, int rng_kind, const hostemu_out_t* o) {
  if (!spec_ok(spec_lists, spec_bytes) || !spec_ok(spec_run, spec_bytes)) return -1;
  if (!dcsim_arrival_inputs_equal((const dcsim_spec_t*)spec_lists, (const dcsim_spec_t*)spec_run)) return -1;
  dcsim_kparams_t* P = (dcsim_kparams_t*)calloc(1, sizeof(dcsim_kparams_t));
  memcpy(&P->spec, spec_run, sizeof(dcsim_spec_t));
  uint32_t local_counts[4] = {0, 0, 0, 0};
  P->rec.trace = o->trace; P->rec.jobs = o->jobs; P->rec.cluster = o->cluster;
  P->rec.counts = o->counts ? o->counts : local_counts;
  P->rec.counts[0] = P->rec.counts[1] = P->rec.counts[2] = 0;
  P->rec.trace_cap = o->trace_cap; P->rec.jobs_cap = o->jobs_cap; P->rec.cluster_cap = o->cluster_cap;
  P->rec.trace_replica = o->trace ? o->rec_replica : -1; P->rec.log_replica = (o->jobs || o->cluster) ? o->rec_replica : -1;
  P->n_replicas = n_replicas; P->seed0 = seed0; P->max_events = chunk_events;
  P->summary = o->summary;
  P->lat_hist = o->lat_hist;
  P->ens = o->ens; P->ens_cap = o->ens ? o->ens_cap : 0u;
  if (o->jens) {
    P->jens = o->jens; P->jens_hist = o->jens_hist; P->jens_bin = o->jens_bin;
    P->jens_windows = dcsim_jens_windows(P->spec.end_time, o->jens_bin);
  }
  P->jwait = o->jwait; P->jwait_hist = o->jwait_hist;
  P->jres = o->jres; P->jres_mix = o->jres_mix; P->jres_hist = o->jres_hist;
  if (o->pp) {
    P->pp = o->pp; P->pp_threshold = o->pp_threshold;
    P->pp_work = (double*)calloc(n_replicas * (size_t)DCSIM_PPW_N, sizeof(double));
  }
  if (o->occ) {
    P->occ = o->occ;
    P->occ_work = (double*)calloc(n_replicas * (size_t)P->spec.n_dc * DCSIM_OCCW_N, sizeof(double));
  }
  P->tail = o->tail; P->tail_cols = o->tail_cols; P->tail_sla = o->tail_sla;
  if (o->cost) {
    P->cost = o->cost;
    P->cost_work = (double*)calloc(n_replicas * (size_t)P->spec.n_dc * DCSIM_COSTW_N, sizeof(double));
  }
  dcsim_derive_kparams(P);

  /* the pre-pass and the merge: the owner's spec and the layout it implies (dcsim_prepare) */
  const dcsim_spec_t* sl = (const dcsim_spec_t*)spec_lists;
  P->cap_arr = dcsim_cap_arr(sl);
  P->max_transfer = dcsim_max_transfer(sl, dcsim_test_time_quantum);
  const size_t ne = n_replicas * (size_t)P->cap_arr;
  P->arr_t = (double*)malloc(ne * sizeof(double));
  P->arr_raw = (double*)malloc(ne * sizeof(double));
  P->arr_meta = (uint32_t*)malloc(ne * sizeof(uint32_t));
  P->arr_pred = (uint32_t*)malloc(ne * sizeof(uint32_t));
  P->arr_tx = (double*)malloc(ne * sizeof(double));
  P->arr_fin = (uint32_t*)calloc(ne, sizeof(uint32_t));
  P->ml_t = (double*)malloc(2 * ne * sizeof(double));
  P->ml_aux = (double*)malloc(2 * ne * sizeof(double));
  P->ml_meta = (uint32_t*)malloc(2 * ne * sizeof(uint32_t));
  P->arr_hdr = (dcsim_arrhdr_t*)calloc(n_replicas, sizeof(dcsim_arrhdr_t));
  /* an entry the pre-pass or the merge never wrote would show */
  memset(P->arr_t, 0xee, ne * sizeof(double)); memset(P->arr_raw, 0xee, ne * sizeof(double));
  memset(P->arr_meta, 0xee, ne * sizeof(uint32_t)); memset(P->arr_pred, 0xee, ne * sizeof(uint32_t));
  memset(P->arr_tx, 0xee, ne * sizeof(double));
  memset(P->ml_t, 0xee, 2 * ne * sizeof(double)); memset(P->ml_aux, 0xee, 2 * ne * sizeof(double));
  memset(P->ml_meta, 0xee, 2 * ne * sizeof(uint32_t));
  if (rng_kind == 1) P->mt_state = (uint32_t*)calloc(n_replicas * (size_t)DCSIM_MT_N, sizeof(uint32_t));
  {
    memcpy(&P->spec, sl, sizeof(dcsim_spec_t));
    dcsim_make_layout(&P->spec, &P->L, /*job_log=*/0);
    double clocks[2 * DCSIM_MAX_ING];
    uint32_t last[2 * DCSIM_MAX_ING];
    uint32_t ring[DCSIM_TRNG_RING];
    static dcsim_merge_ring_t merge_ring;
    for (uint64_t r = 0; r < n_replicas; ++r) {
      if (rng_kind == 1) dcsim_generate_arrivals<true>(P, r, clocks, last, ring, 1); else dcsim_generate_arrivals<false>(P, r, clocks, last, ring, 1);
      dcsim_merge_arrivals(P, r, 0, &merge_ring);
      /* self-check: the merged list is a gap-free, (t)-sorted permutation of the replica's events */
      const dcsim_arrhdr_t* ah = P->arr_hdr + r;
      const double* mt = P->ml_t + 2 * r * (uint64_t)P->cap_arr;
      const uint32_t* mm = P->ml_meta + 2 * r * (uint64_t)P->cap_arr;
      for (uint32_t p = 0; p < ah->ml_count; ++p)
        if (mm[p] == 0xeeeeeeeeu || (p && mt[p] < mt[p - 1])) { fprintf(stderr, "hostemu: merged list broken at %u of %u (replica %llu)\n", p, ah->ml_count, (unsigned long long)r); abort(); }
    }
  }

  long long total = 0;
  if (!o->lists_only) { /* the member's own spec and layout from here on */
    memcpy(&P->spec, spec_run, sizeof(dcsim_spec_t));
    dcsim_make_layout(&P->spec, &P->L, dcsim_job_fields(o->jobs != NULL, P->jwait, P->tail, P->jres));
    if (o->layout) { o->layout[0] = P->L.total_bytes; o->layout[1] = (P->L.xring_mask + 1) / 2; o->layout[2] = P->L.cap_run;
                     o->layout[3] = P->L.cap_q[0]; o->layout[4] = P->L.cap_q[1]; o->layout[5] = P->L.rec_off; }
    if (P->tail) memset(P->tail, 0xff, 2 * ne * sizeof(double)); /* NaN: not finished (as dcsim_recorder_enable fills it) */
    P->state = (char*)calloc(n_replicas, (size_t)P->L.total_bytes);
    P->queues = (char*)calloc(n_replicas, (size_t)P->L.queue_bytes + 16);
    char* work = (char*)malloc((size_t)P->L.total_bytes);
    const char* rm = getenv("DCSIM_RECORDS");
    const bool head_only = rm && rm[0] == 'g';
    const size_t staged = head_only ? (size_t)P->L.rec_off : (size_t)P->L.total_bytes;
    for (uint64_t r = 0; r < n_replicas; ++r) {
      char* home = P->state + r * (uint64_t)P->L.total_bytes;
      char* rec = head_only ? home : work;
      for (int guard = 0; guard < 100000000; ++guard) {
        const bool fresh = ((dcsim_hdr_t*)home)->initialized == 0u;
        if (!fresh) memcpy(work, home, staged); /* stage in */
        total += P->L.cap_stale ? (head_only ? step<true, true>(P, r, work, rec, fresh) : step<true, false>(P, r, work, rec, fresh))
                                 : (head_only ? step<false, true>(P, r, work, rec, fresh) : step<false, false>(P, r, work, rec, fresh));
        memcpy(home, work, staged);             /* stage out */
        const dcsim_hdr_t* H = (const dcsim_hdr_t*)home;
        if (H->done || H->status || chunk_events == 0) break;
      }
    }
    if (P->tail && P->tail_cols) {
      dcsim_tail_smem_t* S = (dcsim_tail_smem_t*)malloc(sizeof(dcsim_tail_smem_t));
      for (uint64_t r = 0; r < n_replicas; ++r) dcsim_tail_select(P, r, 0, 1, S);
      free(S);
    }
    free(work); free(P->state); free(P->queues);
  }
  if (o->arr_t) memcpy(o->arr_t, P->arr_t, ne * sizeof(double));
  if (o->arr_raw) memcpy(o->arr_raw, P->arr_raw, ne * sizeof(double));
  if (o->arr_meta) memcpy(o->arr_meta, P->arr_meta, ne * sizeof(uint32_t));
  if (o->arr_pred) memcpy(o->arr_pred, P->arr_pred, ne * sizeof(uint32_t));
  if (o->arr_tx) memcpy(o->arr_tx, P->arr_tx, ne * sizeof(double));
  if (o->ml_t) memcpy(o->ml_t, P->ml_t, 2 * ne * sizeof(double));
  if (o->ml_aux) memcpy(o->ml_aux, P->ml_aux, 2 * ne * sizeof(double));
  if (o->ml_meta) memcpy(o->ml_meta, P->ml_meta, 2 * ne * sizeof(uint32_t));
  if (o->arr_hdr) memcpy(o->arr_hdr, P->arr_hdr, n_replicas * sizeof(dcsim_arrhdr_t));
  free(P->arr_t); free(P->arr_raw); free(P->arr_meta); free(P->arr_pred); free(P->arr_tx); free(P->arr_fin);
  free(P->ml_t); free(P->ml_aux); free(P->ml_meta); free(P->arr_hdr); free(P->mt_state);
  free(P->pp_work); free(P->occ_work); free(P->cost_work); free(P);
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
