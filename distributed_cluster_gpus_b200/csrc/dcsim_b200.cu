/*
 * dcsim_b200.cu — sm_90a kernels and the C-ABI of include/dcsim_b200.h.
 *
 * Kernels
 *   dcsim_arrivals_kernel     one thread per replica: the replica's arrival sequence (instants, routed DCs, size deviates).
 *   dcsim_merge_kernel        one warp per replica: job sizes, xfer_done instants and the merged, time-ordered
 *                             {arrival, xfer_done} list the event loop consumes.
 *   dcsim_advance_kernel      one warp per replica; stages the replica's state block HBM -> shared memory, runs the
 *                             event loop of dcsim_core.cuh, stages it back, writes the summary row.  Instantiated
 *                             over <CAP, MODE> (power-cap controller compiled in / what is staged) and picked per handle.
 *   dcsim_reduce_kernel       [n_replicas][K] summaries -> DCSIM_AGG_K doubles (the only cross-GPU payload).
 *   dcsim_hist_reduce_kernel  per-replica job-latency histograms -> one [2][128] histogram (opt-in); the same for the
 *                             per-DC [n_dc][2][128] histograms of the job-log ensemble.
 *   dcsim_ens_*_kernel        the cluster-log and job-log ensembles (opt-in) and the paired comparison of two batches
 *                             with the same keys -> per-column moments, then spread + histograms.
 *   dcsim_tail_select_kernel  one CTA per replica: the per-run tail-latency columns (opt-in) from the slot buffer, an
 *                             exact multi-target radix select (dcsim_tail_select, dcsim_core.cuh).
 *
 * Handles of one group (dcsim_create_shared) share the pre-pass's buffers and the merged lists it leaves: the arrival
 * lists do not depend on the policy (dcsim_arrival_inputs_equal, dcsim_core.cuh).
 *
 * Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -fmad=false (see __graft_entry__.build()).
 * -fmad=false matters: the reference is CPython float arithmetic, one rounding per operation.
 */
#include <cuda_runtime.h>
#include <dlfcn.h>

#include <float.h>
#include <new>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#define DCSIM_ADV_SUFFIX _g32
#include "dcsim_advance_impl.cuh" /* the 32-lanes-per-replica event loop (and dcsim_core.cuh) */

/* the builds with several replicas per warp live in their own translation units (dcsim_advance_g8.cu, _g16.cu) */
cudaError_t dcsim_adv_launch_g16(const dcsim_kparams_t*, unsigned long long*, int, int, int, int, int, cudaStream_t);
cudaError_t dcsim_adv_attrs_g16(int, int, int, int, int, int*, int*, int*);
cudaError_t dcsim_adv_launch_g8(const dcsim_kparams_t*, unsigned long long*, int, int, int, int, int, cudaStream_t);
cudaError_t dcsim_adv_attrs_g8(int, int, int, int, int, int*, int*, int*);
int dcsim_adv_min_ctas_g16(void);
int dcsim_adv_min_ctas_g8(void);

/* Arrival pre-pass: one THREAD per replica draws that replica's whole arrival sequence in the reference's draw order;
 * consecutive threads = consecutive replicas, so all 32 lanes of a warp run the samplers that the event loop would
 * otherwise run on one lane.  Per-thread scratch in shared memory, [slot][thread]: 2*n_ing stream clocks (f64),
 * 2*n_ing "latest arrival of the stream" indices (u32), DCSIM_TRNG_RING staged random words (u32), DCSIM_ARR_STAGE
 * staged arrivals (2 x f64 + 2 x u32). */
#define DCSIM_ARRIVALS_THREADS 128
/* 5 resident CTAs per SM: 132 x 5 x 128 = 84 480 threads on an H100, so the largest per-GPU batch of the BASELINE configs
 * (65 536 replicas) is ONE wave of this kernel, and the register cap it implies leaves both paths without spills (88
 * registers for the Philox path, 90 for MT19937 on sm_90a).  Shared memory allows the 5 CTAs up to 4 ingresses (40 KB per
 * CTA); at 8 ingresses a CTA takes 52 KB and 4 fit, 67 584 threads: still one wave of 65 536.  A tighter bound
 * (7: 72 registers) spills and bought nothing measurable on the H100: the kernel's time was the same at 7, 5 and 4
 * (measured before the output staging, when the kernel's time went to its scattered stores, DESIGN.md §4.0). */
#define DCSIM_ARRIVALS_MIN_CTAS 5
static size_t dcsim_arrivals_scratch_bytes(int n_ing) { /* per CTA: [slot][thread] arrays for 2 * n_ing streams, ring, stage */
  return (size_t)DCSIM_ARRIVALS_THREADS * ((size_t)(2 * n_ing) * (sizeof(double) + sizeof(uint32_t)) + DCSIM_TRNG_RING * sizeof(uint32_t) +
                                           DCSIM_ARR_STAGE * (2 * sizeof(double) + 2 * sizeof(uint32_t)));
}
extern __shared__ __align__(16) double dcsim_arr_scratch[];
template <bool MT>
__global__ void __launch_bounds__(DCSIM_ARRIVALS_THREADS, DCSIM_ARRIVALS_MIN_CTAS) dcsim_arrivals_kernel(const __grid_constant__ dcsim_kparams_t P) {
  const uint64_t r = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r - (threadIdx.x & 31u) >= P.n_replicas) return; /* whole warps only: the output flush needs every lane of a warp */
  const int n_streams = 2 * P.spec.n_ing;
  double* clocks = dcsim_arr_scratch + threadIdx.x;                                             /* [stream][thread] */
  uint32_t* last = reinterpret_cast<uint32_t*>(dcsim_arr_scratch + n_streams * blockDim.x) + threadIdx.x; /* [stream][thread] */
  uint32_t* ring = last + n_streams * blockDim.x;                                               /* [word][thread] */
  dcsim_arr_stage_t st;                                                                          /* [slot][thread] */
  st.t = reinterpret_cast<double*>(ring - threadIdx.x + DCSIM_TRNG_RING * blockDim.x) + threadIdx.x; /* 8-byte aligned: blockDim.x is even */
  st.raw = st.t + DCSIM_ARR_STAGE * blockDim.x;
  st.meta = reinterpret_cast<uint32_t*>(st.raw - threadIdx.x + DCSIM_ARR_STAGE * blockDim.x) + threadIdx.x;
  st.pred = st.meta + DCSIM_ARR_STAGE * blockDim.x;
  dcsim_generate_arrivals<MT>(&P, r, clocks, last, ring, (int)blockDim.x, st);
}

/* List merge: one WARP per replica (lane-parallel over the replica's arrivals), a sliding window of them in shared memory. */
#define DCSIM_MERGE_THREADS 128
__global__ void __launch_bounds__(DCSIM_MERGE_THREADS) dcsim_merge_kernel(const __grid_constant__ dcsim_kparams_t P) {
  __shared__ dcsim_merge_ring_t rings[DCSIM_MERGE_THREADS / 32];
  const uint64_t r = (uint64_t)blockIdx.x * (DCSIM_MERGE_THREADS / 32) + (threadIdx.x >> 5);
  if (r >= P.n_replicas) return;
  dcsim_merge_arrivals(&P, r, (int)(threadIdx.x & 31u), &rings[threadIdx.x >> 5]);
}

/* Per-run tail latency: one CTA per replica (grid-stride), its scratch a constant 18 KB of shared memory. */
#define DCSIM_TAIL_THREADS 256
__global__ void __launch_bounds__(DCSIM_TAIL_THREADS) dcsim_tail_select_kernel(const __grid_constant__ dcsim_kparams_t P) {
  __shared__ dcsim_tail_smem_t S;
  for (uint64_t r = blockIdx.x; r < P.n_replicas; r += gridDim.x) dcsim_tail_select(&P, r, (int)threadIdx.x, (int)blockDim.x, &S);
}

/* Sums per-replica histogram rows of `row_len` counts: thread t of every block owns bins t, t + blockDim.x, ...
 * (coalesced rows).  `status` (or NULL): the replicas whose word is not 0 are left out. */
__global__ void dcsim_hist_reduce_kernel(const uint32_t* __restrict__ hist, uint64_t n, uint32_t row_len,
                                         const uint32_t* __restrict__ status, unsigned long long* __restrict__ out) {
  for (uint32_t b = threadIdx.x; b < row_len; b += blockDim.x) {
    unsigned long long acc = 0ull;
    for (uint64_t r = blockIdx.x; r < n; r += gridDim.x)
      if (!status || status[r] == 0u) acc += hist[r * row_len + b];
    if (acc) atomicAdd(out + b, acc);
  }
}

/* Aggregates the summaries; every block reduces a slice, then one atomicAdd per component. */
__global__ void dcsim_reduce_kernel(const double* __restrict__ summary, uint64_t n, double* __restrict__ out) {
  double acc[DCSIM_AGG_K];
#pragma unroll
  for (int k = 0; k < DCSIM_AGG_K; ++k) acc[k] = 0.0;
  for (uint64_t r = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; r < n; r += (uint64_t)gridDim.x * blockDim.x) {
    const double* s = summary + r * DCSIM_SUMMARY_K;
    const double fin = s[DCSIM_S_JOBS_FINISHED], e = s[DCSIM_S_TOTAL_ENERGY_J];
    const double ml = fin > 0.0 ? s[DCSIM_S_LAT_SUM] / fin : 0.0;
    acc[DCSIM_A_REPLICAS] += 1.0;
    acc[DCSIM_A_FAILED] += (s[DCSIM_S_STATUS] != 0.0 || s[DCSIM_S_DONE] == 0.0) ? 1.0 : 0.0;
    acc[DCSIM_A_EVENTS] += s[DCSIM_S_EVENTS];
    acc[DCSIM_A_JOBS] += fin;
    acc[DCSIM_A_ENERGY] += e;
    acc[DCSIM_A_ENERGY_SQ] += e * e;
    acc[DCSIM_A_LAT_SUM] += s[DCSIM_S_LAT_SUM];
    acc[DCSIM_A_MEANLAT_SUM] += ml;
    acc[DCSIM_A_MEANLAT_SQ] += ml * ml;
    acc[DCSIM_A_RNG_WORDS] += s[DCSIM_S_RNG_WORDS];
    acc[DCSIM_A_RUNNING] += (s[DCSIM_S_STATUS] == 0.0 && s[DCSIM_S_DONE] == 0.0) ? 1.0 : 0.0;
  }
#pragma unroll
  for (int k = 0; k < DCSIM_AGG_K; ++k) {
    double v = acc[k];
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if ((threadIdx.x & 31u) == 0u && v != 0.0) atomicAdd(out + k, v);
  }
}

/* ---- ensemble reductions (cluster log, job log) ---------------------------------------------------------------
 * A column is one value per replica.  One CTA per column: thread t takes replicas t, t + 256, ... in order, then a
 * fixed shuffle tree and the warps' partials in warp order — the float sums depend on the replica count only, so they
 * are bit-identical from run to run (no float atomics).  A column source (Src) says where a column's values are, which
 * replicas count, and whether the column is an integer field:
 *   Src::at(col) -> a view whose get(r, v) loads replica r's value into v, false when r does not count;
 *   Src::integral(col). */
#define DCSIM_ENS_THREADS 256

/* Column `field` of every replica's summary row (as u32) into out[0, n), the maximum into out[n]: the ticks each replica
 * recorded (DCSIM_S_EV_LOG, the maximum is the capacity check) or its status bits (DCSIM_S_STATUS). */
__global__ void dcsim_ens_counts_kernel(const double* __restrict__ summary, uint64_t n, int field, uint32_t* __restrict__ out) {
  uint32_t m = 0u;
  for (uint64_t r = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; r < n; r += (uint64_t)gridDim.x * blockDim.x) {
    const uint32_t k = (uint32_t)summary[r * DCSIM_SUMMARY_K + field];
    out[r] = k;
    m = k > m ? k : m;
  }
  m = __reduce_max_sync(0xffffffffu, m);
  if ((threadIdx.x & 31u) == 0u && m) atomicMax(out + n, m);
}

/* Cluster-log ensemble: column (tick, field, dc) = n_replicas contiguous doubles, counted by the replicas that recorded
 * the tick (tick < nlog[r]). */
struct dcsim_ens_cluster_src {
  const double* ens;
  const uint32_t* nlog;
  uint64_t n;
  uint32_t cols_per_tick;
  int n_dc;
  struct view {
    const double* x;
    const uint32_t* nlog;
    uint32_t tick;
    __device__ __forceinline__ bool get(uint64_t r, double& v) const {
      if (!(tick < nlog[r])) return false;
      v = x[r];
      return true;
    }
  };
  __device__ __forceinline__ view at(uint64_t col) const { return view{ens + col * n, nlog, (uint32_t)(col / cols_per_tick)}; }
  __device__ __forceinline__ bool integral(uint64_t col) const {
    const int field = (int)((col / (uint64_t)n_dc) % DCSIM_ENS_FIELDS);
    return field >= DCSIM_ENS_BUSY && field <= DCSIM_ENS_Q_TRAIN;
  }
};

/* Job-log ensemble: column (row, field, dc, jtype), `cells` = n_dc * 2 per field.  JOBS and LAT_SUM are stored
 * ([row][DCSIM_JENS_STORED][cell][replica]); MEAN_LATENCY = LAT_SUM / JOBS over the replicas with a job in the cell.
 * Only replicas with status 0 count. */
struct dcsim_ens_job_src {
  const double* jens;
  const uint32_t* status;
  uint64_t n;
  uint32_t cells;
  struct view {
    const double* jobs;
    const double* lat;
    const uint32_t* status;
    int field;
    __device__ __forceinline__ bool get(uint64_t r, double& v) const {
      if (status[r] != 0u) return false;
      if (field == DCSIM_JENS_JOBS) { v = jobs[r]; return true; }
      if (field == DCSIM_JENS_LAT_SUM) { v = lat[r]; return true; }
      const double k = jobs[r];
      if (!(k > 0.0)) return false;
      v = lat[r] / k;
      return true;
    }
  };
  __device__ __forceinline__ view at(uint64_t col) const {
    const uint64_t row = col / ((uint64_t)DCSIM_JENS_FIELDS * cells), cell = col % cells;
    const double* jobs = jens + (row * DCSIM_JENS_STORED * cells + cell) * n;
    return view{jobs, jobs + (uint64_t)cells * n, status, (int)((col / cells) % DCSIM_JENS_FIELDS)};
  }
  __device__ __forceinline__ bool integral(uint64_t col) const { return (col / cells) % DCSIM_JENS_FIELDS == DCSIM_JENS_JOBS; }
};

/* Waiting and response times: column (row, field, dc, jtype) as the job-log ensemble's, `cells` = n_dc * 2 per field.
 * WAITED, WAIT_SUM and RESP_SUM are stored ([row][DCSIM_JWAIT_STORED][cell][replica]) and count for every valid replica;
 * MEAN_WAIT = WAIT_SUM / JOBS and MEAN_RESPONSE = RESP_SUM / JOBS for those with a job in the cell (JOBS: the job-log
 * ensemble's count of the same cell).  Only replicas with status 0 count. */
struct dcsim_ens_wait_src {
  const double* jwait;
  const double* jens;
  const uint32_t* status;
  uint64_t n;
  uint32_t cells;
  struct view {
    const double* x;
    const double* jobs;
    const uint32_t* status;
    bool mean;
    __device__ __forceinline__ bool get(uint64_t r, double& v) const {
      if (status[r] != 0u) return false;
      if (!mean) { v = x[r]; return true; }
      const double k = jobs[r];
      if (!(k > 0.0)) return false;
      v = x[r] / k;
      return true;
    }
  };
  __device__ __forceinline__ view at(uint64_t col) const {
    const uint64_t row = col / ((uint64_t)DCSIM_JWAIT_FIELDS * cells), cell = col % cells;
    const int field = (int)((col / cells) % DCSIM_JWAIT_FIELDS);
    const bool mean = field >= DCSIM_JWAIT_STORED;
    const uint64_t stored = mean ? (uint64_t)(field - DCSIM_JWAIT_STORED + DCSIM_JWAIT_WAIT_SUM) : (uint64_t)field;
    const double* x = jwait + ((row * DCSIM_JWAIT_STORED + stored) * cells + cell) * n;
    const double* jobs = jens + ((row * DCSIM_JENS_STORED + DCSIM_JENS_JOBS) * cells + cell) * n;
    return view{x, jobs, status, mean};
  }
  __device__ __forceinline__ bool integral(uint64_t col) const { return (col / cells) % DCSIM_JWAIT_FIELDS == DCSIM_JWAIT_WAITED; }
};

/* Job resources: first the windowed columns (row, field, dc, jtype) as the job-log ensemble's, `cells` = n_dc * 2 per
 * field — GPU_SUM, FREQ_SUM and ENERGY_SUM stored ([row][DCSIM_JRES_STORED][cell][replica]) and counted for every valid
 * replica, MEAN_* = *_SUM / JOBS for those with a job in the cell (JOBS: the job-log ensemble's count of the same cell) —
 * then the `count_cols` u32 count columns as stored (the mix, then the energy bins: [cells * (MIX_COLS + EBINS)][n]).
 * Only replicas with status 0 count. */
struct dcsim_ens_res_src {
  const double* jres;
  const double* jens;
  const uint32_t* counts;
  const uint32_t* status;
  uint64_t n;
  uint32_t cells;
  uint64_t win_cols; /* (W + 1) * DCSIM_JRES_FIELDS * cells */
  struct view {
    const double* x;
    const double* jobs;
    const uint32_t* u;
    const uint32_t* status;
    bool mean;
    __device__ __forceinline__ bool get(uint64_t r, double& v) const {
      if (status[r] != 0u) return false;
      if (u) { v = (double)u[r]; return true; }
      if (!mean) { v = x[r]; return true; }
      const double k = jobs[r];
      if (!(k > 0.0)) return false;
      v = x[r] / k;
      return true;
    }
  };
  __device__ __forceinline__ view at(uint64_t col) const {
    if (col >= win_cols) return view{nullptr, nullptr, counts + (col - win_cols) * n, status, false};
    const uint64_t row = col / ((uint64_t)DCSIM_JRES_FIELDS * cells), cell = col % cells;
    const int field = (int)((col / cells) % DCSIM_JRES_FIELDS);
    const bool mean = field >= DCSIM_JRES_STORED;
    const uint64_t stored = mean ? (uint64_t)(field - DCSIM_JRES_STORED) : (uint64_t)field;
    const double* x = jres + ((row * DCSIM_JRES_STORED + stored) * cells + cell) * n;
    const double* jobs = jens + ((row * DCSIM_JENS_STORED + DCSIM_JENS_JOBS) * cells + cell) * n;
    return view{x, jobs, nullptr, status, mean};
  }
  __device__ __forceinline__ bool integral(uint64_t col) const {
    return col >= win_cols || (col / cells) % DCSIM_JRES_FIELDS == DCSIM_JRES_GPU_SUM;
  }
};

/* Per-run tail latency: column c of the [DCSIM_TAIL_COLS(n_dc)][n] columns as stored.  A replica counts when its status
 * is 0 and the value is not NaN (an empty group's statistics, SLA_MET without a job or an SLA).  JOBS, UNFINISHED and
 * SLA_MET are the integer columns. */
struct dcsim_ens_tail_src {
  const double* cols;
  const uint32_t* status;
  uint64_t n;
  uint32_t group_cols; /* 2 * (n_dc + 1) * DCSIM_TAIL_GROUP_FIELDS: the SLA_MET columns follow */
  struct view {
    const double* x;
    const uint32_t* status;
    __device__ __forceinline__ bool get(uint64_t r, double& v) const {
      if (status[r] != 0u) return false;
      v = x[r];
      return v == v;
    }
  };
  __device__ __forceinline__ view at(uint64_t col) const { return view{cols + col * n, status}; }
  __device__ __forceinline__ bool integral(uint64_t col) const {
    return col >= group_cols || col % DCSIM_TAIL_GROUP_FIELDS <= DCSIM_TAIL_UNFINISHED;
  }
};

/* Paired comparison: column (metric, field) over replica r's summary rows of a base and a variant batch (the same keys).
 * Counted when both rows have status 0 and the metric is defined in both; fields base, variant, variant - base,
 * variant < base, variant > base (include/dcsim_b200.h DCSIM_PAIR_*). */
struct dcsim_ens_pair_src {
  const double* base;
  const double* var;
  int n_dc;
  struct view {
    const double* base;
    const double* var;
    int metric, field, n_dc;
    __device__ __forceinline__ static bool value(const double* s, int metric, int n_dc, double& v) {
      switch (metric) {
        case DCSIM_PAIR_ENERGY_J: v = s[DCSIM_S_TOTAL_ENERGY_J]; return true;
        case DCSIM_PAIR_ENERGY_PER_JOB_J:
          if (!(s[DCSIM_S_JOBS_FINISHED] > 0.0)) return false;
          v = s[DCSIM_S_TOTAL_ENERGY_J] / s[DCSIM_S_JOBS_FINISHED]; return true;
        case DCSIM_PAIR_JOBS_INF: v = s[DCSIM_S_FIN_INF]; return true;
        case DCSIM_PAIR_JOBS_TRN: v = s[DCSIM_S_FIN_TRN]; return true;
        case DCSIM_PAIR_MEAN_LAT_INF_S:
          if (!(s[DCSIM_S_FIN_INF] > 0.0)) return false;
          v = s[DCSIM_S_LAT_SUM_INF] / s[DCSIM_S_FIN_INF]; return true;
        case DCSIM_PAIR_MEAN_LAT_TRN_S:
          if (!(s[DCSIM_S_FIN_TRN] > 0.0)) return false;
          v = s[DCSIM_S_LAT_SUM_TRN] / s[DCSIM_S_FIN_TRN]; return true;
        case DCSIM_PAIR_UNFINISHED: {
          double u = 0.0;
          for (int d = 0; d < n_dc; ++d) {
            const double* g = s + DCSIM_S_DC0 + d * DCSIM_S_DC_STRIDE;
            u += g[DCSIM_SD_Q_INF] + g[DCSIM_SD_Q_TRN] + g[DCSIM_SD_RUNNING];
          }
          v = u; return true;
        }
        default: v = s[DCSIM_S_DC0 + (metric - DCSIM_PAIR_DC_ENERGY_J) * DCSIM_S_DC_STRIDE + DCSIM_SD_ENERGY_J]; return true;
      }
    }
    __device__ __forceinline__ bool get(uint64_t r, double& v) const {
      const double* b = base + r * DCSIM_SUMMARY_K;
      const double* x = var + r * DCSIM_SUMMARY_K;
      if (b[DCSIM_S_STATUS] != 0.0 || x[DCSIM_S_STATUS] != 0.0) return false;
      double vb, vx;
      if (!value(b, metric, n_dc, vb) || !value(x, metric, n_dc, vx)) return false;
      switch (field) {
        case DCSIM_PAIR_BASE: v = vb; break;
        case DCSIM_PAIR_VARIANT: v = vx; break;
        case DCSIM_PAIR_DIFF: v = vx - vb; break;
        case DCSIM_PAIR_LOWER: v = vx < vb ? 1.0 : 0.0; break;
        default: v = vx > vb ? 1.0 : 0.0; break;
      }
      return true;
    }
  };
  __device__ __forceinline__ view at(uint64_t col) const {
    return view{base, var, (int)(col / DCSIM_PAIR_FIELDS), (int)(col % DCSIM_PAIR_FIELDS), n_dc};
  }
  __device__ __forceinline__ bool integral(uint64_t col) const {
    const int metric = (int)(col / DCSIM_PAIR_FIELDS), field = (int)(col % DCSIM_PAIR_FIELDS);
    return field >= DCSIM_PAIR_LOWER || metric == DCSIM_PAIR_JOBS_INF || metric == DCSIM_PAIR_JOBS_TRN || metric == DCSIM_PAIR_UNFINISHED;
  }
};

/* Power profile: column c = n contiguous doubles ([DCSIM_PP_FIELDS + n_dc + DCSIM_PP_BINS][n]), counted by the replicas
 * with status 0. */
struct dcsim_ens_pp_src {
  const double* pp;
  const uint32_t* status;
  uint64_t n;
  struct view {
    const double* x;
    const uint32_t* status;
    __device__ __forceinline__ bool get(uint64_t r, double& v) const {
      if (status[r] != 0u) return false;
      v = x[r];
      return true;
    }
  };
  __device__ __forceinline__ view at(uint64_t col) const { return view{pp + col * n, status}; }
  __device__ __forceinline__ bool integral(uint64_t col) const {
    return col == DCSIM_PP_EXCURSIONS || col == DCSIM_PP_OUT_OF_RANGE;
  }
};

/* Energy cost: column c = n contiguous doubles ([DCSIM_COST_COLS(n_dc)][n]), counted by the replicas with status 0; no
 * integer columns. */
struct dcsim_ens_cost_src {
  const double* cost;
  const uint32_t* status;
  uint64_t n;
  using view = dcsim_ens_pp_src::view;
  __device__ __forceinline__ view at(uint64_t col) const { return view{cost + col * n, status}; }
  __device__ __forceinline__ bool integral(uint64_t) const { return false; }
};

/* Occupancy: the first DCSIM_OCC_FIELDS * n_dc columns are the statistics (field, dc) — the stored per-DC field over
 * PROFILE_S, the two maxima as stored — then the 2 * DCSIM_OCC_BINS * n_dc bins as stored
 * ([1 + DCSIM_OCC_FIELDS * n_dc + 2 * DCSIM_OCC_BINS * n_dc][n], column c of the source at stored column 1 + c).  A
 * replica counts when its status is 0 and PROFILE_S > 0. */
struct dcsim_ens_occ_src {
  const double* occ;
  const uint32_t* status;
  uint64_t n;
  uint32_t stat_cols; /* DCSIM_OCC_FIELDS * n_dc */
  uint32_t n_dc;
  struct view {
    const double* x;
    const double* profile;
    const uint32_t* status;
    bool share;
    __device__ __forceinline__ bool get(uint64_t r, double& v) const {
      const double p = profile[r];
      if (status[r] != 0u || !(p > 0.0)) return false;
      v = share ? x[r] / p : x[r];
      return true;
    }
  };
  __device__ __forceinline__ static bool is_max(int field) { return field == DCSIM_OCC_Q_INF_MAX || field == DCSIM_OCC_Q_TRN_MAX; }
  __device__ __forceinline__ view at(uint64_t col) const {
    const bool share = col < stat_cols && !is_max((int)(col / n_dc));
    return view{occ + (col + 1) * n, occ, status, share};
  }
  __device__ __forceinline__ bool integral(uint64_t col) const { return col < stat_cols && is_max((int)(col / n_dc)); }
};

__device__ __forceinline__ double dcsim_ens_min(double a, double b) { return b < a ? b : a; }
__device__ __forceinline__ double dcsim_ens_max(double a, double b) { return b > a ? b : a; }

/* Pass 1: out = [4][n_cols] {n, sum, min, max} over the replicas that count in the column. */
template <class Src>
__global__ void __launch_bounds__(DCSIM_ENS_THREADS) dcsim_ens_moments_kernel(const Src src, uint64_t n, uint64_t n_cols,
                                                                              double* __restrict__ out) {
  __shared__ double s_sum[DCSIM_ENS_THREADS / 32], s_lo[DCSIM_ENS_THREADS / 32], s_hi[DCSIM_ENS_THREADS / 32];
  __shared__ uint32_t s_cnt[DCSIM_ENS_THREADS / 32];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  for (uint64_t col = blockIdx.x; col < n_cols; col += gridDim.x) {
    const typename Src::view x = src.at(col);
    double sum = 0.0, lo = DCSIM_INF, hi = -DCSIM_INF;
    uint32_t cnt = 0u;
    for (uint64_t r = threadIdx.x; r < n; r += DCSIM_ENS_THREADS) {
      double v;
      if (x.get(r, v)) { sum += v; lo = dcsim_ens_min(lo, v); hi = dcsim_ens_max(hi, v); ++cnt; }
    }
    for (int o = 16; o > 0; o >>= 1) {
      sum += __shfl_xor_sync(0xffffffffu, sum, o);
      lo = dcsim_ens_min(lo, __shfl_xor_sync(0xffffffffu, lo, o));
      hi = dcsim_ens_max(hi, __shfl_xor_sync(0xffffffffu, hi, o));
      cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
    }
    if (lane == 0) { s_sum[w] = sum; s_lo[w] = lo; s_hi[w] = hi; s_cnt[w] = cnt; }
    __syncthreads();
    if (threadIdx.x == 0) {
      for (int k = 1; k < DCSIM_ENS_THREADS / 32; ++k) {
        sum += s_sum[k]; lo = dcsim_ens_min(lo, s_lo[k]); hi = dcsim_ens_max(hi, s_hi[k]); cnt += s_cnt[k];
      }
      out[col] = (double)cnt; out[n_cols + col] = sum; out[2 * n_cols + col] = lo; out[3 * n_cols + col] = hi;
    }
    __syncthreads();
  }
}

/* Pass 2: m2[col] = sum (x - mean)^2 and hist[col][DCSIM_ENS_BINS] over [lo, hi] (bin rule: include/dcsim_b200.h). */
template <class Src>
__global__ void __launch_bounds__(DCSIM_ENS_THREADS) dcsim_ens_spread_kernel(const Src src, uint64_t n, uint64_t n_cols,
                                                                             const double* __restrict__ mean, const double* __restrict__ lo_in,
                                                                             const double* __restrict__ hi_in, double* __restrict__ m2_out,
                                                                             unsigned long long* __restrict__ hist_out) {
  __shared__ uint32_t bins[DCSIM_ENS_BINS];
  __shared__ double s_m2[DCSIM_ENS_THREADS / 32];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  for (uint64_t col = blockIdx.x; col < n_cols; col += gridDim.x) {
    for (int b = threadIdx.x; b < DCSIM_ENS_BINS; b += DCSIM_ENS_THREADS) bins[b] = 0u;
    __syncthreads();
    const bool integral = src.integral(col);
    const double mu = mean[col], lo = lo_in[col], hi = hi_in[col];
    double width = 0.0; /* 0: everything in bin 0 */
    if (hi > lo) {
      if (integral) { const double span = hi - lo + 1.0; width = span <= (double)DCSIM_ENS_BINS ? 1.0 : ceil(span / (double)DCSIM_ENS_BINS); }
      else width = (hi - lo) / (double)DCSIM_ENS_BINS;
    }
    const typename Src::view x = src.at(col);
    double m2 = 0.0;
    for (uint64_t r = threadIdx.x; r < n; r += DCSIM_ENS_THREADS) {
      double v;
      if (x.get(r, v)) {
        const double dv = v - mu;
        m2 += dv * dv;
        int b = 0;
        if (width > 0.0) {
          const double f = floor((v - lo) / width);
          b = f >= (double)(DCSIM_ENS_BINS - 1) ? DCSIM_ENS_BINS - 1 : (f > 0.0 ? (int)f : 0);
        }
        atomicAdd(&bins[b], 1u);
      }
    }
    for (int o = 16; o > 0; o >>= 1) m2 += __shfl_xor_sync(0xffffffffu, m2, o);
    if (lane == 0) s_m2[w] = m2;
    __syncthreads();
    if (threadIdx.x == 0) {
      for (int k = 1; k < DCSIM_ENS_THREADS / 32; ++k) m2 += s_m2[k];
      m2_out[col] = m2;
    }
    for (int b = threadIdx.x; b < DCSIM_ENS_BINS; b += DCSIM_ENS_THREADS) hist_out[col * DCSIM_ENS_BINS + b] = bins[b];
    __syncthreads();
  }
}

/* ================================================================================================
 * C-ABI
 * ============================================================================================== */
/* What the handles of one group share: the arrival pre-pass's buffers and the merged lists it leaves, the replica keys,
 * the RNG kind and the stream every launch of the group goes to (so prepare -> advances -> reset -> prepare stay in
 * stream order).  A handle made by dcsim_create owns a group of one; dcsim_create_shared adds members whose specs have
 * the same arrival inputs (dcsim_arrival_inputs_equal).  Released with the last handle. */
struct dcsim_group {
  int refs;
  int device;
  dcsim_spec_t spec; /* the owner's: the pre-pass runs with it */
  uint64_t n_replicas, seed0;
  uint64_t generation; /* bumped by every reset of the owner */
  cudaStream_t stream, own_stream;
  int arrivals_ready;
  int rng_kind;
  uint32_t cap_arr;
  double max_transfer;
  double* d_arr_t;
  double* d_arr_raw;
  uint32_t* d_arr_meta;
  uint32_t* d_arr_pred;
  double* d_arr_tx;
  uint32_t* d_arr_fin;
  double* d_ml_t;
  double* d_ml_aux;
  uint32_t* d_ml_meta;
  dcsim_arrhdr_t* d_arr_hdr;
  uint32_t* d_mt; /* [624][n_replicas] Mersenne Twister states, rng_kind == DCSIM_RNG_MT19937 only */
#ifdef DCSIM_TEST_HOOKS
  double test_quantum; /* the time quantum of dcsim_test_set_time_quantum when the group was made */
#endif
};

static void group_release(dcsim_group* g) {
  if (!g || --g->refs > 0) return;
  cudaSetDevice(g->device);
  if (g->stream) cudaStreamSynchronize(g->stream);
  cudaFree(g->d_arr_t); cudaFree(g->d_arr_raw); cudaFree(g->d_arr_meta); cudaFree(g->d_arr_pred); cudaFree(g->d_arr_tx);
  cudaFree(g->d_arr_fin); cudaFree(g->d_ml_t); cudaFree(g->d_ml_aux); cudaFree(g->d_ml_meta); cudaFree(g->d_arr_hdr);
  cudaFree(g->d_mt);
  if (g->own_stream) cudaStreamDestroy(g->own_stream);
  delete g;
}

/* An opt-in batch recorder of a handle: its device buffers (d[0] != NULL: enabled), its resolved argument (bin_s,
 * threshold_w or sla_s; 0 for the others) and its rows (cluster ensemble: the tick capacity; job ensemble, job waits,
 * job resources: W + 1; the others: 1).  All zero while it is off. */
struct dcsim_slot {
  void* d[2];
  double arg;
  uint64_t rows;
};

struct dcsim {
  dcsim_spec_t spec;
  dcsim_layout_t L;
  dcsim_group* g;      /* arrival lists, keys, RNG kind, stream (shared with the rest of the group) */
  int member;          /* 1: made by dcsim_create_shared (owns neither keys nor stream) */
  uint64_t generation; /* the group generation this handle's batch was (re)set for */
  uint64_t n_replicas;
  int device, sm_count, warps_per_cta, ctas, smem_bytes, regs, resident_warps;
  int lanes; /* lanes per replica of the advance kernel picked for this handle: 32, 16 or 8 */
  char* d_state;
  char* d_queues;
  double* d_summary;
  double* h_summary_pinned; /* page-locked host mirror of d_summary, allocated on first use (dcsim_fetch_summary_host) */
  unsigned long long* d_events;
  double* d_agg;                 /* DCSIM_AGG_K doubles: scratch of dcsim_all_done */
  unsigned long long* d_hist_out; /* [2][DCSIM_LAT_BINS]: scratch of dcsim_fetch_latency_histogram */
  uint32_t* d_counts;
  dcsim_trace_rec_t* d_trace;
  dcsim_job_rec_t* d_jobs;
  dcsim_cluster_rec_t* d_cluster;
  uint32_t trace_cap, jobs_cap, cluster_cap;
  uint32_t jobs_alloc, cluster_alloc; /* rows the log buffers can hold (kept across set_logging calls) */
  int want_job_log;                   /* layout the NEXT batch needs; applied lazily by ensure_layout() */
  int64_t trace_replica, log_replica;
  int launches;
  int mode; /* DCSIM_MODE_* of the advance kernel for this handle's layout */
  uint32_t* d_hist;
  dcsim_slot rec[DCSIM_STATS]; /* the opt-in batch recorders, by DCSIM_STAT_* (their buffers: recorder_table) */
  int tail_fresh;          /* 1: the tail columns were selected from this batch's finished slots */
  uint32_t* d_ens_nlog; /* [n_replicas] ticks each cluster-ensemble replica recorded, + 1 word: the largest DCSIM_S_EV_LOG */
  unsigned long long* d_jens_hist_out;  /* [n_dc][2][DCSIM_LAT_BINS]: scratch of the job ensemble's histogram */
  unsigned long long* d_jwait_hist_out; /* [n_dc][2][2][DCSIM_LAT_BINS]: scratch of the job waits' histogram */
  uint32_t* d_status; /* [n_replicas] status words (+ 1 word: their maximum) of the recorder reductions, refreshed on
                         the stream ahead of every one of them (status_words) */
  unsigned long long events_seen;
  char err[512];
};

static thread_local char g_create_err[512] = "";

/* The byte sizes of the recorders' buffers (recorder_table): a whole buffer, or one row of those sized by rows. */
static size_t ens_tick_bytes(const dcsim_t* h) { /* one tick of the cluster-log ensemble */
  return (size_t)DCSIM_ENS_FIELDS * (size_t)h->spec.n_dc * (size_t)h->n_replicas * sizeof(double);
}

static size_t jens_row_bytes(const dcsim_t* h) { /* one row (window) of the job-log ensemble */
  return (size_t)DCSIM_JENS_STORED * (size_t)h->spec.n_dc * 2 * (size_t)h->n_replicas * sizeof(double);
}
static size_t jens_hist_bytes(const dcsim_t* h) {
  return (size_t)h->n_replicas * (size_t)h->spec.n_dc * 2 * DCSIM_LAT_BINS * sizeof(uint32_t);
}

static size_t jwait_row_bytes(const dcsim_t* h) {
  return (size_t)DCSIM_JWAIT_STORED * (size_t)h->spec.n_dc * 2 * (size_t)h->n_replicas * sizeof(double);
}
static size_t jwait_hist_bytes(const dcsim_t* h) { return 2 * jens_hist_bytes(h); }

static size_t jres_row_bytes(const dcsim_t* h) {
  return (size_t)DCSIM_JRES_STORED * (size_t)h->spec.n_dc * 2 * (size_t)h->n_replicas * sizeof(double);
}
static uint64_t jres_mix_cols(const dcsim_t* h) { /* per replica */
  return 2ull * (uint64_t)h->spec.n_dc * (uint64_t)DCSIM_JRES_MIX_COLS(DCSIM_JRES_G(h->spec.max_gpus_per_job));
}
static uint64_t jres_hist_cols(const dcsim_t* h) { return 2ull * (uint64_t)h->spec.n_dc * DCSIM_JRES_EBINS; }
static size_t jres_mix_bytes(const dcsim_t* h) { return (size_t)jres_mix_cols(h) * (size_t)h->n_replicas * sizeof(uint32_t); }
static size_t jres_ebin_bytes(const dcsim_t* h) { return (size_t)jres_hist_cols(h) * (size_t)h->n_replicas * sizeof(uint32_t); }
static size_t jres_cnt_bytes(const dcsim_t* h) { return jres_mix_bytes(h) + jres_ebin_bytes(h); }

static uint64_t pp_cols(const dcsim_t* h) { return (uint64_t)(DCSIM_PP_FIELDS + h->spec.n_dc + DCSIM_PP_BINS); }
static size_t pp_bytes(const dcsim_t* h) { return (size_t)pp_cols(h) * (size_t)h->n_replicas * sizeof(double); }
static size_t pp_work_bytes(const dcsim_t* h) { return (size_t)h->n_replicas * DCSIM_PPW_N * sizeof(double); }

static uint64_t occ_stat_cols(const dcsim_t* h) { return (uint64_t)DCSIM_OCC_FIELDS * (uint64_t)h->spec.n_dc; }
static uint64_t occ_cols(const dcsim_t* h) { return occ_stat_cols(h) + 2ull * DCSIM_OCC_BINS * (uint64_t)h->spec.n_dc; }
static size_t occ_bytes(const dcsim_t* h) { return (size_t)(1 + occ_cols(h)) * (size_t)h->n_replicas * sizeof(double); }
static size_t occ_work_bytes(const dcsim_t* h) {
  return (size_t)h->n_replicas * (size_t)h->spec.n_dc * DCSIM_OCCW_N * sizeof(double);
}

static uint64_t cost_cols(const dcsim_t* h) { return (uint64_t)DCSIM_COST_COLS(h->spec.n_dc); }
static size_t cost_bytes(const dcsim_t* h) { return (size_t)cost_cols(h) * (size_t)h->n_replicas * sizeof(double); }
static size_t cost_work_bytes(const dcsim_t* h) {
  return (size_t)h->n_replicas * (size_t)h->spec.n_dc * DCSIM_COSTW_N * sizeof(double);
}

static size_t tail_slot_bytes(const dcsim_t* h) { return (size_t)h->n_replicas * (size_t)h->g->cap_arr * 2 * sizeof(double); }
static size_t tail_cols_bytes(const dcsim_t* h) {
  return (size_t)DCSIM_TAIL_COLS(h->spec.n_dc) * (size_t)h->n_replicas * sizeof(double);
}

static int set_err(dcsim_t* h, int code, const char* fmt, const char* a = "", long long b = 0) {
  char* dst = h ? h->err : g_create_err;
  snprintf(dst, 512, fmt, a, b);
  return code;
}

#define CUDA_TRY(h, call)                                                                  \
  do {                                                                                     \
    cudaError_t e_ = (call);                                                               \
    if (e_ != cudaSuccess)                                                                 \
      return set_err(h, e_ == cudaErrorMemoryAllocation ? DCSIM_E_NOMEM : DCSIM_E_CUDA,    \
                     "CUDA error: %s (line %lld)", cudaGetErrorString(e_), (long long)__LINE__); \
  } while (0)

/* ---- the opt-in batch recorders: what each one does differently, by DCSIM_STAT_* ------------------------------------
 * Enabling one (dcsim_recorder_enable) checks, in this order: its argument, that the job ensemble is on (needs_jens),
 * that the handle is not a group member (unless member_ok), and — unless a re-targeting recorder is asked for the target
 * it has — that the batch has not advanced.  A re-targeting recorder (the two ensembles: their rows depend on the
 * argument) frees its buffers and those of the recorders that need it, then allocates anew; the others keep theirs and
 * only take the new argument.  Every buffer is filled with its `fill` byte on enable and on dcsim_reset (-1: left as it
 * is).  A fetch (dcsim_recorder_fetch) copies the recorder's parts, each one a buffer or the next `bytes` of it. */
enum { ARG_NONE, ARG_TICKS, ARG_BIN, ARG_LIMIT }; /* max_ticks; bin_s (finite, >= 0); threshold_w / sla_s (>= 0, +inf: none) */
typedef size_t (*rec_bytes_fn)(const dcsim_t*);
struct rec_buf { rec_bytes_fn bytes; bool per_row; int fill; };
struct rec_part { int buf; rec_bytes_fn bytes; /* NULL: the whole buffer */ };
struct rec_desc {
  const char* name;
  int arg;
  const char* arg_name;
  rec_buf buf[2];      /* bytes == NULL: no second buffer */
  rec_part part[3];
  int parts;
  bool retarget, needs_jens, member_ok;
  const char* nomem_hint;
  int (*ready)(dcsim_t*); /* the read precondition beyond recorder_ready (NULL: none) */
};

static int ens_counts(dcsim_t* h);
static int tail_ready(dcsim_t* h);

static const char* const FEWER = "run fewer replicas";
static const char* const WIDER = "a wider bin_s or fewer replicas";
static const rec_desc recorder_table[DCSIM_STATS] = {
  /* DCSIM_STAT_CLUSTER_ENSEMBLE: [ticks][FIELDS][n_dc][n] rows, NaN until recorded */
  {"cluster ensemble", ARG_TICKS, "max_ticks", {{ens_tick_bytes, true, 0xff}, {}}, {{0, NULL}}, 1,
   true, false, true, FEWER, ens_counts},
  /* DCSIM_STAT_JOB_ENSEMBLE: rows, per-replica latency histograms */
  {"job ensemble", ARG_BIN, "bin_s", {{jens_row_bytes, true, 0}, {jens_hist_bytes, false, 0}}, {{0, NULL}, {1, NULL}}, 2,
   true, false, true, WIDER, NULL},
  /* DCSIM_STAT_POWER_PROFILE: columns, working state */
  {"power profile", ARG_LIMIT, "threshold_w", {{pp_bytes, false, 0}, {pp_work_bytes, false, 0}}, {{0, NULL}}, 1,
   false, false, false, FEWER, NULL},
  /* DCSIM_STAT_JOB_WAITS: rows, per-replica wait and response histograms */
  {"job waits", ARG_NONE, NULL, {{jwait_row_bytes, true, 0}, {jwait_hist_bytes, false, 0}}, {{0, NULL}, {1, NULL}}, 2,
   false, true, false, WIDER, NULL},
  /* DCSIM_STAT_OCCUPANCY: columns, working state */
  {"occupancy", ARG_NONE, NULL, {{occ_bytes, false, 0}, {occ_work_bytes, false, 0}}, {{0, NULL}}, 1,
   false, false, false, FEWER, NULL},
  /* DCSIM_STAT_TAIL_LATENCY: the slot buffer (NaN: not finished), the columns the selection pass writes; a fetch copies
   * the columns (dcsim_fetch_tail_jobs reads the slots by replica range) */
  {"tail latency", ARG_LIMIT, "sla_s", {{tail_slot_bytes, false, 0xff}, {tail_cols_bytes, false, -1}}, {{1, NULL}}, 1,
   false, false, false, FEWER, tail_ready},
  /* DCSIM_STAT_JOB_RESOURCES: rows, then the counts: the mix, then the energy bins */
  {"job resources", ARG_NONE, NULL, {{jres_row_bytes, true, 0}, {jres_cnt_bytes, false, 0}},
   {{0, NULL}, {1, jres_mix_bytes}, {1, jres_ebin_bytes}}, 3, false, true, false, WIDER, NULL},
  /* DCSIM_STAT_ENERGY_COST: columns, working state */
  {"energy cost", ARG_NONE, NULL, {{cost_bytes, false, 0}, {cost_work_bytes, false, 0}}, {{0, NULL}}, 1,
   false, false, false, FEWER, NULL},
};

static size_t rec_buf_bytes(const dcsim_t* h, int stat, int k) {
  const rec_buf& b = recorder_table[stat].buf[k];
  return (b.per_row ? (size_t)h->rec[stat].rows : 1) * b.bytes(h);
}

static int check_stat(dcsim_t* h, int stat) {
  if (stat >= 0 && stat < DCSIM_STATS) return DCSIM_OK;
  return set_err(h, DCSIM_E_INVALID, "unknown statistic %s%lld (DCSIM_STAT_*)", "", (long long)stat);
}

/* A read of recorder `stat` needs it enabled and the batch advanced. */
static int recorder_ready(dcsim_t* h, int stat) {
  const char* name = recorder_table[stat].name;
  if (!h->rec[stat].d[0]) { snprintf(h->err, sizeof(h->err), "%s not enabled (dcsim_recorder_enable)", name); return DCSIM_E_STATE; }
  if (!h->launches) { snprintf(h->err, sizeof(h->err), "%s read before the first advance", name); return DCSIM_E_STATE; }
  CUDA_TRY(h, cudaSetDevice(h->device));
  return DCSIM_OK;
}

/* ... then the recorder's own read precondition (the tick counts, the tail selection), on the stream ahead of the read:
 * what its fetches and its reductions run first. */
static int recorder_read(dcsim_t* h, int stat) {
  const int rc = recorder_ready(h, stat);
  return rc != DCSIM_OK || !recorder_table[stat].ready ? rc : recorder_table[stat].ready(h);
}

/* The buffers of recorder `stat`, when it is on, filled with their fill bytes on the stream. */
static int recorder_fill(dcsim_t* h, int stat) {
  for (int k = 0; k < 2 && h->rec[stat].d[k]; ++k) {
    const int fill = recorder_table[stat].buf[k].fill;
    if (fill >= 0) CUDA_TRY(h, cudaMemsetAsync(h->rec[stat].d[k], fill, rec_buf_bytes(h, stat, k), h->g->stream));
  }
  return DCSIM_OK;
}

static void recorder_free(dcsim_t* h, int stat) {
  cudaFree(h->rec[stat].d[0]);
  cudaFree(h->rec[stat].d[1]);
  h->rec[stat] = dcsim_slot{};
}

/* Column `field` of every replica's summary row into out[0, n_replicas), their maximum into out[n_replicas]. */
static int summary_counts(dcsim_t* h, int field, uint32_t* out) {
  CUDA_TRY(h, cudaMemsetAsync(out + h->n_replicas, 0, sizeof(uint32_t), h->g->stream));
  int blocks = (int)((h->n_replicas + 255) / 256);
  if (blocks > 4 * h->sm_count) blocks = 4 * h->sm_count;
  dcsim_ens_counts_kernel<<<blocks, 256, 0, h->g->stream>>>(h->d_summary, h->n_replicas, field, out);
  CUDA_TRY(h, cudaGetLastError());
  return DCSIM_OK;
}

/* Before a reduction over recorder `stat` (after recorder_read): every replica's status word into d_status, on
 * the stream, where the reduction that reads it follows.  The cluster ensemble's columns count by the tick counts
 * instead. */
static int status_words(dcsim_t* h, int stat) {
  const int rc = recorder_read(h, stat);
  if (rc != DCSIM_OK || stat == DCSIM_STAT_CLUSTER_ENSEMBLE) return rc;
  return summary_counts(h, DCSIM_S_STATUS, h->d_status);
}

/* Sums the per-replica histogram rows hist[n_replicas][row_len] (without the replicas whose `status` word is not 0, when
 * given) into the device scratch `sum`, then copies that to the host `out`; synchronises. */
static cudaError_t hist_reduce(dcsim_t* h, const uint32_t* hist, uint32_t row_len, const uint32_t* status,
                               unsigned long long* sum, uint64_t* out) {
  const size_t bytes = (size_t)row_len * sizeof(uint64_t);
  cudaError_t e = cudaMemsetAsync(sum, 0, bytes, h->g->stream);
  if (e == cudaSuccess) {
    int blocks = 8 * h->sm_count;
    if ((uint64_t)blocks > h->n_replicas) blocks = (int)h->n_replicas;
    dcsim_hist_reduce_kernel<<<blocks, 2 * DCSIM_LAT_BINS, 0, h->g->stream>>>(hist, h->n_replicas, row_len, status, sum);
    e = cudaGetLastError();
  }
  if (e == cudaSuccess) e = cudaMemcpyAsync(out, sum, bytes, cudaMemcpyDeviceToHost, h->g->stream);
  if (e == cudaSuccess) e = cudaStreamSynchronize(h->g->stream);
  return e;
}

/* The two passes of a batch-wide statistic over the n_cols columns of `src` (n replicas) on the handle's stream: one CTA
 * per column, at most 2^20 CTAs (the kernels stride over the rest). */
static int ens_grid(uint64_t n_cols) { return (int)(n_cols < (1ull << 20) ? n_cols : (1ull << 20)); }

template <class Src>
static int ens_moments(dcsim_t* h, const Src& src, uint64_t n, uint64_t n_cols, double* dev_out) {
  if (!n_cols) return DCSIM_OK;
  dcsim_ens_moments_kernel<<<ens_grid(n_cols), DCSIM_ENS_THREADS, 0, h->g->stream>>>(src, n, n_cols, dev_out);
  CUDA_TRY(h, cudaGetLastError());
  return DCSIM_OK;
}

template <class Src>
static int ens_spread(dcsim_t* h, const Src& src, uint64_t n, uint64_t n_cols, const double* dev_mean, const double* dev_lo,
                      const double* dev_hi, double* dev_m2_out, uint64_t* dev_hist_out) {
  if (!n_cols) return DCSIM_OK;
  dcsim_ens_spread_kernel<<<ens_grid(n_cols), DCSIM_ENS_THREADS, 0, h->g->stream>>>(src, n, n_cols, dev_mean, dev_lo, dev_hi,
                                                                                   dev_m2_out, (unsigned long long*)dev_hist_out);
  CUDA_TRY(h, cudaGetLastError());
  return DCSIM_OK;
}

extern "C" {

size_t dcsim_sizeof_spec(void) { return sizeof(dcsim_spec_t); }
uint32_t dcsim_abi_version(void) { return DCSIM_ABI_VERSION; }
int dcsim_summary_k(void) { return DCSIM_SUMMARY_K; }

#ifdef DCSIM_TEST_HOOKS
/* TEST-ONLY (the library built with -DDCSIM_TEST_HOOKS; not declared in include/dcsim_b200.h, not in the product
 * library): handles created after this call round every arrival and xfer_done instant up to a multiple of q (0 = off),
 * like the oracle's and the host build's hook, so that same-instant events become common on the device.  The quantum
 * reaches the pre-pass and the merge through one __device__ variable, written in stream order by each group's prepare:
 * groups with different quanta must not prepare concurrently. */
static double g_test_time_quantum = 0.0;
int dcsim_test_set_time_quantum(double q) {
  if (!(q >= 0.0 && q <= DBL_MAX)) return set_err(NULL, DCSIM_E_INVALID, "test_set_time_quantum: q must be finite and >= 0%s%lld");
  g_test_time_quantum = q;
  return DCSIM_OK;
}
#endif

static int validate_spec(const dcsim_spec_t* sp) {
  if (sp->magic != DCSIM_SPEC_MAGIC) return set_err(NULL, DCSIM_E_INVALID, "spec: bad magic%s%lld");
  if (sp->abi_version != DCSIM_ABI_VERSION) return set_err(NULL, DCSIM_E_INVALID, "spec: ABI version mismatch%s%lld");
  if (sp->spec_bytes != sizeof(dcsim_spec_t)) return set_err(NULL, DCSIM_E_INVALID, "spec: struct size mismatch (producer says %s%lld bytes)", "", sp->spec_bytes);
  if (sp->n_dc < 1 || sp->n_dc > DCSIM_MAX_DC || sp->n_ing < 1 || sp->n_ing > DCSIM_MAX_ING)
    return set_err(NULL, DCSIM_E_INVALID, "spec: n_dc / n_ing out of range%s%lld");
  if (!(sp->log_interval > 0.0)) return set_err(NULL, DCSIM_E_INVALID, "spec: log_interval must be > 0%s%lld");
  if (sp->policy_name != DCSIM_POLICY_ENERGY_AWARE && sp->policy_name != DCSIM_POLICY_PERF_FIRST)
    return set_err(NULL, DCSIM_E_INVALID, "Unknown policy name%s%lld"); /* policy.py:41 */
  for (int k = 0; k < 2; ++k) {
    const dcsim_arrival_t* a = &sp->arr[k];
    if (a->mode < DCSIM_ARR_OFF || a->mode > DCSIM_ARR_SINUSOID) return set_err(NULL, DCSIM_E_INVALID, "Unknown mode%s%lld"); /* arrivals.py:33 */
    if (a->mode == DCSIM_ARR_SINUSOID && !(a->rate > 0.0 && a->period > 0.0))
      return set_err(NULL, DCSIM_E_INVALID, "sinusoid arrivals need rate > 0 and period > 0%s%lld");
    if (a->mode == DCSIM_ARR_SINUSOID && (a->amp > 1.0 || a->amp < -1.0))
      return set_err(NULL, DCSIM_E_INVALID, "sinusoid arrivals with |amp| > 1 never terminate in the reference (arrivals.py:41-45)%s%lld");
  }
  for (int d = 0; d < sp->n_dc; ++d) {
    const dcsim_dc_t* c = &sp->dc[d];
    if (c->total_gpus < 0 || c->n_freq < 1 || c->n_freq > DCSIM_MAX_FREQ)
      return set_err(NULL, DCSIM_E_INVALID, "spec: DC %s%lld has bad total_gpus / n_freq", "", d);
    if (c->total_gpus > 65535) /* a running record packs the job's GPU count into 16 bits */
      return set_err(NULL, DCSIM_E_INVALID, "spec: DC %s%lld has more than 65535 GPUs", "", d);
  }
  if (sp->cap_arrivals < 0 || (uint32_t)sp->cap_arrivals >= DCSIM_MAX_ARRIVALS)
    return set_err(NULL, DCSIM_E_INVALID, "spec: cap_arrivals must be below 2^24 (%s%lld given)", "", sp->cap_arrivals);
  if (sp->algo < DCSIM_ALGO_DEFAULT || sp->algo > DCSIM_ALGO_CAP_GREEDY)
    return set_err(NULL, DCSIM_E_UNSUPPORTED, "spec: unknown algo id %s%lld", "", sp->algo);
  return DCSIM_OK;
}

/* Launch geometry for the handle's current state-block layout: lanes per replica (32 / 16 / 8), what is staged (whole
 * block / head only / nothing), warps per CTA, shared memory.
 *   DCSIM_GROUP=32|16|8     forces the lanes per replica (default: see pick below);
 *   DCSIM_RECORDS=shared|global forces the whole-block / head-only staging (A/B runs). */
typedef cudaError_t (*dcsim_adv_launch_fn)(const dcsim_kparams_t*, unsigned long long*, int, int, int, int, int, cudaStream_t);
typedef cudaError_t (*dcsim_adv_attrs_fn)(int, int, int, int, int, int*, int*, int*);
static dcsim_adv_launch_fn adv_launch_for(int lanes) { return lanes == 8 ? dcsim_adv_launch_g8 : (lanes == 16 ? dcsim_adv_launch_g16 : dcsim_adv_launch_g32); }
static dcsim_adv_attrs_fn adv_attrs_for(int lanes) { return lanes == 8 ? dcsim_adv_attrs_g8 : (lanes == 16 ? dcsim_adv_attrs_g16 : dcsim_adv_attrs_g32); }
static int min_ctas_for(int lanes) { return lanes == 8 ? dcsim_adv_min_ctas_g8() : (lanes == 16 ? dcsim_adv_min_ctas_g16() : dcsim_adv_min_ctas_g32()); }

static int resident_warps_for(int bytes_per_warp, int smem_optin, int smem_sm, int max_warps, int* wpc_out) {
  /* warps per CTA: whichever of 4 / 2 / 1 keeps the most warps resident (each CTA also reserves 1 KB of shared
   * memory and an SM holds at most 32 CTAs); small state blocks end up at 4 x 8 CTAs, large ones at 1 or 2 */
  int wpc = 0, best_warps = 0;
  for (int cand = DCSIM_MAX_WARPS_PER_CTA; cand >= 1; cand >>= 1) {
    const long long per_cta = (long long)cand * bytes_per_warp;
    if (per_cta > smem_optin) continue;
    int ctas = (int)(smem_sm / (per_cta + 1024));
    if (ctas > 32) ctas = 32;
    int warps = ctas * cand;
    if (warps > max_warps) warps = max_warps; /* register bound */
    if (warps > best_warps) { best_warps = warps; wpc = cand; }
  }
  *wpc_out = wpc;
  return best_warps;
}

static cudaError_t size_launch(dcsim_t* h) {
  cudaError_t e;
  int smem_optin = 0, smem_sm = 0;
  if ((e = cudaDeviceGetAttribute(&smem_optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, h->device)) != cudaSuccess) return e;
  if ((e = cudaDeviceGetAttribute(&smem_sm, cudaDevAttrMaxSharedMemoryPerMultiprocessor, h->device)) != cudaSuccess) return e;
  /* Lanes per replica.  Four replicas per warp share everything warp-wide in an event (pop-min, DC sweep, the lane-0
   * handler's issue slots) and pay whenever the event set fits one round of 8 lanes: up to 5 DCs (n_dc finish slots +
   * list + log + stale).  Above that (8 DC x 256: two slots per lane, all 8 lanes in the sweep) it keeps the whole
   * warp. */
  int lanes = h->spec.n_dc <= 5 ? 8 : 32;
  if (lanes == 8) {
    /* ... unless four blocks per warp leave the SM with hardly more resident REPLICAS than one per warp would (very
     * large heads: the power-cap controller's pools — cap_greedy 4 x 64: 12 vs 14 replicas per SM; the bandit's
     * tables, 52 vs 32, stay on 8 lanes) */
    int w8 = 0, w32 = 0, unused = 0;
    const int bytes8 = 4 * h->L.rec_off, bytes32 = h->L.rec_off; /* head-staged: the smallest footprint of each */
    w8 = resident_warps_for(bytes8, smem_optin, smem_sm, min_ctas_for(8) * DCSIM_MAX_WARPS_PER_CTA, &unused);
    w32 = resident_warps_for(bytes32, smem_optin, smem_sm, min_ctas_for(32) * DCSIM_MAX_WARPS_PER_CTA, &unused);
    if (2 * (4 * w8) < 3 * w32) lanes = 32; /* fewer than 1.5x the replicas per SM */
  }
  { const char* g = getenv("DCSIM_GROUP"); if (g) { const int v = atoi(g); if (v == 8 || v == 16 || v == 32) lanes = v; } }
  const int rpw = 32 / lanes; /* replicas per warp */
  const int max_warps = min_ctas_for(lanes) * DCSIM_MAX_WARPS_PER_CTA;
  int wpc_full = 0, wpc_head = 0;
  const int warps_full = resident_warps_for(rpw * h->L.total_bytes, smem_optin, smem_sm, max_warps, &wpc_full);
  const int warps_head = resident_warps_for(rpw * h->L.rec_off, smem_optin, smem_sm, max_warps, &wpc_head);
  const char* force = getenv("DCSIM_RECORDS");
  int mode, wpc, bytes;
  if (wpc_full >= 1 && (warps_full >= warps_head || (force && force[0] == 's')) && !(force && force[0] == 'g' && wpc_head >= 1)) {
    mode = DCSIM_MODE_STAGED; wpc = wpc_full; bytes = h->L.total_bytes;   /* records staged with the rest */
  } else if (wpc_head >= 1) {
    mode = DCSIM_MODE_HEAD; wpc = wpc_head; bytes = h->L.rec_off;          /* records stay in HBM/L2 */
  } else { /* not even the head fits a CTA's shared memory: run in place out of HBM/L2 */
    mode = DCSIM_MODE_INPLACE; wpc = DCSIM_MAX_WARPS_PER_CTA; bytes = 0;
  }
  h->lanes = lanes;
  h->mode = mode;
  h->warps_per_cta = wpc;
  h->smem_bytes = wpc * rpw * bytes;
  const uint64_t per_cta = (uint64_t)wpc * (uint64_t)rpw;
  h->ctas = (int)((h->n_replicas + per_cta - 1) / per_cta);
  int blocks_per_sm = 0, min_ctas = 0;
  if ((e = adv_attrs_for(lanes)(h->L.cap_stale != 0, h->mode, wpc * 32, h->smem_bytes, smem_optin, &h->regs, &blocks_per_sm, &min_ctas)) != cudaSuccess) return e;
  h->resident_warps = blocks_per_sm * wpc;
  return cudaSuccess;
}

/* job_log.csv and some recorders need job fields in the running records (dcsim_job_fields); switching them on or off
 * re-lays the state block out. */
static int relayout(dcsim_t* h, int job_log) {
  dcsim_layout_t L;
  dcsim_make_layout(&h->spec, &L, dcsim_job_fields(job_log, h->rec[DCSIM_STAT_JOB_WAITS].d[0], h->rec[DCSIM_STAT_TAIL_LATENCY].d[0],
                                                       h->rec[DCSIM_STAT_JOB_RESOURCES].d[0]));
  if (L.lean == h->L.lean) return DCSIM_OK;
  CUDA_TRY(h, cudaStreamSynchronize(h->g->stream));
  h->L = L;
  CUDA_TRY(h, size_launch(h));
  if (h->d_state) { cudaFree(h->d_state); h->d_state = NULL; }
  const size_t state_bytes = (size_t)h->n_replicas * (size_t)h->L.total_bytes;
  CUDA_TRY(h, cudaMalloc(&h->d_state, state_bytes));
  CUDA_TRY(h, cudaMemsetAsync(h->d_state, 0, state_bytes, h->g->stream));
  return DCSIM_OK;
}

static int create_handle(const dcsim_spec_t* sp, dcsim_group* g, int member, dcsim_t** out);

int dcsim_create(const void* spec_blob, size_t spec_bytes, uint64_t n_replicas, uint64_t base_seed,
                 uint64_t first_replica_id, int device, dcsim_t** out) {
  if (!out) return set_err(NULL, DCSIM_E_INVALID, "create: out is NULL%s%lld");
  *out = NULL;
  if (!spec_blob || spec_bytes != sizeof(dcsim_spec_t))
    return set_err(NULL, DCSIM_E_INVALID, "create: spec blob must be %s%lld bytes", "", (long long)sizeof(dcsim_spec_t));
  if (n_replicas == 0) return set_err(NULL, DCSIM_E_INVALID, "create: n_replicas must be > 0%s%lld");
  if (n_replicas > 0xffffffffull) /* the event loop keeps the local replica index in 32 bits */
    return set_err(NULL, DCSIM_E_INVALID, "create: n_replicas must be below 2^32 per handle%s%lld");
  dcsim_spec_t sp;
  memcpy(&sp, spec_blob, sizeof(sp));
  int rc = validate_spec(&sp);
  if (rc != DCSIM_OK) return rc;

  dcsim_group* g = new (std::nothrow) dcsim_group();
  if (!g) return set_err(NULL, DCSIM_E_NOMEM, "create: host allocation failed%s%lld");
  memset(g, 0, sizeof(*g));
  g->refs = 1;
  g->device = device;
  g->spec = sp;
  g->n_replicas = n_replicas;
  g->seed0 = base_seed + first_replica_id;
  g->cap_arr = dcsim_cap_arr(&sp);
#ifdef DCSIM_TEST_HOOKS
  g->test_quantum = g_test_time_quantum;
  g->max_transfer = dcsim_max_transfer(&sp, g->test_quantum);
#else
  g->max_transfer = dcsim_max_transfer(&sp, 0.0);
#endif

#define GROUP_TRY(call)                                                                   \
  do {                                                                                    \
    cudaError_t e_ = (call);                                                              \
    if (e_ != cudaSuccess) {                                                              \
      rc = set_err(NULL, e_ == cudaErrorMemoryAllocation ? DCSIM_E_NOMEM : DCSIM_E_CUDA,  \
                   "CUDA error in create: %s (line %lld)", cudaGetErrorString(e_), (long long)__LINE__); \
      group_release(g);                                                                   \
      return rc;                                                                          \
    }                                                                                     \
  } while (0)

  GROUP_TRY(cudaSetDevice(device));
  GROUP_TRY(cudaStreamCreateWithFlags(&g->own_stream, cudaStreamNonBlocking));
  g->stream = g->own_stream;
  {
    const size_t ne = (size_t)n_replicas * (size_t)g->cap_arr;
    GROUP_TRY(cudaMalloc(&g->d_arr_t, ne * sizeof(double)));
    GROUP_TRY(cudaMalloc(&g->d_arr_raw, ne * sizeof(double)));
    GROUP_TRY(cudaMalloc(&g->d_arr_meta, ne * sizeof(uint32_t)));
    GROUP_TRY(cudaMalloc(&g->d_arr_pred, ne * sizeof(uint32_t)));
    GROUP_TRY(cudaMalloc(&g->d_arr_tx, ne * sizeof(double)));
    GROUP_TRY(cudaMalloc(&g->d_arr_fin, ne * sizeof(uint32_t)));
    GROUP_TRY(cudaMalloc(&g->d_ml_t, 2 * ne * sizeof(double)));
    GROUP_TRY(cudaMalloc(&g->d_ml_aux, 2 * ne * sizeof(double)));
    GROUP_TRY(cudaMalloc(&g->d_ml_meta, 2 * ne * sizeof(uint32_t)));
    GROUP_TRY(cudaMalloc(&g->d_arr_hdr, (size_t)n_replicas * sizeof(dcsim_arrhdr_t)));
  }
#undef GROUP_TRY
  rc = create_handle(&sp, g, /*member=*/0, out);
  group_release(g); /* the handle holds its own reference (or, on failure, none) */
  return rc;
}

/* A handle of group `g` (takes a reference on success): its own state block, queues, summary and scratch. */
static int create_handle(const dcsim_spec_t* sp, dcsim_group* g, int member, dcsim_t** out) {
  int rc = DCSIM_OK;
  dcsim_t* h = new (std::nothrow) dcsim();
  if (!h) return set_err(NULL, DCSIM_E_NOMEM, "create: host allocation failed%s%lld");
  memset(h, 0, sizeof(*h));
  h->spec = *sp;
  dcsim_make_layout(&h->spec, &h->L, /*job_log=*/0);
  h->g = g;
  ++g->refs;
  h->member = member;
  h->generation = g->generation;
  h->n_replicas = g->n_replicas;
  h->device = g->device;
  h->trace_replica = -1;
  h->log_replica = -1;
  const uint64_t n_replicas = h->n_replicas;

#define CREATE_TRY(call)                                                                  \
  do {                                                                                    \
    cudaError_t e_ = (call);                                                              \
    if (e_ != cudaSuccess) {                                                              \
      rc = set_err(NULL, e_ == cudaErrorMemoryAllocation ? DCSIM_E_NOMEM : DCSIM_E_CUDA,  \
                   "CUDA error in create: %s (line %lld)", cudaGetErrorString(e_), (long long)__LINE__); \
      dcsim_destroy(h);                                                                   \
      return rc;                                                                          \
    }                                                                                     \
  } while (0)

  CREATE_TRY(cudaSetDevice(h->device));
  CREATE_TRY(cudaDeviceGetAttribute(&h->sm_count, cudaDevAttrMultiProcessorCount, h->device));
  CREATE_TRY(size_launch(h));
  const size_t state_bytes = (size_t)n_replicas * (size_t)h->L.total_bytes;
  if (h->L.queue_bytes >= (1ull << 32)) /* the event loop addresses inside one replica's FIFOs with 32 bits */
  {
    rc = set_err(NULL, DCSIM_E_INVALID, "create: one replica's FIFO queues exceed 4 GB (cap_q_inf / cap_q_trn too large)%s%lld");
    dcsim_destroy(h);
    return rc;
  }
  const size_t queue_bytes = (size_t)n_replicas * (size_t)h->L.queue_bytes;
  CREATE_TRY(cudaMalloc(&h->d_state, state_bytes));
  CREATE_TRY(cudaMalloc(&h->d_queues, queue_bytes ? queue_bytes : 16));
  CREATE_TRY(cudaMalloc(&h->d_summary, (size_t)n_replicas * DCSIM_SUMMARY_K * sizeof(double)));
  CREATE_TRY(cudaMalloc(&h->d_events, sizeof(unsigned long long)));
  CREATE_TRY(cudaMalloc(&h->d_agg, DCSIM_AGG_K * sizeof(double)));
  CREATE_TRY(cudaMalloc(&h->d_hist_out, 2 * DCSIM_LAT_BINS * sizeof(unsigned long long)));
  CREATE_TRY(cudaMalloc(&h->d_counts, 4 * sizeof(uint32_t)));
  CREATE_TRY(cudaMemsetAsync(h->d_state, 0, state_bytes, h->g->stream)); /* hdr.initialized == 0 => fresh replica */
  CREATE_TRY(cudaMemsetAsync(h->d_summary, 0, (size_t)n_replicas * DCSIM_SUMMARY_K * sizeof(double), h->g->stream));
  CREATE_TRY(cudaMemsetAsync(h->d_events, 0, sizeof(unsigned long long), h->g->stream));
  CREATE_TRY(cudaMemsetAsync(h->d_counts, 0, 4 * sizeof(uint32_t), h->g->stream));
  CREATE_TRY(cudaStreamSynchronize(h->g->stream));
#undef CREATE_TRY
  *out = h;
  return DCSIM_OK;
}

/* A blob of the right size holding a valid spec, copied into *sp. */
static int spec_from_blob(const void* spec_blob, size_t spec_bytes, dcsim_spec_t* sp) {
  if (!spec_blob || spec_bytes != sizeof(dcsim_spec_t))
    return set_err(NULL, DCSIM_E_INVALID, "spec blob must be %s%lld bytes", "", (long long)sizeof(dcsim_spec_t));
  memcpy(sp, spec_blob, sizeof(*sp));
  return validate_spec(sp);
}

int dcsim_arrivals_compatible(const void* spec_a, size_t a_bytes, const void* spec_b, size_t b_bytes, int* equal_out) {
  if (!equal_out) return set_err(NULL, DCSIM_E_INVALID, "arrivals_compatible: equal_out is NULL%s%lld");
  *equal_out = 0;
  dcsim_spec_t a, b;
  int rc = spec_from_blob(spec_a, a_bytes, &a);
  if (rc == DCSIM_OK) rc = spec_from_blob(spec_b, b_bytes, &b);
  if (rc != DCSIM_OK) return DCSIM_E_INVALID;
  *equal_out = dcsim_arrival_inputs_equal(&a, &b) ? 1 : 0;
  return DCSIM_OK;
}

int dcsim_create_shared(const void* spec_blob, size_t spec_bytes, dcsim_t* owner, dcsim_t** out) {
  if (!out) return set_err(NULL, DCSIM_E_INVALID, "create_shared: out is NULL%s%lld");
  *out = NULL;
  if (!owner) return set_err(NULL, DCSIM_E_INVALID, "create_shared: owner is NULL%s%lld");
  if (owner->member) return set_err(NULL, DCSIM_E_INVALID, "create_shared: the owner is itself a member of a group%s%lld");
  dcsim_spec_t sp;
  int rc = spec_from_blob(spec_blob, spec_bytes, &sp);
  if (rc != DCSIM_OK) return rc;
  const char* field = NULL;
  if (!dcsim_arrival_inputs_equal(&owner->g->spec, &sp, &field)) {
    snprintf(g_create_err, sizeof(g_create_err), "create_shared: the spec draws other arrivals than the owner's (%s differs)", field);
    return DCSIM_E_INVALID;
  }
  return create_handle(&sp, owner->g, /*member=*/1, out);
}

int dcsim_reset(dcsim_t* h, uint64_t base_seed, uint64_t first_replica_id) {
  if (!h) return DCSIM_E_INVALID;
  if (h->member && base_seed + first_replica_id != h->g->seed0)
    return set_err(h, DCSIM_E_INVALID, "reset: a member must pass the owner's keys (base_seed + first_replica_id = %s%lld)", "",
                   (long long)h->g->seed0);
  CUDA_TRY(h, cudaSetDevice(h->device));
  /* hdr.initialized == 0 marks a fresh replica; the FIFOs need no clearing (head == tail == 0) */
  CUDA_TRY(h, cudaMemsetAsync(h->d_state, 0, (size_t)h->n_replicas * (size_t)h->L.total_bytes, h->g->stream));
  CUDA_TRY(h, cudaMemsetAsync(h->d_counts, 0, 4 * sizeof(uint32_t), h->g->stream));
  if (h->d_hist) CUDA_TRY(h, cudaMemsetAsync(h->d_hist, 0, (size_t)h->n_replicas * 2 * DCSIM_LAT_BINS * sizeof(uint32_t), h->g->stream));
  for (int s = 0; s < DCSIM_STATS; ++s) {
    const int rc = recorder_fill(h, s);
    if (rc != DCSIM_OK) return rc;
  }
  h->tail_fresh = 0;
  if (!h->member) { /* new keys: the group's lists are redrawn by its next prepare / advance */
    h->g->seed0 = base_seed + first_replica_id;
    h->g->arrivals_ready = 0;
    ++h->g->generation;
  }
  h->generation = h->g->generation;
  h->launches = 0; /* a reset batch is "fresh": recorders may be re-targeted before its first advance */
  return DCSIM_OK;
}

int dcsim_set_stream(dcsim_t* h, void* cuda_stream) {
  if (!h) return DCSIM_E_INVALID;
  if (h->member) return set_err(h, DCSIM_E_STATE, "set_stream on a member: the group's stream is the owner's%s%lld");
  CUDA_TRY(h, cudaSetDevice(h->device));
  CUDA_TRY(h, cudaStreamSynchronize(h->g->stream));
  h->g->stream = cuda_stream ? (cudaStream_t)cuda_stream : h->g->own_stream;
  return DCSIM_OK;
}

int dcsim_set_trace(dcsim_t* h, uint64_t replica, uint32_t capacity) {
  if (!h) return DCSIM_E_INVALID;
  if (h->launches) return set_err(h, DCSIM_E_STATE, "set_trace must precede the first advance%s%lld");
  CUDA_TRY(h, cudaSetDevice(h->device));
  if (h->d_trace) { cudaFree(h->d_trace); h->d_trace = NULL; }
  h->trace_cap = 0; h->trace_replica = -1;
  if (capacity == 0) return DCSIM_OK;
  if (replica >= h->n_replicas) return set_err(h, DCSIM_E_INVALID, "set_trace: replica out of range%s%lld");
  CUDA_TRY(h, cudaMalloc(&h->d_trace, (size_t)capacity * sizeof(dcsim_trace_rec_t)));
  h->trace_cap = capacity; h->trace_replica = (int64_t)replica;
  return DCSIM_OK;
}

int dcsim_set_logging(dcsim_t* h, uint64_t replica, uint32_t job_capacity, uint32_t cluster_capacity) {
  if (!h) return DCSIM_E_INVALID;
  if (h->launches) return set_err(h, DCSIM_E_STATE, "set_logging must precede the first advance%s%lld");
  CUDA_TRY(h, cudaSetDevice(h->device));
  h->jobs_cap = h->cluster_cap = 0; h->log_replica = -1;
  h->want_job_log = 0; /* the state block is re-laid out (if at all) by the batch's first launch: a caller that
                          switches logging off and on again between batches pays for neither */
  if (replica >= h->n_replicas && (job_capacity || cluster_capacity))
    return set_err(h, DCSIM_E_INVALID, "set_logging: replica out of range%s%lld");
  if (job_capacity == 0 && cluster_capacity == 0) return DCSIM_OK;
  if (job_capacity > h->jobs_alloc) { /* buffers only ever grow; a smaller request reuses them */
    if (h->d_jobs) { cudaFree(h->d_jobs); h->d_jobs = NULL; h->jobs_alloc = 0; }
    CUDA_TRY(h, cudaMalloc(&h->d_jobs, (size_t)job_capacity * sizeof(dcsim_job_rec_t)));
    h->jobs_alloc = job_capacity;
  }
  if (cluster_capacity > h->cluster_alloc) {
    if (h->d_cluster) { cudaFree(h->d_cluster); h->d_cluster = NULL; h->cluster_alloc = 0; }
    CUDA_TRY(h, cudaMalloc(&h->d_cluster, (size_t)cluster_capacity * sizeof(dcsim_cluster_rec_t)));
    h->cluster_alloc = cluster_capacity;
  }
  h->jobs_cap = job_capacity; h->cluster_cap = cluster_capacity; h->log_replica = (int64_t)replica;
  h->want_job_log = job_capacity != 0;
  return DCSIM_OK;
}

static void fill_kparams(const dcsim_t* h, dcsim_kparams_t* P, uint64_t max_events) {
  memset(P, 0, sizeof(*P));
  P->spec = h->spec;
  P->L = h->L;
  P->rec.trace = h->d_trace; P->rec.jobs = h->jobs_cap ? h->d_jobs : NULL; P->rec.cluster = h->cluster_cap ? h->d_cluster : NULL; P->rec.counts = h->d_counts;
  P->rec.trace_cap = h->trace_cap; P->rec.jobs_cap = h->jobs_cap; P->rec.cluster_cap = h->cluster_cap;
  P->rec.trace_replica = h->trace_replica; P->rec.log_replica = h->log_replica;
  P->n_replicas = h->n_replicas;
  P->seed0 = h->g->seed0;
  P->max_events = max_events;
  P->state = h->d_state; P->queues = h->d_queues; P->summary = h->d_summary;
  P->arr_t = h->g->d_arr_t; P->arr_raw = h->g->d_arr_raw; P->arr_meta = h->g->d_arr_meta; P->arr_pred = h->g->d_arr_pred;
  P->arr_tx = h->g->d_arr_tx; P->arr_fin = h->g->d_arr_fin;
  P->ml_t = h->g->d_ml_t; P->ml_aux = h->g->d_ml_aux; P->ml_meta = h->g->d_ml_meta;
  P->arr_hdr = h->g->d_arr_hdr; P->cap_arr = h->g->cap_arr;
  P->max_transfer = h->g->max_transfer;
  P->lat_hist = h->d_hist;
  P->mt_state = h->g->d_mt;
  const dcsim_slot* R = h->rec;
  const dcsim_slot &ens = R[DCSIM_STAT_CLUSTER_ENSEMBLE], &jens = R[DCSIM_STAT_JOB_ENSEMBLE], &jres = R[DCSIM_STAT_JOB_RESOURCES];
  P->ens = (double*)ens.d[0]; P->ens_cap = (uint32_t)ens.rows;
  P->jens = (double*)jens.d[0]; P->jens_hist = (uint32_t*)jens.d[1]; P->jens_bin = jens.arg; P->jens_windows = jens.rows ? jens.rows - 1 : 0;
  P->tail = (double*)R[DCSIM_STAT_TAIL_LATENCY].d[0]; P->tail_cols = (double*)R[DCSIM_STAT_TAIL_LATENCY].d[1];
  P->tail_sla = R[DCSIM_STAT_TAIL_LATENCY].arg;
  P->pp = (double*)R[DCSIM_STAT_POWER_PROFILE].d[0]; P->pp_work = (double*)R[DCSIM_STAT_POWER_PROFILE].d[1];
  P->pp_threshold = R[DCSIM_STAT_POWER_PROFILE].arg;
  P->jwait = (double*)R[DCSIM_STAT_JOB_WAITS].d[0]; P->jwait_hist = (uint32_t*)R[DCSIM_STAT_JOB_WAITS].d[1];
  P->occ = (double*)R[DCSIM_STAT_OCCUPANCY].d[0]; P->occ_work = (double*)R[DCSIM_STAT_OCCUPANCY].d[1];
  P->cost = (double*)R[DCSIM_STAT_ENERGY_COST].d[0]; P->cost_work = (double*)R[DCSIM_STAT_ENERGY_COST].d[1];
  P->jres = (double*)jres.d[0]; P->jres_mix = (uint32_t*)jres.d[1];
  P->jres_hist = jres.d[0] ? (uint32_t*)jres.d[1] + jres_mix_cols(h) * h->n_replicas : NULL;
  dcsim_derive_kparams(P);
}

/* A member whose batch was set up for an earlier generation of the group's lists must be reset first. */
static int check_generation(dcsim_t* h) {
  if (h->generation == h->g->generation) return DCSIM_OK;
  return set_err(h, DCSIM_E_STATE, "arrival source was reset: reset this member with the owner's keys%s%lld");
}

int dcsim_prepare(dcsim_t* h) {
  if (!h) return DCSIM_E_INVALID;
  int rc = check_generation(h);
  if (rc != DCSIM_OK) return rc;
  CUDA_TRY(h, cudaSetDevice(h->device));
  if (h->launches == 0) { const int rc0 = relayout(h, h->want_job_log); if (rc0 != DCSIM_OK) return rc0; }
  if (h->g->arrivals_ready) return DCSIM_OK;
  dcsim_kparams_t P;
  fill_kparams(h, &P, 0);
  /* the owner's launch parameters: its spec and the layout it implies (the merge checks the seq ring against it); both
   * give what this handle's would (dcsim_arrival_inputs_equal, dcsim_create_shared) */
  P.spec = h->g->spec;
  dcsim_make_layout(&h->g->spec, &P.L, /*job_log=*/0);
  const int nb = (int)((h->n_replicas + DCSIM_ARRIVALS_THREADS - 1) / DCSIM_ARRIVALS_THREADS);
  const size_t scratch = dcsim_arrivals_scratch_bytes(h->spec.n_ing); /* 52 KB at 8 ingresses: above the 48 KB default */
#ifdef DCSIM_TEST_HOOKS
  CUDA_TRY(h, cudaMemcpyToSymbolAsync(dcsim_test_time_quantum_dev, &h->g->test_quantum, sizeof(double), 0, cudaMemcpyHostToDevice,
                                      h->g->stream));
#endif
  if (h->g->rng_kind == DCSIM_RNG_MT19937) {
    CUDA_TRY(h, cudaFuncSetAttribute(dcsim_arrivals_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)scratch));
    dcsim_arrivals_kernel<true><<<nb, DCSIM_ARRIVALS_THREADS, scratch, h->g->stream>>>(P);
  } else {
    CUDA_TRY(h, cudaFuncSetAttribute(dcsim_arrivals_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)scratch));
    dcsim_arrivals_kernel<false><<<nb, DCSIM_ARRIVALS_THREADS, scratch, h->g->stream>>>(P);
  }
  CUDA_TRY(h, cudaGetLastError());
  const int wpb = DCSIM_MERGE_THREADS / 32;
  dcsim_merge_kernel<<<(int)((h->n_replicas + wpb - 1) / wpb), DCSIM_MERGE_THREADS, 0, h->g->stream>>>(P);
  CUDA_TRY(h, cudaGetLastError());
  h->g->arrivals_ready = 1;
  h->launches += 2;
  return DCSIM_OK;
}

#ifdef DCSIM_TEST_HOOKS
/* TEST-ONLY (hook build only, like dcsim_test_set_time_quantum): fills the group's arrival, merge-scratch, list and
 * header buffers with 0xee bytes, so that an entry the pre-pass or the merge fails to write cannot pass by holding the
 * value an earlier batch left.  Only before the batch's prepare: the lists are read by every later advance. */
int dcsim_test_poison_prepass(dcsim_t* h) {
  if (!h) return DCSIM_E_INVALID;
  if (h->g->arrivals_ready) return set_err(h, DCSIM_E_STATE, "test_poison_prepass: the batch's lists are already drawn%s%lld");
  CUDA_TRY(h, cudaSetDevice(h->device));
  const size_t ne = (size_t)h->g->n_replicas * (size_t)h->g->cap_arr;
  cudaStream_t s = h->g->stream;
  CUDA_TRY(h, cudaMemsetAsync(h->g->d_arr_t, 0xee, ne * sizeof(double), s));
  CUDA_TRY(h, cudaMemsetAsync(h->g->d_arr_raw, 0xee, ne * sizeof(double), s));
  CUDA_TRY(h, cudaMemsetAsync(h->g->d_arr_meta, 0xee, ne * sizeof(uint32_t), s));
  CUDA_TRY(h, cudaMemsetAsync(h->g->d_arr_pred, 0xee, ne * sizeof(uint32_t), s));
  CUDA_TRY(h, cudaMemsetAsync(h->g->d_arr_tx, 0xee, ne * sizeof(double), s));
  CUDA_TRY(h, cudaMemsetAsync(h->g->d_arr_fin, 0xee, ne * sizeof(uint32_t), s));
  CUDA_TRY(h, cudaMemsetAsync(h->g->d_ml_t, 0xee, 2 * ne * sizeof(double), s));
  CUDA_TRY(h, cudaMemsetAsync(h->g->d_ml_aux, 0xee, 2 * ne * sizeof(double), s));
  CUDA_TRY(h, cudaMemsetAsync(h->g->d_ml_meta, 0xee, 2 * ne * sizeof(uint32_t), s));
  CUDA_TRY(h, cudaMemsetAsync(h->g->d_arr_hdr, 0xee, (size_t)h->g->n_replicas * sizeof(dcsim_arrhdr_t), s));
  CUDA_TRY(h, cudaStreamSynchronize(s));
  return DCSIM_OK;
}

/* TEST-ONLY: copies what the pre-pass and the merge left for local replicas [first, first + count) to host arrays in
 * the device layout: arr_t / arr_raw (after the merge: the job sizes) / arr_meta / arr_pred / arr_tx [count][cap_arr],
 * ml_t / ml_aux / ml_meta [count][2 * cap_arr] and the headers [count] (dcsim_arrhdr_t).  A range, because a large
 * batch's lists take tens of GB. */
int dcsim_test_fetch_prepass(dcsim_t* h, uint64_t first, uint64_t count, double* arr_t, double* arr_raw, uint32_t* arr_meta,
                             uint32_t* arr_pred, double* arr_tx, double* ml_t, double* ml_aux, uint32_t* ml_meta, void* hdr) {
  if (!h || !arr_t || !arr_raw || !arr_meta || !arr_pred || !arr_tx || !ml_t || !ml_aux || !ml_meta || !hdr) return DCSIM_E_INVALID;
  if (first > h->g->n_replicas || count > h->g->n_replicas - first)
    return set_err(h, DCSIM_E_INVALID, "test_fetch_prepass: replicas [first, first + count) out of range%s%lld");
  if (!h->g->arrivals_ready) return set_err(h, DCSIM_E_STATE, "test_fetch_prepass: no lists drawn yet (prepare first)%s%lld");
  CUDA_TRY(h, cudaSetDevice(h->device));
  const size_t c = h->g->cap_arr, o = (size_t)first * c, ne = (size_t)count * c;
  cudaStream_t s = h->g->stream;
  CUDA_TRY(h, cudaMemcpyAsync(arr_t, h->g->d_arr_t + o, ne * sizeof(double), cudaMemcpyDeviceToHost, s));
  CUDA_TRY(h, cudaMemcpyAsync(arr_raw, h->g->d_arr_raw + o, ne * sizeof(double), cudaMemcpyDeviceToHost, s));
  CUDA_TRY(h, cudaMemcpyAsync(arr_meta, h->g->d_arr_meta + o, ne * sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
  CUDA_TRY(h, cudaMemcpyAsync(arr_pred, h->g->d_arr_pred + o, ne * sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
  CUDA_TRY(h, cudaMemcpyAsync(arr_tx, h->g->d_arr_tx + o, ne * sizeof(double), cudaMemcpyDeviceToHost, s));
  CUDA_TRY(h, cudaMemcpyAsync(ml_t, h->g->d_ml_t + 2 * o, 2 * ne * sizeof(double), cudaMemcpyDeviceToHost, s));
  CUDA_TRY(h, cudaMemcpyAsync(ml_aux, h->g->d_ml_aux + 2 * o, 2 * ne * sizeof(double), cudaMemcpyDeviceToHost, s));
  CUDA_TRY(h, cudaMemcpyAsync(ml_meta, h->g->d_ml_meta + 2 * o, 2 * ne * sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
  CUDA_TRY(h, cudaMemcpyAsync(hdr, h->g->d_arr_hdr + first, (size_t)count * sizeof(dcsim_arrhdr_t), cudaMemcpyDeviceToHost, s));
  CUDA_TRY(h, cudaStreamSynchronize(s));
  return DCSIM_OK;
}
#endif

int dcsim_advance(dcsim_t* h, uint64_t max_events_per_replica, uint64_t* total_events_out) {
  if (!h) return DCSIM_E_INVALID;
  if (check_generation(h) != DCSIM_OK) return DCSIM_E_STATE;
  CUDA_TRY(h, cudaSetDevice(h->device));
  if (h->launches == 0) { const int rc0 = relayout(h, h->want_job_log); if (rc0 != DCSIM_OK) return rc0; }
  int rc = dcsim_prepare(h); /* once per (re)seeded batch of the group: the arrival lists of all replicas */
  if (rc != DCSIM_OK) return rc;
  dcsim_kparams_t P;
  fill_kparams(h, &P, max_events_per_replica);
  CUDA_TRY(h, adv_launch_for(h->lanes)(&P, h->d_events, h->L.cap_stale != 0, h->mode, h->ctas, h->warps_per_cta * 32, h->smem_bytes, h->g->stream));
  h->launches++;
  h->tail_fresh = 0;
  if (total_events_out) {
    unsigned long long total = 0;
    CUDA_TRY(h, cudaMemcpyAsync(&total, h->d_events, sizeof(total), cudaMemcpyDeviceToHost, h->g->stream));
    CUDA_TRY(h, cudaStreamSynchronize(h->g->stream));
    *total_events_out = (uint64_t)(total - h->events_seen);
    h->events_seen = total;
  }
  return DCSIM_OK;
}

int dcsim_fetch_summary(dcsim_t* h, double* out, size_t out_bytes) {
  if (!h || !out) return DCSIM_E_INVALID;
  const size_t need = (size_t)h->n_replicas * DCSIM_SUMMARY_K * sizeof(double);
  if (out_bytes < need) return set_err(h, DCSIM_E_INVALID, "fetch_summary: buffer too small (need %s%lld bytes)", "", (long long)need);
  if (!h->launches) return set_err(h, DCSIM_E_STATE, "fetch_summary before the first advance%s%lld");
  CUDA_TRY(h, cudaSetDevice(h->device));
  CUDA_TRY(h, cudaMemcpyAsync(out, h->d_summary, need, cudaMemcpyDeviceToHost, h->g->stream));
  CUDA_TRY(h, cudaStreamSynchronize(h->g->stream));
  return DCSIM_OK;
}

int dcsim_fetch_summary_host(dcsim_t* h, const double** host_ptr_out) {
  if (!h || !host_ptr_out) return DCSIM_E_INVALID;
  *host_ptr_out = NULL;
  if (!h->launches) return set_err(h, DCSIM_E_STATE, "fetch_summary_host before the first advance%s%lld");
  CUDA_TRY(h, cudaSetDevice(h->device));
  const size_t need = (size_t)h->n_replicas * DCSIM_SUMMARY_K * sizeof(double);
  if (!h->h_summary_pinned) CUDA_TRY(h, cudaHostAlloc(&h->h_summary_pinned, need, cudaHostAllocDefault));
  CUDA_TRY(h, cudaMemcpyAsync(h->h_summary_pinned, h->d_summary, need, cudaMemcpyDeviceToHost, h->g->stream));
  CUDA_TRY(h, cudaStreamSynchronize(h->g->stream));
  *host_ptr_out = h->h_summary_pinned;
  return DCSIM_OK;
}

int dcsim_summary_device_ptr(dcsim_t* h, void** dev_ptr_out) {
  if (!h || !dev_ptr_out) return DCSIM_E_INVALID;
  *dev_ptr_out = h->d_summary;
  return DCSIM_OK;
}

int dcsim_all_done(dcsim_t* h, int* done_out) {
  if (!h || !done_out) return DCSIM_E_INVALID;
  *done_out = 0;
  if (!h->launches) return DCSIM_OK;
  CUDA_TRY(h, cudaSetDevice(h->device));
  double* agg = h->d_agg; /* allocated once per handle: the chunked-resume loop calls this after every chunk */
  int rc = dcsim_reduce_summary(h, agg);
  double host[DCSIM_AGG_K];
  if (rc == DCSIM_OK) {
    cudaError_t e = cudaMemcpyAsync(host, agg, sizeof(host), cudaMemcpyDeviceToHost, h->g->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(h->g->stream);
    if (e != cudaSuccess) rc = set_err(h, DCSIM_E_CUDA, "CUDA error: %s%lld", cudaGetErrorString(e));
  }
  if (rc != DCSIM_OK) return rc;
  /* a replica that stopped on a capacity overflow never finishes, so "done" = nothing is still running */
  *done_out = host[DCSIM_A_RUNNING] == 0.0;
  return DCSIM_OK;
}

int dcsim_reduce_summary(dcsim_t* h, double* dev_out) {
  if (!h || !dev_out) return DCSIM_E_INVALID;
  if (!h->launches) return set_err(h, DCSIM_E_STATE, "reduce_summary before the first advance%s%lld");
  CUDA_TRY(h, cudaSetDevice(h->device));
  CUDA_TRY(h, cudaMemsetAsync(dev_out, 0, DCSIM_AGG_K * sizeof(double), h->g->stream));
  int blocks = (int)((h->n_replicas + 255) / 256);
  if (blocks > 4 * h->sm_count) blocks = 4 * h->sm_count;
  dcsim_reduce_kernel<<<blocks, 256, 0, h->g->stream>>>(h->d_summary, h->n_replicas, dev_out);
  CUDA_TRY(h, cudaGetLastError());
  return DCSIM_OK;
}

/* The run's only collective for callers that own an NCCL communicator (C / C++ hosts; Python callers use
 * dcsim_reduce_summary + torch.distributed).  NCCL is resolved at run time from whatever the process has loaded (or
 * libnccl.so.2), so the library carries no link-time dependency on a particular NCCL build. */
typedef int (*dcsim_nccl_allreduce_fn)(const void*, void*, size_t, int /*ncclDataType_t*/, int /*ncclRedOp_t*/, void* /*ncclComm_t*/, cudaStream_t);
int dcsim_allreduce_summary(dcsim_t* h, void* nccl_comm, double* out) {
  if (!h || !out) return DCSIM_E_INVALID;
  if (!nccl_comm) return set_err(h, DCSIM_E_INVALID, "allreduce_summary: nccl_comm is NULL%s%lld");
  static dcsim_nccl_allreduce_fn fn = NULL;
  if (!fn) {
    void* sym = dlsym(RTLD_DEFAULT, "ncclAllReduce");
    if (!sym) {
      void* lib = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
      if (lib) sym = dlsym(lib, "ncclAllReduce");
    }
    if (!sym) return set_err(h, DCSIM_E_UNSUPPORTED, "allreduce_summary: no NCCL in this process (ncclAllReduce not found)%s%lld");
    fn = (dcsim_nccl_allreduce_fn)sym;
  }
  int rc = dcsim_reduce_summary(h, h->d_agg);
  if (rc != DCSIM_OK) return rc;
  const int nccl_rc = fn(h->d_agg, h->d_agg, DCSIM_AGG_K, /*ncclFloat64*/ 8, /*ncclSum*/ 0, nccl_comm, h->g->stream);
  if (nccl_rc != 0) return set_err(h, DCSIM_E_CUDA, "allreduce_summary: ncclAllReduce failed with code %s%lld", "", (long long)nccl_rc);
  CUDA_TRY(h, cudaMemcpyAsync(out, h->d_agg, DCSIM_AGG_K * sizeof(double), cudaMemcpyDeviceToHost, h->g->stream));
  CUDA_TRY(h, cudaStreamSynchronize(h->g->stream));
  return DCSIM_OK;
}

int dcsim_set_rng(dcsim_t* h, int rng_kind) {
  if (!h) return DCSIM_E_INVALID;
  if (rng_kind != DCSIM_RNG_PHILOX && rng_kind != DCSIM_RNG_MT19937) return set_err(h, DCSIM_E_INVALID, "set_rng: unknown rng kind %s%lld", "", (long long)rng_kind);
  if (h->member) return set_err(h, DCSIM_E_STATE, "set_rng on a member: the group's RNG kind is the owner's%s%lld");
  if (h->launches || h->g->arrivals_ready) return set_err(h, DCSIM_E_STATE, "set_rng must precede the first advance%s%lld");
  CUDA_TRY(h, cudaSetDevice(h->device));
  if (rng_kind == DCSIM_RNG_MT19937 && !h->g->d_mt)
    CUDA_TRY(h, cudaMalloc(&h->g->d_mt, (size_t)h->n_replicas * DCSIM_MT_N * sizeof(uint32_t)));
  h->g->rng_kind = rng_kind;
  return DCSIM_OK;
}

int dcsim_enable_latency_histogram(dcsim_t* h) {
  if (!h) return DCSIM_E_INVALID;
  if (h->d_hist) return DCSIM_OK;
  if (h->launches) return set_err(h, DCSIM_E_STATE, "enable_latency_histogram must precede the first advance%s%lld");
  CUDA_TRY(h, cudaSetDevice(h->device));
  const size_t bytes = (size_t)h->n_replicas * 2 * DCSIM_LAT_BINS * sizeof(uint32_t);
  CUDA_TRY(h, cudaMalloc(&h->d_hist, bytes));
  CUDA_TRY(h, cudaMemsetAsync(h->d_hist, 0, bytes, h->g->stream));
  return DCSIM_OK;
}

int dcsim_fetch_latency_histogram(dcsim_t* h, uint64_t* out, size_t out_bytes) {
  if (!h || !out) return DCSIM_E_INVALID;
  if (!h->d_hist) return set_err(h, DCSIM_E_STATE, "latency histogram not enabled (dcsim_enable_latency_histogram)%s%lld");
  const size_t need = 2 * DCSIM_LAT_BINS * sizeof(uint64_t);
  if (out_bytes < need) return set_err(h, DCSIM_E_INVALID, "fetch_latency_histogram: buffer too small (need %s%lld bytes)", "", (long long)need);
  if (!h->launches) return set_err(h, DCSIM_E_STATE, "fetch_latency_histogram before the first advance%s%lld");
  CUDA_TRY(h, cudaSetDevice(h->device));
  const cudaError_t e = hist_reduce(h, h->d_hist, 2 * DCSIM_LAT_BINS, NULL, h->d_hist_out, out);
  if (e != cudaSuccess) return set_err(h, DCSIM_E_CUDA, "CUDA error: %s%lld", cudaGetErrorString(e));
  return DCSIM_OK;
}

extern "C++" {
/* The cluster ensemble's read precondition: every replica's recorded tick count into d_ens_nlog; fails when one of them
 * went past the capacity (synchronises). */
static int ens_counts(dcsim_t* h) {
  const int rc = summary_counts(h, DCSIM_S_EV_LOG, h->d_ens_nlog);
  if (rc != DCSIM_OK) return rc;
  uint32_t most = 0u;
  CUDA_TRY(h, cudaMemcpyAsync(&most, h->d_ens_nlog + h->n_replicas, sizeof(most), cudaMemcpyDeviceToHost, h->g->stream));
  CUDA_TRY(h, cudaStreamSynchronize(h->g->stream));
  const uint32_t cap = (uint32_t)h->rec[DCSIM_STAT_CLUSTER_ENSEMBLE].rows;
  if (most > cap) {
    snprintf(h->err, sizeof(h->err), "cluster ensemble overflow: a replica recorded %u log ticks, capacity %u", most, cap);
    return DCSIM_E_STATE;
  }
  return DCSIM_OK;
}

/* The tail recorder's read precondition: the columns of the finished batch, selected once per batch on the stream. */
static int tail_ready(dcsim_t* h) {
  if (h->tail_fresh) return DCSIM_OK;
  int done = 0, rc;
  if ((rc = dcsim_all_done(h, &done)) != DCSIM_OK) return rc;
  if (!done) return set_err(h, DCSIM_E_STATE, "tail latency read while replicas are still running (advance to the end first)%s%lld");
  dcsim_kparams_t P;
  fill_kparams(h, &P, 0);
  const uint64_t per_sm = 8; /* 256 threads and 18 KB each: 8 CTAs fit an SM */
  const uint64_t grid = h->n_replicas < per_sm * (uint64_t)h->sm_count ? h->n_replicas : per_sm * (uint64_t)h->sm_count;
  dcsim_tail_select_kernel<<<(int)grid, DCSIM_TAIL_THREADS, 0, h->g->stream>>>(P);
  CUDA_TRY(h, cudaGetLastError());
  h->tail_fresh = 1;
  return DCSIM_OK;
}
} /* extern "C++" */

static int pair_check(dcsim_t* base, const double* dev_variant_summary, uint64_t n) {
  if (!base || !dev_variant_summary) return DCSIM_E_INVALID;
  if (n != base->n_replicas)
    return set_err(base, DCSIM_E_INVALID, "paired reduction: n must be the base handle's replica count (%s%lld)", "", (long long)base->n_replicas);
  if (!base->launches) return set_err(base, DCSIM_E_STATE, "paired reduction before the base handle's first advance%s%lld");
  CUDA_TRY(base, cudaSetDevice(base->device));
  return DCSIM_OK;
}

static uint64_t pair_cols(const dcsim_t* h) { return (uint64_t)(DCSIM_PAIR_DC_ENERGY_J + h->spec.n_dc) * DCSIM_PAIR_FIELDS; }

int dcsim_paired_moments(dcsim_t* base, const double* dev_variant_summary, uint64_t n, double* dev_out) {
  if (!dev_out) return DCSIM_E_INVALID;
  const int rc = pair_check(base, dev_variant_summary, n);
  if (rc != DCSIM_OK) return rc;
  const dcsim_ens_pair_src src{base->d_summary, dev_variant_summary, base->spec.n_dc};
  return ens_moments(base, src, n, pair_cols(base), dev_out);
}

int dcsim_paired_spread(dcsim_t* base, const double* dev_variant_summary, uint64_t n, const double* dev_mean,
                        const double* dev_lo, const double* dev_hi, double* dev_m2_out, uint64_t* dev_hist_out) {
  if (!dev_mean || !dev_lo || !dev_hi || !dev_m2_out || !dev_hist_out) return DCSIM_E_INVALID;
  const int rc = pair_check(base, dev_variant_summary, n);
  if (rc != DCSIM_OK) return rc;
  const dcsim_ens_pair_src src{base->d_summary, dev_variant_summary, base->spec.n_dc};
  return ens_spread(base, src, n, pair_cols(base), dev_mean, dev_lo, dev_hi, dev_m2_out, dev_hist_out);
}

extern "C++" {
static int enable_err(dcsim_t* h, int code, int stat, const char* a, const char* b = "") {
  snprintf(h->err, sizeof(h->err), "enable %s: %s%s", recorder_table[stat].name, a, b);
  return code;
}

/* The histogram scratch of recorder `stat` (NULL: it has no histogram), and the length of one replica's row of the
 * per-replica histograms, its second buffer [n_replicas][row_len] u32. */
static unsigned long long** hist_scratch(dcsim_t* h, int stat) {
  return stat == DCSIM_STAT_JOB_ENSEMBLE ? &h->d_jens_hist_out : (stat == DCSIM_STAT_JOB_WAITS ? &h->d_jwait_hist_out : NULL);
}
static uint32_t hist_row_len(const dcsim_t* h, int stat) {
  return (uint32_t)(recorder_table[stat].buf[1].bytes(h) / ((size_t)h->n_replicas * sizeof(uint32_t)));
}

/* The buffers of recorder `stat` for its rows, all or none.  Running out of device memory is DCSIM_E_NOMEM with `need`
 * bytes in the message, and clears the sticky error: the handle stays usable. */
static int recorder_alloc(dcsim_t* h, int stat, long long need) {
  const rec_desc& R = recorder_table[stat];
  dcsim_slot& S = h->rec[stat];
  cudaError_t e = cudaSuccess;
  for (int k = 0; k < 2 && R.buf[k].bytes; ++k) {
    const size_t bytes = rec_buf_bytes(h, stat, k);
    e = cudaMalloc(&S.d[k], bytes ? bytes : sizeof(double)); /* a cluster ensemble of no tick is on all the same */
    if (e != cudaSuccess) { S.d[k] = NULL; break; }
  }
  if (e == cudaSuccess) return DCSIM_OK;
  recorder_free(h, stat);
  if (e != cudaErrorMemoryAllocation) return set_err(h, DCSIM_E_CUDA, "CUDA error: %s%lld", cudaGetErrorString(e));
  cudaGetLastError();
  snprintf(h->err, sizeof(h->err), "enable %s: %lld bytes of device memory do not fit (%s)", R.name, need, R.nomem_hint);
  return DCSIM_E_NOMEM;
}

/* Bytes of part `part` of recorder `stat`'s fetch, and where in its buffer it starts. */
static size_t part_bytes(const dcsim_t* h, int stat, int part) {
  const rec_part& p = recorder_table[stat].part[part];
  return p.bytes ? p.bytes(h) : rec_buf_bytes(h, stat, p.buf);
}
static size_t part_offset(const dcsim_t* h, int stat, int part) {
  size_t off = 0;
  for (int q = 0; q < part; ++q)
    if (recorder_table[stat].part[q].buf == recorder_table[stat].part[part].buf) off += part_bytes(h, stat, q);
  return off;
}
} /* extern "C++" */

int dcsim_recorder_enable(dcsim_t* h, int stat, double arg) {
  if (!h) return DCSIM_E_INVALID;
  int rc = check_stat(h, stat);
  if (rc != DCSIM_OK) return rc;
  const rec_desc& R = recorder_table[stat];
  dcsim_slot& S = h->rec[stat];
  double val = 0.0; /* the resolved argument */
  uint64_t rows = 1;
  switch (R.arg) {
    case ARG_TICKS:
      if (!(arg >= 0.0 && arg <= 4294967295.0 && arg == floor(arg)))
        return enable_err(h, DCSIM_E_INVALID, stat, R.arg_name, " must be a whole number in [0, 2^32)");
      rows = arg > 0.0 ? (uint64_t)arg : dcsim_ens_ticks(&h->spec);
      break;
    case ARG_BIN:
      if (!(arg >= 0.0 && arg <= DBL_MAX)) return enable_err(h, DCSIM_E_INVALID, stat, R.arg_name, " must be finite and >= 0");
      val = arg > 0.0 ? arg : h->spec.log_interval;
      rows = dcsim_jens_windows(h->spec.end_time, val) + 1;
      break;
    case ARG_LIMIT:
      if (!(arg >= 0.0)) return enable_err(h, DCSIM_E_INVALID, stat, R.arg_name, " must be >= 0 (+inf: none)");
      val = arg;
      break;
  }
  if (R.needs_jens) {
    if (!h->rec[DCSIM_STAT_JOB_ENSEMBLE].d[0]) return enable_err(h, DCSIM_E_STATE, stat, "needs the job ensemble (enable it first)");
    rows = h->rec[DCSIM_STAT_JOB_ENSEMBLE].rows;
  }
  if (h->member && !R.member_ok) return enable_err(h, DCSIM_E_STATE, stat, "not on a member of a shared group");
  if (R.retarget && S.d[0] && S.rows == rows && S.arg == val) return DCSIM_OK;
  if (h->launches) return enable_err(h, DCSIM_E_STATE, stat, "must precede the first advance");
  CUDA_TRY(h, cudaSetDevice(h->device));
  if (R.retarget) { /* other rows: new buffers, and none for the recorders that live in the job ensemble's rows */
    recorder_free(h, stat);
    for (int s = 0; s < DCSIM_STATS; ++s)
      if (stat == DCSIM_STAT_JOB_ENSEMBLE && recorder_table[s].needs_jens) recorder_free(h, s);
  }
  if (!S.d[0]) {
    double need = 0.0; /* in double: a narrow bin_s asks for more than size_t holds */
    for (int k = 0; k < 2 && R.buf[k].bytes; ++k) need += (R.buf[k].per_row ? (double)rows : 1.0) * (double)R.buf[k].bytes(h);
    const long long need_ll = need < 9.0e18 ? (long long)need : 9000000000000000000ll;
    if (rows > 0xffffffffull || need >= 9.0e18) { /* W capped by dcsim_jens_windows, or past any device */
      snprintf(h->err, sizeof(h->err), "enable %s: %lld bytes of device memory do not fit (%s)", R.name, need_ll, R.nomem_hint);
      return DCSIM_E_NOMEM;
    }
    uint32_t** words = stat == DCSIM_STAT_CLUSTER_ENSEMBLE ? &h->d_ens_nlog : &h->d_status;
    if (!*words) CUDA_TRY(h, cudaMalloc(words, ((size_t)h->n_replicas + 1) * sizeof(uint32_t)));
    unsigned long long** hist = hist_scratch(h, stat);
    if (hist && !*hist) CUDA_TRY(h, cudaMalloc(hist, (size_t)hist_row_len(h, stat) * sizeof(unsigned long long)));
    S.rows = rows;
    if ((rc = recorder_alloc(h, stat, need_ll)) != DCSIM_OK) return rc;
  }
  S.arg = val;
  return recorder_fill(h, stat);
}

int dcsim_recorder_state(dcsim_t* h, int stat, dcsim_recorder_state_t* out) {
  if (!h || !out) return DCSIM_E_INVALID;
  const int rc = check_stat(h, stat);
  if (rc != DCSIM_OK) return rc;
  const dcsim_slot& S = h->rec[stat];
  memset(out, 0, sizeof(*out));
  out->on = S.d[0] != NULL;
  out->parts = recorder_table[stat].parts;
  out->arg = S.arg;
  out->rows = S.rows;
  for (int p = 0; out->on && p < out->parts; ++p) out->part_bytes[p] = part_bytes(h, stat, p);
  return DCSIM_OK;
}

int dcsim_recorder_fetch(dcsim_t* h, int stat, int part, void* out, size_t out_bytes) {
  if (!h || !out) return DCSIM_E_INVALID;
  int rc = check_stat(h, stat);
  if (rc != DCSIM_OK) return rc;
  if (part < 0 || part >= recorder_table[stat].parts)
    return set_err(h, DCSIM_E_INVALID, "recorder_fetch: no part %s%lld of this recorder", "", (long long)part);
  if ((rc = recorder_read(h, stat)) != DCSIM_OK) return rc;
  size_t bytes = part_bytes(h, stat, part);
  if (stat == DCSIM_STAT_CLUSTER_ENSEMBLE) { /* the whole ticks that fit, at most the capacity */
    const uint64_t tick = ens_tick_bytes(h), ticks = out_bytes / tick;
    bytes = (size_t)((ticks < h->rec[stat].rows ? ticks : h->rec[stat].rows) * tick);
  } else if (out_bytes < bytes) {
    return set_err(h, DCSIM_E_INVALID, "recorder_fetch: buffer too small (need %s%lld bytes)", "", (long long)bytes);
  }
  if (!bytes) return DCSIM_OK;
  const char* src = (const char*)h->rec[stat].d[recorder_table[stat].part[part].buf] + part_offset(h, stat, part);
  CUDA_TRY(h, cudaMemcpyAsync(out, src, bytes, cudaMemcpyDeviceToHost, h->g->stream));
  CUDA_TRY(h, cudaStreamSynchronize(h->g->stream));
  return DCSIM_OK;
}

int dcsim_recorder_histogram(dcsim_t* h, int stat, uint64_t* out, size_t out_bytes) {
  if (!h || !out) return DCSIM_E_INVALID;
  int rc = check_stat(h, stat);
  if (rc != DCSIM_OK) return rc;
  unsigned long long** sum = hist_scratch(h, stat);
  if (!sum) return set_err(h, DCSIM_E_INVALID, "recorder_histogram: statistic %s%lld has no histogram", "", (long long)stat);
  const uint32_t row_len = hist_row_len(h, stat);
  const size_t need = (size_t)row_len * sizeof(uint64_t);
  if (out_bytes < need) return set_err(h, DCSIM_E_INVALID, "recorder_histogram: buffer too small (need %s%lld bytes)", "", (long long)need);
  if ((rc = status_words(h, stat)) != DCSIM_OK) return rc;
  CUDA_TRY(h, hist_reduce(h, (const uint32_t*)h->rec[stat].d[1], row_len, h->d_status, *sum, out));
  return DCSIM_OK;
}

int dcsim_power_profile_range(dcsim_t* h, double* hi_out) {
  if (!h || !hi_out) return DCSIM_E_INVALID;
  *hi_out = dcsim_pp_range(&h->spec);
  return DCSIM_OK;
}

int dcsim_fetch_tail_jobs(dcsim_t* h, uint64_t first, uint64_t count, double* out, size_t out_bytes) {
  if (!h || !out) return DCSIM_E_INVALID;
  if (first > h->n_replicas || count > h->n_replicas - first)
    return set_err(h, DCSIM_E_INVALID, "fetch_tail_jobs: replicas [first, first + count) out of range%s%lld");
  const int rc = recorder_ready(h, DCSIM_STAT_TAIL_LATENCY);
  if (rc != DCSIM_OK) return rc;
  const size_t per = (size_t)h->g->cap_arr * 2, need = (size_t)count * per * sizeof(double);
  if (out_bytes < need)
    return set_err(h, DCSIM_E_INVALID, "fetch_tail_jobs: buffer too small (need %s%lld bytes)", "", (long long)need);
  CUDA_TRY(h, cudaMemcpyAsync(out, (const double*)h->rec[DCSIM_STAT_TAIL_LATENCY].d[0] + (size_t)first * per, need,
                              cudaMemcpyDeviceToHost, h->g->stream));
  CUDA_TRY(h, cudaStreamSynchronize(h->g->stream));
  return DCSIM_OK;
}

int dcsim_occupancy_bin_widths(dcsim_t* h, int32_t* w_out) {
  if (!h || !w_out) return DCSIM_E_INVALID;
  for (int d = 0; d < h->spec.n_dc; ++d) w_out[d] = DCSIM_OCC_BUSY_WIDTH(h->spec.dc[d].total_gpus);
  return DCSIM_OK;
}

extern "C++" {
/* The batch recorder `stat` (DCSIM_STAT_*) as the two passes see it: f(src, columns, spread_columns) with its column
 * source and column counts for the handle's current state.  With `ready`, status_words runs first: it fails when the
 * recorder is off or the batch has not advanced, and queues what the source reads (the tick counts, the status words,
 * the tail selection) on the stream ahead of the pass.  Without it this is host arithmetic only. */
template <class F>
static int with_stat(dcsim_t* h, int stat, bool ready, F&& f) {
  int rc = check_stat(h, stat);
  if (rc != DCSIM_OK || (ready && (rc = status_words(h, stat)) != DCSIM_OK)) return rc;
  const int n_dc = h->spec.n_dc;
  const uint32_t cells = 2u * (uint32_t)n_dc;
  const dcsim_slot* R = h->rec;
  const double* jens = (const double*)R[DCSIM_STAT_JOB_ENSEMBLE].d[0];
  const uint64_t rows = jens ? R[DCSIM_STAT_JOB_ENSEMBLE].rows : 1; /* the job ensemble's windows, then the whole run */
  const dcsim_slot& S = R[stat];
  switch (stat) {
    case DCSIM_STAT_CLUSTER_ENSEMBLE: {
      const uint32_t cols_per_tick = DCSIM_ENS_FIELDS * (uint32_t)n_dc;
      const uint64_t cols = S.rows * cols_per_tick;
      return f(dcsim_ens_cluster_src{(const double*)S.d[0], h->d_ens_nlog, h->n_replicas, cols_per_tick, n_dc}, cols, cols);
    }
    case DCSIM_STAT_JOB_ENSEMBLE: {
      const uint64_t cols = rows * DCSIM_JENS_FIELDS * cells;
      return f(dcsim_ens_job_src{jens, h->d_status, h->n_replicas, cells}, cols, cols);
    }
    case DCSIM_STAT_POWER_PROFILE:
      return f(dcsim_ens_pp_src{(const double*)S.d[0], h->d_status, h->n_replicas}, pp_cols(h), (uint64_t)(DCSIM_PP_FIELDS + n_dc));
    case DCSIM_STAT_JOB_WAITS: {
      const uint64_t cols = rows * DCSIM_JWAIT_FIELDS * cells;
      return f(dcsim_ens_wait_src{(const double*)S.d[0], jens, h->d_status, h->n_replicas, cells}, cols, cols);
    }
    case DCSIM_STAT_OCCUPANCY:
      return f(dcsim_ens_occ_src{(const double*)S.d[0], h->d_status, h->n_replicas, (uint32_t)occ_stat_cols(h), (uint32_t)n_dc},
               occ_cols(h), occ_stat_cols(h));
    case DCSIM_STAT_TAIL_LATENCY: {
      const uint32_t group_cols = 2u * (uint32_t)(n_dc + 1) * DCSIM_TAIL_GROUP_FIELDS;
      const uint64_t cols = DCSIM_TAIL_COLS(n_dc);
      return f(dcsim_ens_tail_src{(const double*)S.d[1], h->d_status, h->n_replicas, group_cols}, cols, cols);
    }
    case DCSIM_STAT_JOB_RESOURCES: {
      const uint64_t win_cols = rows * DCSIM_JRES_FIELDS * cells; /* the counts after them need no spread */
      return f(dcsim_ens_res_src{(const double*)S.d[0], jens, (const uint32_t*)S.d[1], h->d_status, h->n_replicas, cells, win_cols},
               win_cols + jres_mix_cols(h) + jres_hist_cols(h), win_cols);
    }
    default: /* DCSIM_STAT_ENERGY_COST */
      return f(dcsim_ens_cost_src{(const double*)S.d[0], h->d_status, h->n_replicas}, cost_cols(h), cost_cols(h));
  }
}
} /* extern "C++" */

int dcsim_stat_columns(dcsim_t* h, int stat, uint64_t* columns_out, uint64_t* spread_columns_out) {
  if (!h || !columns_out || !spread_columns_out) return DCSIM_E_INVALID;
  return with_stat(h, stat, false, [&](const auto&, uint64_t cols, uint64_t spread_cols) {
    *columns_out = cols;
    *spread_columns_out = spread_cols;
    return DCSIM_OK;
  });
}

int dcsim_stat_moments(dcsim_t* h, int stat, double* dev_out) {
  if (!h || !dev_out) return DCSIM_E_INVALID;
  return with_stat(h, stat, true, [&](const auto& src, uint64_t cols, uint64_t) {
    return ens_moments(h, src, h->n_replicas, cols, dev_out);
  });
}

int dcsim_stat_spread(dcsim_t* h, int stat, const double* dev_mean, const double* dev_lo, const double* dev_hi,
                      double* dev_m2_out, uint64_t* dev_hist_out) {
  if (!h || !dev_mean || !dev_lo || !dev_hi || !dev_m2_out || !dev_hist_out) return DCSIM_E_INVALID;
  return with_stat(h, stat, true, [&](const auto& src, uint64_t, uint64_t spread_cols) {
    return ens_spread(h, src, h->n_replicas, spread_cols, dev_mean, dev_lo, dev_hi, dev_m2_out, dev_hist_out);
  });
}

int dcsim_recorder_counts(dcsim_t* h, uint32_t* out3) {
  if (!h || !out3) return DCSIM_E_INVALID;
  CUDA_TRY(h, cudaSetDevice(h->device));
  uint32_t counts[4];
  CUDA_TRY(h, cudaMemcpyAsync(counts, h->d_counts, sizeof(counts), cudaMemcpyDeviceToHost, h->g->stream));
  CUDA_TRY(h, cudaStreamSynchronize(h->g->stream));
  out3[0] = counts[0]; out3[1] = counts[1]; out3[2] = counts[2];
  return DCSIM_OK;
}

static int fetch_records(dcsim_t* h, const void* dev, size_t rec_bytes, uint32_t dev_cap, int which, void* out,
                         uint32_t capacity, uint32_t* n_out) {
  if (!h || !n_out) return DCSIM_E_INVALID;
  *n_out = 0;
  if (!dev) return DCSIM_OK;
  CUDA_TRY(h, cudaSetDevice(h->device));
  uint32_t counts[4];
  CUDA_TRY(h, cudaMemcpyAsync(counts, h->d_counts, sizeof(counts), cudaMemcpyDeviceToHost, h->g->stream));
  CUDA_TRY(h, cudaStreamSynchronize(h->g->stream));
  uint32_t n = counts[which] < dev_cap ? counts[which] : dev_cap;
  if (n > capacity) n = capacity;
  if (n && out) {
    CUDA_TRY(h, cudaMemcpyAsync(out, dev, (size_t)n * rec_bytes, cudaMemcpyDeviceToHost, h->g->stream));
    CUDA_TRY(h, cudaStreamSynchronize(h->g->stream));
  }
  *n_out = n;
  return DCSIM_OK;
}

int dcsim_fetch_trace(dcsim_t* h, dcsim_trace_rec_t* out, uint32_t capacity, uint32_t* n_out) {
  return fetch_records(h, h ? h->d_trace : NULL, sizeof(dcsim_trace_rec_t), h ? h->trace_cap : 0, 0, out, capacity, n_out);
}
int dcsim_fetch_job_log(dcsim_t* h, dcsim_job_rec_t* out, uint32_t capacity, uint32_t* n_out) {
  return fetch_records(h, h && h->jobs_cap ? h->d_jobs : NULL, sizeof(dcsim_job_rec_t), h ? h->jobs_cap : 0, 1, out, capacity, n_out);
}
int dcsim_fetch_cluster_log(dcsim_t* h, dcsim_cluster_rec_t* out, uint32_t capacity, uint32_t* n_out) {
  return fetch_records(h, h && h->cluster_cap ? h->d_cluster : NULL, sizeof(dcsim_cluster_rec_t), h ? h->cluster_cap : 0, 2, out, capacity, n_out);
}

int dcsim_launch_info(dcsim_t* h, dcsim_launch_info_t* out) {
  if (!h || !out) return DCSIM_E_INVALID;
  memset(out, 0, sizeof(*out));
  out->warps_per_cta = h->warps_per_cta; out->ctas = h->ctas; out->smem_bytes_per_cta = h->smem_bytes;
  out->regs_per_thread = h->regs; out->resident_warps_per_sm = h->resident_warps; out->sm_count = h->sm_count;
  out->cap_xfer = (h->L.xring_mask + 1) / 2; out->cap_run = h->L.cap_run; out->cap_q_inf = h->L.cap_q[0]; out->cap_q_trn = h->L.cap_q[1];
  out->kernel_launches = h->launches;
  out->hbm_bytes_state = (uint64_t)h->n_replicas * (uint64_t)h->L.total_bytes;
  out->hbm_bytes_queues = (uint64_t)h->n_replicas * h->L.queue_bytes;
  out->arrivals_prepass = 1;
  /* per arrival: pre-pass output 24 B + merge scratch 12 B + two list entries of 20 B */
  out->hbm_bytes_arrivals = h->member ? 0ull : (uint64_t)h->n_replicas * ((uint64_t)h->g->cap_arr * 76ull + sizeof(dcsim_arrhdr_t));
  out->staging_mode = h->mode; out->state_block_bytes = h->L.total_bytes;
  out->staged_bytes_per_replica = h->warps_per_cta ? h->smem_bytes / (h->warps_per_cta * (32 / h->lanes)) : 0;
  out->lanes_per_replica = h->lanes;
  return DCSIM_OK;
}

const char* dcsim_last_error(const dcsim_t* h) { return h ? h->err : g_create_err; }

void dcsim_destroy(dcsim_t* h) {
  if (!h) return;
  cudaSetDevice(h->device);
  if (h->g && h->g->stream) cudaStreamSynchronize(h->g->stream);
  cudaFree(h->d_state); cudaFree(h->d_queues); cudaFree(h->d_summary); cudaFree(h->d_events); cudaFree(h->d_counts);
  cudaFree(h->d_trace); cudaFree(h->d_jobs); cudaFree(h->d_cluster);
  cudaFree(h->d_hist); cudaFree(h->d_agg); cudaFree(h->d_hist_out);
  if (h->h_summary_pinned) cudaFreeHost(h->h_summary_pinned);
  for (int s = 0; s < DCSIM_STATS; ++s) recorder_free(h, s);
  cudaFree(h->d_ens_nlog); cudaFree(h->d_jens_hist_out); cudaFree(h->d_jwait_hist_out); cudaFree(h->d_status);
  group_release(h->g); /* the arrival lists and the stream go with the group's last handle */
  delete h;
}

} /* extern "C" */
