/*
 * dcsim_b200.h — C-ABI of the H100-native batched discrete-event engine.
 *
 * The reference (filrg/distributed_cluster_GPUs) has no FFI: its seam is the Python constructor
 * MultiIngressPaperSimulator(...) (simcore/simulator_paper_multi.py:31-55) followed by .run()
 * (simcore/simulator_paper_multi.py:412), called from run_sim_paper.py:143-159.  This header is what a
 * ctypes binding of that seam talks to: plain pointers and sizes, int return codes, no torch/C++ types.
 *
 * Ownership / threading
 *   - host buffers are caller-owned; device memory is library-owned;
 *   - one handle <-> one CUDA device <-> one stream; calls on one handle are not thread-safe,
 *     distinct handles are independent;
 *   - nothing throws across the boundary: every entry point returns DCSIM_OK or a negative code and
 *     dcsim_last_error() returns the message.
 */
#ifndef DCSIM_B200_H
#define DCSIM_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define DCSIM_ABI_VERSION 2u
#define DCSIM_SPEC_MAGIC 0x3130304244435344ull /* "DSCDB001" */

#define DCSIM_MAX_DC 8    /* reference ships 8 DCs: configs/paper_config.py:39-64 */
#define DCSIM_MAX_ING 8   /* and 8 ingresses: configs/paper_config.py:184-193 */
#define DCSIM_MAX_FREQ 16 /* reference uses 8 levels: configs/paper_config.py:41 */
#define DCSIM_HOURS 24

/* ---- return codes ------------------------------------------------------------------------- */
enum {
  DCSIM_OK = 0,
  DCSIM_E_INVALID = -1,  /* bad argument / malformed spec (reference: ValueError arrivals.py:33,48, policy.py:41) */
  DCSIM_E_CUDA = -2,     /* CUDA runtime failure */
  DCSIM_E_NOMEM = -3,    /* device or host allocation failed */
  DCSIM_E_STATE = -4,    /* call order violated (e.g. fetch before advance) */
  DCSIM_E_UNSUPPORTED = -5 /* algo outside the accelerated path (chsac_af: simulator_paper_multi.py:555-573) */
};

/* ---- enumerations mirrored from the reference's string-typed knobs ------------------------- */
enum { DCSIM_JT_INFERENCE = 0, DCSIM_JT_TRAINING = 1 };             /* Job.jtype, models.py:9 */
enum { DCSIM_ARR_OFF = 0, DCSIM_ARR_POISSON = 1, DCSIM_ARR_SINUSOID = 2 }; /* ArrivalConfig.mode, arrivals.py:20 */
enum { DCSIM_POLICY_ENERGY_AWARE = 0, DCSIM_POLICY_PERF_FIRST = 1 };    /* PolicyConfig.name, policy.py:7 */
enum {                                                               /* --algo, run_sim_paper.py:78-84 */
  DCSIM_ALGO_DEFAULT = 0,
  DCSIM_ALGO_JOINT_NF = 1,
  DCSIM_ALGO_CARBON_COST = 2,
  DCSIM_ALGO_ECO_ROUTE = 3,
  DCSIM_ALGO_DEBUG = 4,
  DCSIM_ALGO_BANDIT = 5,
  DCSIM_ALGO_CAP_UNIFORM = 6,
  DCSIM_ALGO_CAP_GREEDY = 7
};
/* device-side start rules the host derives from algo (the C oracle ignores these and follows algo) */
enum { DCSIM_ROUTE_RANDOM = 0, DCSIM_ROUTE_ECO = 1 };                 /* simulator_paper_multi.py:544-577 */
enum { DCSIM_START_POLICY = 0, DCSIM_START_NF_LUT = 1, DCSIM_START_BANDIT = 2 }; /* :603-676 / :892-927 */
enum { DCSIM_RNG_PHILOX = 0, DCSIM_RNG_MT19937 = 1 };                 /* oracle only; the GPU is Philox-only */

/* ---- spec blob ----------------------------------------------------------------------------- */
typedef struct dcsim_coeffs {
  /* TrainPowerCoeffs, coeffs.py:4-9:  P_gpu(f) = alpha_p f^3 + beta_p f + gamma_p  [W] (energy_paper.py:4-6) */
  double alpha_p, beta_p, gamma_p;
  /* TrainLatencyCoeffs, coeffs.py:12-17:  T(n,f) per latency_paper.py:4-9  [s/unit] */
  double alpha_t, beta_t, gamma_t;
} dcsim_coeffs_t;

typedef struct dcsim_nf {
  int32_t n;     /* n* */
  int32_t _pad;
  double f;      /* f* */
} dcsim_nf_t;

typedef struct dcsim_dc {
  /* DataCenter, models.py:48-56 and its GPUType, models.py:38-45 */
  int32_t total_gpus;
  int32_t power_gating;
  int32_t n_freq;
  int32_t _pad;
  double p_idle, p_peak, p_sleep, alpha;
  double default_freq;
  double freq_levels[DCSIM_MAX_FREQ];
  double carbon_intensity;                 /* carbon.get(name, 0.0): simulator_paper_multi.py:625 */
  double price_kwh[DCSIM_HOURS];           /* _price_kwh resolved per DC and hour: :986-1005 */
  dcsim_coeffs_t coeffs[2];                /* coeffs_map[(dc, jtype)], [0]=inference [1]=training */
  /* Host-precomputed policy tables (inputs are static per (dc, jtype[, hour])): */
  dcsim_nf_t nf_xfer[2][DCSIM_HOURS];      /* (n*, f*) used at xfer_done: :603-616, :622-645, :668-672 */
  dcsim_nf_t nf_deq[2];                    /* (n*, f*) used in the dequeue loop: :892-902, :909-920 */
  double eco_e_unit[2];                    /* E_unit of best_nf_grid(objective=energy): :1024-1027 */
} dcsim_dc_t;

typedef struct dcsim_arrival {
  /* ArrivalConfig, arrivals.py:18-23 */
  int32_t mode;
  int32_t _pad;
  double rate, amp, period;
} dcsim_arrival_t;

typedef struct dcsim_spec {
  uint64_t magic;
  uint32_t abi_version;
  uint32_t spec_bytes;         /* sizeof(dcsim_spec_t) as seen by the producer */
  int32_t n_dc;                /* D, dict order of `dcs` */
  int32_t n_ing;               /* I, dict order of `ingresses` */
  int32_t algo;                /* DCSIM_ALGO_* */
  int32_t policy_name;         /* DCSIM_POLICY_* */
  int32_t max_gpus_per_job;    /* PolicyConfig, policy.py:8 */
  int32_t inf_priority;        /* policy.py:9 */
  int32_t train_scale_out_low_freq; /* policy.py:12 */
  int32_t num_fixed_gpus;      /* --num_fixed_gpus, algo=debug */
  int32_t route_rule;          /* DCSIM_ROUTE_* */
  int32_t xfer_rule;           /* DCSIM_START_* at xfer_done */
  int32_t deq_rule;            /* DCSIM_START_* in the dequeue loop */
  int32_t control_lower_idle;  /* 1: power_cap>0 and algo in (eco_route, carbon_cost): :221-225 */
  double dvfs_low, dvfs_high;  /* policy.py:10-11 */
  double fixed_freq;           /* 0.0 == not given (the reference tests truthiness: :671) */
  double end_time;             /* sim_duration */
  double log_interval;
  double power_cap;
  /* Sampler constants, evaluated by the HOST's libm exactly where CPython evaluates them, so the device does
   * not re-derive them with its own libm: arrivals.py:7 (xm, 1/alpha), :10 (log(50000), 0.4), :11 (0.1),
   * :8 (1e-9), random.py:102 (NV_MAGICCONST), arrivals.py:30 (2*pi). */
  double pareto_xm, pareto_inv_alpha, lognorm_mu, lognorm_sigma, lognorm_floor, uniform_floor, nv_magicconst, two_pi;
  dcsim_arrival_t arr[2];      /* [0]=arrival_inf [1]=arrival_train */
  /* transfer_s = Lnet_s + data_gb/bottleneck (_net_tuple :482-496); +inf when unreachable */
  double transfer_s[DCSIM_MAX_ING][DCSIM_MAX_DC][2];
  double net_lat_s[DCSIM_MAX_ING][DCSIM_MAX_DC]; /* Lnet_s alone, for job_log.csv net_lat_s */
  dcsim_dc_t dc[DCSIM_MAX_DC];
  /* capacities of the per-replica device structures; 0 = let the library size them from the spec */
  int32_t cap_xfer;            /* in-flight xfer_done events */
  int32_t cap_run;             /* running jobs per DC */
  int32_t cap_q_inf;           /* FIFO entries per DC, inference */
  int32_t cap_q_trn;           /* FIFO entries per DC, training */
  int32_t cap_stale;           /* stale job_finish events (cap_greedy only) */
  int32_t cap_arrivals;        /* entries of the per-replica arrival list written by the arrival pre-pass */
} dcsim_spec_t;

/* ---- per-replica summary (row-major [n_replicas][DCSIM_SUMMARY_K] doubles) ------------------ */
enum {
  DCSIM_S_STATUS = 0,        /* 0 = finished cleanly; else bit mask DCSIM_ST_* */
  DCSIM_S_EVENTS = 1,        /* loop iterations that passed `t > end_time` (:427), incl. stale + log */
  DCSIM_S_JOBS_FINISHED = 2,
  DCSIM_S_JOBS_CREATED = 3,  /* jid counter (:539) */
  DCSIM_S_TOTAL_ENERGY_J = 4,/* sum_dc energy_joules, DC order, left to right */
  DCSIM_S_LAT_SUM = 5,       /* sum of finish-start in finish order (:820) */
  DCSIM_S_LAT_SUM_INF = 6,
  DCSIM_S_FIN_INF = 7,
  DCSIM_S_LAT_SUM_TRN = 8,
  DCSIM_S_FIN_TRN = 9,
  DCSIM_S_RNG_WORDS = 10,    /* 32-bit words consumed from the replica's stream */
  DCSIM_S_LAST_T = 11,       /* time of the last processed event */
  DCSIM_S_SEQ = 12,          /* successful pushes (:163) */
  DCSIM_S_EV_ARRIVAL = 13,
  DCSIM_S_EV_XFER = 14,
  DCSIM_S_EV_FINISH = 15,    /* incl. stale */
  DCSIM_S_EV_LOG = 16,
  DCSIM_S_DONE = 17,         /* 1 once the replica ran to end_time / empty event set and the tail was accrued */
  DCSIM_S_MAX_XFER = 18,     /* high-water marks, for capacity tuning */
  DCSIM_S_MAX_RUN = 19,
  DCSIM_S_MAX_Q = 20,
  DCSIM_S_UTIL_BEGIN = 21,   /* util_begin_ts: the instant of the first processed event (the same for every DC: the sweep :429-437 touches all of them) */
  DCSIM_S_DC0 = 24,          /* then DCSIM_S_DC_STRIDE doubles per DC */
  DCSIM_S_DC_STRIDE = 8,
  DCSIM_SUMMARY_K = 24 + 8 * DCSIM_MAX_DC
};
enum { /* offsets inside a per-DC group */
  DCSIM_SD_ENERGY_J = 0, DCSIM_SD_UTIL_GPU_TIME = 1, DCSIM_SD_ACC_JOB_UNIT = 2, DCSIM_SD_BUSY = 3,
  DCSIM_SD_CURRENT_FREQ = 4, DCSIM_SD_Q_INF = 5, DCSIM_SD_Q_TRN = 6, DCSIM_SD_RUNNING = 7
};
enum { /* status bits: a replica that overflowed a capacity stops and says so — never silently */
  DCSIM_ST_XFER_OVERFLOW = 1, DCSIM_ST_RUN_OVERFLOW = 2, DCSIM_ST_QUEUE_OVERFLOW = 4,
  DCSIM_ST_STALE_OVERFLOW = 8, DCSIM_ST_RNG_RUNAWAY = 16, DCSIM_ST_ARRIVALS_OVERFLOW = 32,
  DCSIM_ST_ARRIVAL_TIE = 64,  /* (unused since ABI 2: arrivals at the same instant are ordered by push rank, as the heap does) */
  DCSIM_ST_SEQ_OVERFLOW = 128 /* a replica pushed more than 2^28 events: the builds that carry several replicas per warp
                                 pack the pop-min's (seq, slot) in one word */
};

/* aggregate vector produced by dcsim_reduce_summary(); the only thing that crosses NVLink */
enum {
  DCSIM_A_REPLICAS = 0, DCSIM_A_FAILED = 1, DCSIM_A_EVENTS = 2, DCSIM_A_JOBS = 3, DCSIM_A_ENERGY = 4,
  DCSIM_A_ENERGY_SQ = 5, DCSIM_A_LAT_SUM = 6, DCSIM_A_MEANLAT_SUM = 7, DCSIM_A_MEANLAT_SQ = 8,
  DCSIM_A_RNG_WORDS = 9, DCSIM_A_FORKS = 10,
  DCSIM_A_RUNNING = 11, /* replicas neither finished nor stopped on a status bit: more dcsim_advance() calls needed */
  DCSIM_AGG_K = 16
};

/* one trace record per processed event of the traced replica */
typedef struct dcsim_trace_rec {
  double t;
  uint32_t seq;
  uint32_t kind; /* 0 arrival_inf, 1 arrival_trn, 2 xfer_done, 3 job_finish, 4 log */
} dcsim_trace_rec_t;

/* one row of job_log.csv (simulator_paper_multi.py:420-421, 815-823), unrounded */
typedef struct dcsim_job_rec {
  uint32_t jid;
  uint32_t n_gpus;                 /* up to the DC's total_gpus (<= 65535, checked by dcsim_create) */
  uint8_t ingress, jtype, dc, _pad0;
  uint32_t _pad1;
  double size, f_used, start_s, finish_s;
} dcsim_job_rec_t;

/* one row of cluster_log.csv (simulator_paper_multi.py:414-418, 944-948), unrounded */
typedef struct dcsim_cluster_rec {
  double time_s;
  double freq;
  double util_gpu_time;
  double util_begin_ts;
  double acc_job_unit;
  double power_w;
  double energy_j;
  int32_t dc, busy, run_total, run_inf, q_inf, q_train;
} dcsim_cluster_rec_t;

typedef struct dcsim dcsim_t;

/* ---- entry points -------------------------------------------------------------------------- */

/* sizeof checks so a binding can verify its struct mirror */
size_t dcsim_sizeof_spec(void);
uint32_t dcsim_abi_version(void);
int dcsim_summary_k(void);

/* Replaces MultiIngressPaperSimulator.__init__ (simulator_paper_multi.py:31-157) for n_replicas
 * independent trajectories.  Replica r (0-based, local) uses Philox key = base_seed + first_replica_id + r,
 * i.e. the key the reference would get from rng_seed (:71) under oracle/philox_random.py.
 * Schedules the first arrival per (ingress, jtype) and the first log tick exactly as :154-157. */
int dcsim_create(const void* spec_blob, size_t spec_bytes, uint64_t n_replicas, uint64_t base_seed,
                 uint64_t first_replica_id, int device, dcsim_t** out);

/* Returns every replica to its freshly-constructed state with new keys (base_seed + first_replica_id + r),
 * keeping all device allocations.  Asynchronous on the handle's stream. */
int dcsim_reset(dcsim_t* h, uint64_t base_seed, uint64_t first_replica_id);

/* Launch on a caller-provided cudaStream_t (e.g. torch's current stream) instead of the handle's own. */
int dcsim_set_stream(dcsim_t* h, void* cuda_stream);

/* Record the first `capacity` processed events of local replica `replica` (debug aid; 0 disables). */
int dcsim_set_trace(dcsim_t* h, uint64_t replica, uint32_t capacity);

/* Record job_log / cluster_log rows of one local replica (the CSV wire formats); capacities in rows. */
int dcsim_set_logging(dcsim_t* h, uint64_t replica, uint32_t job_capacity, uint32_t cluster_capacity);

/* Launches the arrival pre-pass (dcsim_arrivals_kernel) for a freshly created / reset batch if it has not run yet:
 * one thread per replica draws that replica's whole arrival sequence — inter-arrival gaps (arrivals.py:35-48), job
 * sizes (arrivals.py:5-11) and routed DCs (simulator_paper_multi.py:544-577) — in the reference's draw order and
 * writes it as a list the event loop consumes.  Optional: dcsim_advance() calls it when needed; exposed so a
 * caller can time or overlap it.  Asynchronous on the handle's stream.  No-op when the library was asked to keep
 * the samplers inside the event loop (environment DCSIM_PREPASS=0). */
int dcsim_prepare(dcsim_t* h);

/* Replaces MultiIngressPaperSimulator.run (simulator_paper_multi.py:412-480): every replica processes up
 * to max_events_per_replica further events (0 = run to end_time); replicas that reach the end also accrue
 * the tail interval (:469-475).  Asynchronous on the handle's stream unless total_events_out != NULL, in
 * which case it synchronises and returns the number of events processed by this call. */
int dcsim_advance(dcsim_t* h, uint64_t max_events_per_replica, uint64_t* total_events_out);

/* 1 when every replica has DCSIM_S_DONE set (synchronises). */
int dcsim_all_done(dcsim_t* h, int* done_out);

/* Copies [n_replicas][DCSIM_SUMMARY_K] doubles to host memory (synchronises). */
int dcsim_fetch_summary(dcsim_t* h, double* out, size_t out_bytes);

/* The same rows through a page-locked host buffer the library owns (allocated on first use): a full-rate DMA instead of a
 * pageable copy (46 MB for 65 536 replicas: ~2 ms instead of ~20).  *host_ptr_out stays valid until the next call on
 * this handle or dcsim_destroy(); synchronises. */
int dcsim_fetch_summary_host(dcsim_t* h, const double** host_ptr_out);

/* Device pointer of the same array, for zero-copy consumers on the same device. */
int dcsim_summary_device_ptr(dcsim_t* h, void** dev_ptr_out);

/* Reduces the per-replica summaries to DCSIM_AGG_K doubles on the device, written to `dev_out` (a device
 * pointer, e.g. a torch tensor's data_ptr) on the handle's stream.  This vector is what the caller
 * all-reduces over NCCL at end of run; no other data crosses GPUs. */
int dcsim_reduce_summary(dcsim_t* h, double* dev_out);

/* The same vector summed over all ranks of `nccl_comm` (an ncclComm_t the caller created, one rank per GPU): reduces on
 * the device, ncclAllReduce(sum, double, DCSIM_AGG_K) on the handle's stream, copies the result to `out` (host memory,
 * DCSIM_AGG_K doubles) and synchronises.  The run's only collective, for hosts that drive NCCL themselves (SURVEY.md
 * App. D b200sim_allreduce_summary); NCCL is looked up at run time, DCSIM_E_UNSUPPORTED if the process has none. */
int dcsim_allreduce_summary(dcsim_t* h, void* nccl_comm, double* out);

/* Job-latency histogram of the whole batch (latency = finish - start, the job_log.csv latency_s column,
 * simulator_paper_multi.py:820): DCSIM_LAT_BINS bins per job type, 4 per octave starting at 2^-20 s — bin index =
 * 4 * (exponent + 20) + top two mantissa bits, clamped — summed over all replicas on the device.  `out` receives
 * [2][DCSIM_LAT_BINS] counts ([0] = inference, [1] = training).  Quantiles (p50 / p99 ...) follow on the host. */
#define DCSIM_LAT_BINS 128
/* Opt-in (before the first advance of a batch; stays on across dcsim_reset): allocates the per-replica histograms and
 * makes the finish handler feed them (one fire-and-forget RED per finished job, ~1 % of kernel time). */
int dcsim_enable_latency_histogram(dcsim_t* h);
int dcsim_fetch_latency_histogram(dcsim_t* h, uint64_t* out, size_t out_bytes);

/* Cluster-log ensemble: at every log tick, for EVERY replica, the values the replica's cluster_log.csv row of each DC
 * would hold (simulator_paper_multi.py write_csv_logs), unrounded.  Device layout [tick][field][dc][replica] doubles,
 * replica fastest (the reductions read it coalesced).  Tick k is the k-th processed log event (instant: the chain
 * t += log_interval from 0, the same in every replica).  A replica writes ticks < capacity and keeps counting past that
 * (its true count is DCSIM_S_EV_LOG of its summary row); a fetch or reduction that finds a replica past the capacity
 * fails with DCSIM_E_STATE instead of truncating. */
enum {
  DCSIM_ENS_FREQ = 0,        /* current_freq, after the control_lower_idle rewrite (:221-225) */
  DCSIM_ENS_BUSY = 1,        /* busy GPUs */
  DCSIM_ENS_RUN_TOTAL = 2,   /* running jobs */
  DCSIM_ENS_RUN_INF = 3,
  DCSIM_ENS_RUN_TRAIN = 4,   /* run_total - run_inf */
  DCSIM_ENS_Q_INF = 5,
  DCSIM_ENS_Q_TRAIN = 6,
  DCSIM_ENS_UTIL_AVG = 7,    /* util_gpu_time / (total * max(1e-9, now - (util_begin or now))), 0 when total == 0 */
  DCSIM_ENS_ACC_JOB_UNIT = 8,
  DCSIM_ENS_POWER_W = 9,
  DCSIM_ENS_ENERGY_J = 10,   /* unrounded (the CSV shows energy_kJ) */
  DCSIM_ENS_FIELDS = 11
};
#define DCSIM_ENS_BINS 1024
/* Opt-in (before the first advance of a batch; stays on across dcsim_reset, like the latency histogram).  max_ticks = 0:
 * the exact number of log ticks of the spec (the t += log_interval chain replayed against the loop's t > end_time
 * cut-off).  DCSIM_E_NOMEM (with the byte count in dcsim_last_error) when the buffer does not fit. */
int dcsim_enable_cluster_ensemble(dcsim_t* h, uint32_t max_ticks);
/* Tick capacity of the recorder (0 = not enabled). */
int dcsim_cluster_ensemble_capacity(dcsim_t* h, uint32_t* ticks_out);
/* Copies the first min(capacity, out_bytes / row bytes) ticks of the raw values, [tick][field][dc][replica] doubles,
 * to host memory (synchronises).  Ticks a replica did not reach read as NaN.  For tests and small batches. */
int dcsim_fetch_cluster_ensemble(dcsim_t* h, double* out, size_t out_bytes);
/* Pass 1, per column (tick, field, dc) over the replicas that recorded the tick: dev_out = [4][capacity * FIELDS * n_dc]
 * doubles {n, sum, min, max} (an empty column: 0, 0, +inf, -inf).  The caller all-reduces rows 0-1 (sum), 2 (min), 3
 * (max).  Fixed summation order (a function of the replica count only): bit-identical run to run.  Synchronises once to
 * check the capacity. */
int dcsim_ensemble_moments(dcsim_t* h, double* dev_out);
/* Pass 2, given the global per-column mean, lo (min) and hi (max): dev_m2_out[column] = sum (x - mean)^2 (fixed order)
 * and dev_hist_out[column][DCSIM_ENS_BINS] counts over [lo, hi].  Integer fields (busy, run_*, q_*) use unit bins
 * centred on the integers lo, lo+1, ... when hi - lo + 1 <= DCSIM_ENS_BINS, else integer width ceil((hi - lo + 1) / BINS);
 * the others width (hi - lo) / BINS, bin = min(BINS - 1, floor((x - lo) / width)) (all in bin 0 when hi == lo).  The
 * caller all-reduces both (sum). */
int dcsim_ensemble_spread(dcsim_t* h, const double* dev_mean, const double* dev_lo, const double* dev_hi, double* dev_m2_out,
                          uint64_t* dev_hist_out);

/* Job-log ensemble: for EVERY replica, what its job_log.csv rows (simulator_paper_multi.py:820) add up to per finish
 * window, DC and job type.  Window k of W = max(1, ceil(end_time / bin_s)) covers [k * bin_s, (k + 1) * bin_s); a job
 * finishing at t goes to window min(floor(t / bin_s), W - 1) (f64; finishes at end_time and in the 1e-9 slack behind it
 * fold into the last window), and every job also to row W, the whole run.  Per replica and cell two f64 sums, added in
 * finish order: JOBS (count) and LAT_SUM (sum of finish - start, the latency_s column).  Device layout
 * [W + 1][DCSIM_JENS_STORED][n_dc][2 jtypes][n_replicas] doubles, replica fastest (the reductions read it coalesced), and
 * a per-DC job-latency histogram [n_replicas][n_dc][2][DCSIM_LAT_BINS] u32 (the bin rule of the batch histogram above;
 * summed over DCs it is that histogram's row of the replica).  The reductions add a third, derived field: MEAN_LATENCY =
 * LAT_SUM / JOBS, over the replicas with at least one job in the cell.  A replica whose status is not 0 counts in no
 * column and no histogram. */
enum {
  DCSIM_JENS_JOBS = 0,         /* jobs finished in the cell */
  DCSIM_JENS_LAT_SUM = 1,      /* sum of their latencies [s] */
  DCSIM_JENS_STORED = 2,       /* fields the recorder stores per replica */
  DCSIM_JENS_MEAN_LATENCY = 2, /* LAT_SUM / JOBS (reductions only) */
  DCSIM_JENS_FIELDS = 3        /* fields of the reductions' columns */
};
/* Opt-in (before the first advance of a batch; stays on across dcsim_reset, zeroed by it).  bin_s = 0: log_interval.
 * DCSIM_E_INVALID when bin_s is negative or not finite, DCSIM_E_NOMEM (with the byte count in dcsim_last_error) when
 * the buffers do not fit, DCSIM_E_STATE after the first advance. */
int dcsim_enable_job_ensemble(dcsim_t* h, double bin_s);
/* W, the number of finish windows (0 = not enabled); the rows are W + 1. */
int dcsim_job_ensemble_windows(dcsim_t* h, uint32_t* windows_out);
/* Copies the raw per-replica data to host memory (synchronises): `rows` [W + 1][STORED][n_dc][2][n_replicas] doubles,
 * `hist` [n_replicas][n_dc][2][DCSIM_LAT_BINS] u32.  Either may be NULL; a buffer smaller than its array is
 * DCSIM_E_INVALID.  For tests and small batches. */
int dcsim_fetch_job_ensemble(dcsim_t* h, double* rows, size_t rows_bytes, uint32_t* hist, size_t hist_bytes);
/* Pass 1, per column (row, field, dc, jtype) over the valid replicas: dev_out = [4][(W + 1) * JENS_FIELDS * n_dc * 2]
 * doubles {n, sum, min, max}, the same contract as dcsim_ensemble_moments.  Pass 2: as dcsim_ensemble_spread; JOBS is
 * the integer field (unit bins when its range allows).  Both run on the handle's stream, with device pointers. */
int dcsim_job_ensemble_moments(dcsim_t* h, double* dev_out);
int dcsim_job_ensemble_spread(dcsim_t* h, const double* dev_mean, const double* dev_lo, const double* dev_hi,
                              double* dev_m2_out, uint64_t* dev_hist_out);
/* The per-DC job-latency histograms summed over the valid replicas: `out` [n_dc][2][DCSIM_LAT_BINS] u64 (synchronises). */
int dcsim_fetch_dc_latency_histogram(dcsim_t* h, uint64_t* out, size_t out_bytes);

/* Word source of the replicas' random streams (before the first advance of a batch; stays across dcsim_reset).
 *   DCSIM_RNG_PHILOX   (default) Philox4x32-10, key = base_seed + replica id: counter-based, no state.
 *   DCSIM_RNG_MT19937  CPython's own Mersenne Twister seeded like random.seed(base_seed + replica id)
 *                      (simulator_paper_multi.py:71): replica r then reproduces the STOCK reference run with
 *                      rng_seed = base_seed + first_replica_id + r — no re-binding of `random` on the reference side.
 *                      Costs 2.5 kB of HBM per replica and a slower pre-pass; needs the arrival pre-pass
 *                      (DCSIM_E_UNSUPPORTED under DCSIM_PREPASS=0). */
#define DCSIM_RNG_PHILOX 0
#define DCSIM_RNG_MT19937 1
int dcsim_set_rng(dcsim_t* h, int rng_kind);

/* Rows the recorders WOULD have written so far: out3 = {trace, job_log, cluster_log}.  The kernels keep counting past
 * a recorder's capacity (and stop writing), so out3[i] > capacity means the fetched rows are a truncated prefix —
 * callers that need every row (the CSV wire formats) check this and re-run with a larger capacity. */
int dcsim_recorder_counts(dcsim_t* h, uint32_t* out3);

int dcsim_fetch_trace(dcsim_t* h, dcsim_trace_rec_t* out, uint32_t capacity, uint32_t* n_out);
int dcsim_fetch_job_log(dcsim_t* h, dcsim_job_rec_t* out, uint32_t capacity, uint32_t* n_out);
int dcsim_fetch_cluster_log(dcsim_t* h, dcsim_cluster_rec_t* out, uint32_t capacity, uint32_t* n_out);

/* Launch/occupancy facts of the advance kernel for this handle (for bench.py / DESIGN.md). */
typedef struct dcsim_launch_info {
  int32_t warps_per_cta, ctas, smem_bytes_per_cta, regs_per_thread;
  int32_t resident_warps_per_sm, sm_count, cap_xfer, cap_run;
  int32_t cap_q_inf, cap_q_trn, kernel_launches, arrivals_prepass;
  uint64_t hbm_bytes_state, hbm_bytes_queues, hbm_bytes_arrivals;
  int32_t staging_mode;            /* 1 whole state block in shared memory, 2 head only (running-job records stay in
                                      HBM/L2), 0 nothing (in place) */
  int32_t state_block_bytes;       /* one replica's state block */
  int32_t staged_bytes_per_replica;/* the part of it that is staged in shared memory during a launch */
  int32_t lanes_per_replica;       /* 32: one warp per replica; 16 / 8: a warp carries 2 / 4 replicas on lane groups */
} dcsim_launch_info_t;
int dcsim_launch_info(dcsim_t* h, dcsim_launch_info_t* out);

const char* dcsim_last_error(const dcsim_t* h); /* h may be NULL: last create() error of this thread */
void dcsim_destroy(dcsim_t* h);

#ifdef __cplusplus
}
#endif
#endif /* DCSIM_B200_H */
