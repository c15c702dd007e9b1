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
 *     distinct handles are independent — except the members of one group (dcsim_create_shared), which share
 *     the owner's arrival lists and stream and are driven from one thread;
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

/* Launch on a caller-provided cudaStream_t (e.g. torch's current stream) instead of the handle's own.  On the owner of a
 * group it sets the stream of every handle of the group; on a member DCSIM_E_STATE. */
int dcsim_set_stream(dcsim_t* h, void* cuda_stream);

/* ---- policy comparisons on common random numbers ------------------------------------------------------------------
 * Arrivals do not depend on the policy: the arrival pre-pass and the list merge read only the spec's arrival inputs
 * (arr[2], n_ing, n_dc, end_time, the sampler constants, transfer_s, route_rule, cap_arrivals, and eco_e_unit when
 * route_rule is ECO), the replica keys / RNG kind, and the size of the seq ring of in-flight transfers that cap_xfer
 * implies (the merge flags DCSIM_ST_XFER_OVERFLOW in the list header when a transfer lies too far ahead for it); the
 * event loop never writes the list or the header they leave.  So batches
 * of specs that differ in algo, policy, power cap, DVFS thresholds, prices, carbon, nf tables ... can share ONE pre-pass,
 * and replica r of each sees the same jobs at the same instants: the per-replica difference of two policies has far
 * less variance than the difference of two independent batches.
 *
 * dcsim_arrivals_compatible: *equal_out = 1 when the two specs give every replica the same arrival list (host only;
 * DCSIM_E_INVALID for a malformed blob).
 *
 * dcsim_create_shared: a MEMBER of the owner's group.  It takes replica count, keys, RNG kind, device and stream from
 * the owner, allocates its own state, queues and summary, and reads the group's arrival lists (no pre-pass buffers of
 * its own: dcsim_launch_info reports hbm_bytes_arrivals = 0).  DCSIM_E_INVALID when the arrival inputs differ (the
 * message names the first differing field) or the owner is itself a member.
 *   - The first dcsim_prepare / dcsim_advance of ANY handle of the group runs the pre-pass, once.
 *   - dcsim_reset(owner, ...) draws new keys: the group's next prepare / advance re-runs the pre-pass.  A member must
 *     then be reset with the owner's keys (base_seed + first_replica_id equal; DCSIM_E_INVALID otherwise) before it
 *     advances again: until then dcsim_advance returns DCSIM_E_STATE ("arrival source was reset").
 *   - dcsim_set_stream and dcsim_set_rng on a member: DCSIM_E_STATE (set them on the owner, before the group's first
 *     prepare).
 *   - Handles may be destroyed in any order: the lists live until the group's last handle is destroyed. */
int dcsim_arrivals_compatible(const void* spec_a, size_t a_bytes, const void* spec_b, size_t b_bytes, int* equal_out);
int dcsim_create_shared(const void* spec_blob, size_t spec_bytes, dcsim_t* owner, dcsim_t** out);

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

/* Waiting and response times (beside the job-log ensemble, in its cells): a finished job's arrival instant `arr`
 * (simulator_paper_multi.py:539-540), its xfer_done instant `tx` (SIM:580-588) and its start and finish give
 *   wait = start - tx        (the time in its DC's FIFO, SIM:678 -> SIM:840-927; exactly 0.0 when it started at tx)
 *   resp = finish - arr      (time in system: WAN transfer + wait + service)
 * each one f64 subtraction.  Per replica and cell (the job ensemble's window k and row W, DC, job type), added in finish
 * order: WAITED (jobs with wait > 0), WAIT_SUM, RESP_SUM.  Device layout [W + 1][DCSIM_JWAIT_STORED][n_dc][2 jtypes]
 * [n_replicas] doubles, replica fastest, and per-DC histograms [n_replicas][n_dc][2 kinds: wait, resp][2 jtypes]
 * [DCSIM_LAT_BINS] u32 (the bin rule of the latency histograms; a zero wait falls in bin 0).  The reductions' columns
 * are (row, field, dc, jtype): the three stored fields over every valid replica (WAITED the integer one), then
 * MEAN_WAIT = WAIT_SUM / JOBS and MEAN_RESPONSE = RESP_SUM / JOBS over the replicas with JOBS > 0 in the cell (JOBS from
 * the job ensemble). */
enum {
  DCSIM_JWAIT_WAITED = 0,        /* finished jobs of the cell whose wait was > 0 */
  DCSIM_JWAIT_WAIT_SUM = 1,      /* sum of their waits [s] (all finished jobs of the cell) */
  DCSIM_JWAIT_RESP_SUM = 2,      /* sum of their response times [s] */
  DCSIM_JWAIT_STORED = 3,        /* fields the recorder stores per replica */
  DCSIM_JWAIT_MEAN_WAIT = 3,     /* WAIT_SUM / JOBS (reductions only) */
  DCSIM_JWAIT_MEAN_RESPONSE = 4, /* RESP_SUM / JOBS (reductions only) */
  DCSIM_JWAIT_FIELDS = 5         /* fields of the reductions' columns */
};
/* Opt-in, after dcsim_enable_job_ensemble and before the first advance of a batch (stays on across dcsim_reset, zeroed
 * by it; a later dcsim_enable_job_ensemble with another bin_s switches it off).  The running-job records then carry the
 * job id (the layout job_log.csv uses).  DCSIM_E_STATE without the job
 * ensemble, after the first advance or on a member of a shared group; DCSIM_E_NOMEM (with the byte count in
 * dcsim_last_error) when the buffers do not fit. */
int dcsim_enable_job_waits(dcsim_t* h);
/* Copies the raw per-replica data to host memory (synchronises): `rows` [W + 1][DCSIM_JWAIT_STORED][n_dc][2]
 * [n_replicas] doubles, `hist` [n_replicas][n_dc][2][2][DCSIM_LAT_BINS] u32.  Either may be NULL; a buffer smaller than
 * its array is DCSIM_E_INVALID. */
int dcsim_fetch_job_waits(dcsim_t* h, double* rows, size_t rows_bytes, uint32_t* hist, size_t hist_bytes);
/* The two passes over the columns (row, field, dc, jtype), [4][(W + 1) * DCSIM_JWAIT_FIELDS * n_dc * 2]: the contract
 * of dcsim_job_ensemble_moments / _spread; WAITED is the integer field. */
int dcsim_job_waits_moments(dcsim_t* h, double* dev_out);
int dcsim_job_waits_spread(dcsim_t* h, const double* dev_mean, const double* dev_lo, const double* dev_hi,
                           double* dev_m2_out, uint64_t* dev_hist_out);
/* The per-DC wait and response histograms summed over the valid replicas: `out` [n_dc][2 kinds][2][DCSIM_LAT_BINS] u64
 * (synchronises). */
int dcsim_fetch_dc_wait_histogram(dcsim_t* h, uint64_t* out, size_t out_bytes);

/* Job resources (beside the job-log ensemble, in its cells): what every finished job (the set the job ensemble counts)
 * ran on and what the model predicted it would cost.  For a job of DC d with GPU count g (job_log.csv n_gpus), frequency
 * f (its f_used: the frequency of its running record at finish, SIM:713-716, the value job_log.csv writes) and size:
 *   E_job = E_pred * size,  E_pred = P_pred * T_pred = task_power_w(g, f) * step_time_s(g, f)   [J]
 * (SIM:715-716, policy_paper.py:7-16; the oracle's product order, oracle/dcsim_oracle.c:696).
 * Windowed, per replica and cell (the job ensemble's window k and row W, DC, job type), added in finish order:
 * GPU_SUM (sum of g), FREQ_SUM (sum of f [GHz]), ENERGY_SUM (sum of E_job [J]).  Device layout
 * [W + 1][DCSIM_JRES_STORED][n_dc][2 jtypes][n_replicas] doubles, replica fastest.
 * Whole run, per replica, DC d and job type, u32 counts of the finished jobs:
 *   MIX      [DCSIM_JRES_MIX_COLS(G)]: column (min(g, G) - 1) * DCSIM_MAX_FREQ + q for f == freq_levels_d[q] (exact
 *            equality, q < n_freq_d: the match dcsim_bandit_update makes), G = DCSIM_JRES_G(max_gpus_per_job), and a last
 *            column OFF_LEVEL = G * DCSIM_MAX_FREQ for an f that matches no level;
 *   E_HIST   [DCSIM_JRES_EBINS]: quarter-octave bins of E_job anchored at 1 J, bin = clamp(floor(4 * log2(E_job)), 0,
 *            127), decided exactly (DCSIM_JRES_OCT1..3 are the smallest doubles >= 2^(1/4), 2^(1/2), 2^(3/4)).
 * Device layouts [n_dc][2][DCSIM_JRES_MIX_COLS(G)][n_replicas] and [n_dc][2][DCSIM_JRES_EBINS][n_replicas] u32.
 * Bytes per replica: 8 * (W + 1) * 3 * 2 * n_dc + 4 * 2 * n_dc * (MIX_COLS(G) + 128); the bench workload (4 DCs,
 * max_gpus_per_job 8, 120 s in 5 s windows: W = 24) 13 024 B, 854 MB at 65 536 replicas.
 * The reductions' columns: first (row, field, dc, jtype) over DCSIM_JRES_FIELDS fields — the three stored sums over every
 * valid replica, then MEAN_GPUS = GPU_SUM / JOBS, MEAN_FREQ = FREQ_SUM / JOBS and MEAN_ENERGY = ENERGY_SUM / JOBS over
 * the replicas with JOBS > 0 in the cell (JOBS from the job ensemble) — then the mix and the energy bins as stored. */
enum {
  DCSIM_JRES_GPU_SUM = 0,     /* sum of the GPU counts of the cell's finished jobs */
  DCSIM_JRES_FREQ_SUM = 1,    /* sum of their frequencies [GHz] */
  DCSIM_JRES_ENERGY_SUM = 2,  /* sum of their E_job [J] */
  DCSIM_JRES_STORED = 3,      /* fields the recorder stores per replica */
  DCSIM_JRES_MEAN_GPUS = 3,   /* GPU_SUM / JOBS (reductions only) */
  DCSIM_JRES_MEAN_FREQ = 4,   /* FREQ_SUM / JOBS (reductions only) */
  DCSIM_JRES_MEAN_ENERGY = 5, /* ENERGY_SUM / JOBS (reductions only) */
  DCSIM_JRES_FIELDS = 6       /* fields of the reductions' windowed columns */
};
#define DCSIM_JRES_MAX_G 32
#define DCSIM_JRES_G(max_gpus_per_job) ((max_gpus_per_job) < 1 ? 1 : ((max_gpus_per_job) > DCSIM_JRES_MAX_G ? DCSIM_JRES_MAX_G : (max_gpus_per_job)))
#define DCSIM_JRES_MIX_COLS(G) ((G) * DCSIM_MAX_FREQ + 1)
#define DCSIM_JRES_EBINS 128
#define DCSIM_JRES_OCT1 0x1.306fe0a31b716p+0
#define DCSIM_JRES_OCT2 0x1.6a09e667f3bcdp+0
#define DCSIM_JRES_OCT3 0x1.ae89f995ad3aep+0
/* Opt-in, after dcsim_enable_job_ensemble and before the first advance of a batch (stays on across dcsim_reset, zeroed
 * by it; a later dcsim_enable_job_ensemble with another bin_s switches it off).  The running-job records then carry the
 * size and frequency (the layout job_log.csv uses).  DCSIM_E_STATE without the job ensemble, after the first advance or
 * on a member of a shared group; DCSIM_E_NOMEM (with the byte count in dcsim_last_error) when the buffers do not fit. */
int dcsim_enable_job_resources(dcsim_t* h);
/* Copies the raw per-replica data to host memory (synchronises): `rows` [W + 1][DCSIM_JRES_STORED][n_dc][2][n_replicas]
 * doubles, `mix` [n_dc][2][DCSIM_JRES_MIX_COLS(G)][n_replicas] u32, `hist` [n_dc][2][DCSIM_JRES_EBINS][n_replicas] u32.
 * Any may be NULL; a buffer smaller than its array is DCSIM_E_INVALID. */
int dcsim_fetch_job_resources(dcsim_t* h, double* rows, size_t rows_bytes, uint32_t* mix, size_t mix_bytes, uint32_t* hist,
                              size_t hist_bytes);
/* Pass 1 over every column, (W + 1) * DCSIM_JRES_FIELDS * n_dc * 2 windowed, then n_dc * 2 * (MIX_COLS(G) + EBINS)
 * counts: dev_out = [4][columns] {n, sum, min, max}; the count columns' sums are the pooled mix and energy histogram.
 * Pass 2 over the windowed columns only: the contract of dcsim_job_ensemble_spread, GPU_SUM the integer field.  Replicas with
 * status 0 count.  Both on the handle's stream, with device pointers. */
int dcsim_job_resources_moments(dcsim_t* h, double* dev_out);
int dcsim_job_resources_spread(dcsim_t* h, const double* dev_mean, const double* dev_lo, const double* dev_hi,
                               double* dev_m2_out, uint64_t* dev_hist_out);

/* Power profile: for EVERY replica, the cluster power P(t) its total energy integrates, as a step function, and what a
 * site is sized by — peak, time and energy over a threshold, a time-weighted power histogram.
 *   - Each inter-event interval (t_{k-1}, t_k] of positive length has power sum_d P_d, summed in DC order from 0.0,
 *     P_d being the estimate the per-event accrual uses (SIM:168-179, 437) as it stood after event k-1; the tail
 *     (t_last, end_time] has the tail's own power (instantaneous_power_w at current_freq, models.py:82-91, SIM:475).
 *   - The profile starts at the first processed event (DCSIM_S_UTIL_BEGIN); a replica without one has an empty profile
 *     (every field 0).  Zero-length intervals are ignored.
 *   - Consecutive intervals of bitwise-equal power form one LEVEL, whose length is its end minus its start.
 * Per replica (threshold compared with a strict >, +inf = none):
 *   PROFILE_S        end_time - the first event's instant
 *   PEAK_W           largest level power;  T_PEAK_S  start of the first level at it
 *   OVER_S / OVER_J  total length of the levels above the threshold / sum (power - threshold) * length over them
 *   EXCURSIONS       maximal runs of consecutive levels above the threshold;  LONGEST_OVER_S  the longest, end - start
 *   OUT_OF_RANGE     levels outside the histogram range [0, hi], clamped into the end bins: must be 0, never silent
 *   then DC_PEAK_W[d] largest P_d over the positive-length intervals (tail included), then DCSIM_PP_BINS bins of
 *   seconds over [0, hi]: bin = min(BINS - 1, floor(P / (hi / BINS))), each level adding its length to its bin in level
 *   order.
 * Device layout [DCSIM_PP_FIELDS + n_dc + DCSIM_PP_BINS][n_replicas] doubles, replica fastest. */
enum {
  DCSIM_PP_PROFILE_S = 0, DCSIM_PP_PEAK_W = 1, DCSIM_PP_T_PEAK_S = 2, DCSIM_PP_OVER_S = 3, DCSIM_PP_OVER_J = 4,
  DCSIM_PP_EXCURSIONS = 5, DCSIM_PP_LONGEST_OVER_S = 6, DCSIM_PP_OUT_OF_RANGE = 7,
  DCSIM_PP_FIELDS = 8 /* then n_dc DC_PEAK_W columns, then DCSIM_PP_BINS histogram columns */
};
#define DCSIM_PP_BINS 1024
/* Opt-in (before the first advance of a batch; stays on across dcsim_reset, zeroed by it).  threshold_w = +inf: no
 * threshold (the OVER_* / EXCURSIONS fields stay 0).  DCSIM_E_INVALID for a NaN or negative threshold, DCSIM_E_STATE
 * after the first advance or on a member of a shared group, DCSIM_E_NOMEM (with the byte count in dcsim_last_error)
 * when the rows do not fit. */
int dcsim_enable_power_profile(dcsim_t* h, double threshold_w);
/* hi: the histogram's upper end, an upper bound on the cluster power of any state the spec allows — sum over DCs of
 * total_gpus * max(idle or sleep power, per-GPU busy power at every (job type, frequency) a job can run at, the tail
 * formula's per-GPU active power at those frequencies), times (1 + 2^-20) for the rounding of the sums.  Host only;
 * works whether or not the profile is enabled. */
int dcsim_power_profile_range(dcsim_t* h, double* hi_out);
/* Copies the raw per-replica columns to host memory (synchronises); a smaller buffer is DCSIM_E_INVALID. */
int dcsim_fetch_power_profile(dcsim_t* h, double* out, size_t out_bytes);
/* Pass 1 over every column (the fields, DC_PEAK_W, the bins) and the replicas with status 0: dev_out =
 * [4][DCSIM_PP_FIELDS + n_dc + DCSIM_PP_BINS] {n, sum, min, max}; the bins' sums are the pooled power-duration curve.
 * Pass 2 over the first DCSIM_PP_FIELDS + n_dc columns only (the bins need no spread): m2 and histograms, the contract
 * of dcsim_ensemble_spread; EXCURSIONS and OUT_OF_RANGE are the integer columns.  Both on the handle's stream, with
 * device pointers. */
int dcsim_power_profile_moments(dcsim_t* h, double* dev_out);
int dcsim_power_profile_spread(dcsim_t* h, const double* dev_mean, const double* dev_lo, const double* dev_hi,
                               double* dev_m2_out, uint64_t* dev_hist_out);

/* Energy cost and carbon: for EVERY replica and DC d, the energy d drew in each hour of the day, priced at d's hourly
 * tariff (price_kwh[d][h], USD/kWh) and weighted by its carbon intensity (carbon_intensity[d], gCO2/kWh).
 *   - P_d(t) is the step function d's energy integrates: over each inter-event interval (t_{k-1}, t_k] the estimate the
 *     per-event accrual uses (SIM:168-179, 437) as it stood after event k-1; over the tail (t_last, end_time] the tail's
 *     own power (instantaneous_power_w at current_freq, models.py:82-91).  It starts at the first processed event
 *     (DCSIM_S_UTIL_BEGIN); a replica without one has an empty profile (every column 0).
 *   - A LEVEL of DC d is a maximal run of positive-length intervals whose P_d are bitwise equal (the power profile's
 *     rule, per DC).
 *   - Hour windows are [3600 k, 3600 (k + 1)], boundaries exact doubles.  A level [s, e] is cut at every boundary
 *     strictly inside it; a piece [a, b] lies in window k = floor(a / 3600), corrected so that 3600 k <= a < 3600 (k + 1)
 *     holds for the exact products, and goes to hour of day h = k mod 24 (simulated time 0 is midnight, _current_hour).
 *   - E[d][h] = sum of P * (b - a) over the pieces in hour h, in time order (levels of several days fold into one h).
 * Per replica, columns:
 *   HOUR_J[d][h]   E[d][h]                                             column DCSIM_COST_HOUR_J(n_dc, d, h)
 *   ENERGY_J[d]    sum over h of E[d][h], in h order                   column DCSIM_COST_ENERGY_J(n_dc, d)
 *   COST_USD[d]    sum over h of (E[d][h] / 3.6e6) * price_kwh[d][h], in h order (policy_paper._objective_score's)
 *   CARBON_G[d]    (ENERGY_J[d] / 3.6e6) * carbon_intensity[d]
 *   TOTAL_J, TOTAL_USD, TOTAL_G   the sums over d in DC order from 0.0
 * ENERGY_J[d] is NOT DCSIM_SD_ENERGY_J bit for bit: the summary adds one product per event, this column one per level
 * piece.  The two agree to a relative 1e-10 (the tests pin it).
 * Device layout [DCSIM_COST_COLS(n_dc)][n_replicas] doubles, replica fastest, plus a working row of 3 doubles per replica
 * and DC: (27 n_dc + 3) * 8 + 24 n_dc bytes per replica, 984 B at 4 DCs. */
#define DCSIM_COST_HOUR_J(n_dc, d, h) ((d) * DCSIM_HOURS + (h))
#define DCSIM_COST_ENERGY_J(n_dc, d) (DCSIM_HOURS * (n_dc) + (d))
#define DCSIM_COST_USD(n_dc, d) ((DCSIM_HOURS + 1) * (n_dc) + (d))
#define DCSIM_COST_CARBON_G(n_dc, d) ((DCSIM_HOURS + 2) * (n_dc) + (d))
#define DCSIM_COST_TOTAL_J(n_dc) ((DCSIM_HOURS + 3) * (n_dc))
#define DCSIM_COST_TOTAL_USD(n_dc) ((DCSIM_HOURS + 3) * (n_dc) + 1)
#define DCSIM_COST_TOTAL_G(n_dc) ((DCSIM_HOURS + 3) * (n_dc) + 2)
#define DCSIM_COST_COLS(n_dc) ((DCSIM_HOURS + 3) * (n_dc) + 3)
/* Opt-in (before the first advance of a batch; stays on across dcsim_reset, zeroed by it).  DCSIM_E_STATE after the
 * first advance or on a member of a shared group, DCSIM_E_NOMEM (with the byte count in dcsim_last_error) when the rows
 * and their working state do not fit. */
int dcsim_enable_energy_cost(dcsim_t* h);
/* Copies the raw per-replica columns to host memory (synchronises); a smaller buffer is DCSIM_E_INVALID. */
int dcsim_fetch_energy_cost(dcsim_t* h, double* out, size_t out_bytes);
/* The two passes over every column and the replicas with status 0: the contract of dcsim_ensemble_moments / _spread
 * (no integer columns).  Both on the handle's stream, with device pointers. */
int dcsim_energy_cost_moments(dcsim_t* h, double* dev_out);
int dcsim_energy_cost_spread(dcsim_t* h, const double* dev_mean, const double* dev_lo, const double* dev_hi,
                             double* dev_m2_out, uint64_t* dev_hist_out);

/* Occupancy: for EVERY replica and DC d, how long the queues were and how full the DC was over time.  Step functions over
 * [t0, end_time]: Qi(t) = len(q_inf), Qt(t) = len(q_train), Q = Qi + Qt, N(t) = running jobs, B(t) = busy GPUs.
 *   - t0 is the first processed event (DCSIM_S_UTIL_BEGIN); a replica without one has an empty profile (every field 0).
 *   - Over each inter-event interval (t_{k-1}, t_k] the value is the state before event k (the state the energy and
 *     utilisation accrual integrates, SIM:429-437); over the tail (t_last, end_time] the final state.
 *   - A LEVEL of one function is a maximal run of positive-length intervals with the same value.  Every field is a sum
 *     over that function's levels in time order, a level adding value * (end - start) or its length end - start.
 * Per replica PROFILE_S = end_time - t0, then per DC (column 1 + field * n_dc + d):
 *   Q_INF_AREA, Q_TRN_AREA, RUN_AREA   sum of value * length over the levels of Qi, Qt, N
 *   Q_INF_MAX, Q_TRN_MAX               largest level value, 0 if none (<= the instantaneous DCSIM_S_MAX_Q)
 *   QUEUED_S                           total length of the levels of Q with Q > 0
 *   SATURATED_S / IDLE_S               total length of the levels of B with B == total_gpus / B == 0
 * then DCSIM_OCC_BINS queue-length bins per DC (seconds at each Q: bin min(Q, DCSIM_OCC_BINS - 1)) and DCSIM_OCC_BINS
 * busy-GPU bins per DC (seconds at each B: bin B / DCSIM_OCC_BUSY_WIDTH(total_gpus)).
 * Device layout [1 + DCSIM_OCC_FIELDS * n_dc + 2 * DCSIM_OCC_BINS * n_dc][n_replicas] doubles, replica fastest: the
 * queue bins of DC d at column 1 + FIELDS * n_dc + d * BINS, its busy bins at 1 + FIELDS * n_dc + (n_dc + d) * BINS. */
enum {
  DCSIM_OCC_Q_INF_AREA = 0, DCSIM_OCC_Q_TRN_AREA = 1, DCSIM_OCC_RUN_AREA = 2, DCSIM_OCC_Q_INF_MAX = 3,
  DCSIM_OCC_Q_TRN_MAX = 4, DCSIM_OCC_QUEUED_S = 5, DCSIM_OCC_SATURATED_S = 6, DCSIM_OCC_IDLE_S = 7,
  DCSIM_OCC_FIELDS = 8 /* per DC, after the PROFILE_S column */
};
#define DCSIM_OCC_BINS 128
/* Busy-GPU bin width of a DC with `total` GPUs: ceil((total + 1) / DCSIM_OCC_BINS), 1 for up to 127 GPUs. */
#define DCSIM_OCC_BUSY_WIDTH(total) (((total) + DCSIM_OCC_BINS) / DCSIM_OCC_BINS)
/* Opt-in (before the first advance of a batch; stays on across dcsim_reset, zeroed by it).  DCSIM_E_STATE after the
 * first advance or on a member of a shared group, DCSIM_E_NOMEM (with the byte count in dcsim_last_error) when the rows
 * and their working state do not fit. */
int dcsim_enable_occupancy(dcsim_t* h);
/* w_out[n_dc]: each DC's busy-GPU bin width (DCSIM_OCC_BUSY_WIDTH). */
int dcsim_occupancy_bin_widths(dcsim_t* h, int32_t* w_out);
/* Copies the raw per-replica columns to host memory (synchronises); a smaller buffer is DCSIM_E_INVALID. */
int dcsim_fetch_occupancy(dcsim_t* h, double* out, size_t out_bytes);
/* Columns: first DCSIM_OCC_FIELDS * n_dc statistics (field, dc), field-major, per replica Q_INF_AREA / PROFILE_S,
 * Q_TRN_AREA / PROFILE_S, RUN_AREA / PROFILE_S, Q_INF_MAX, Q_TRN_MAX, QUEUED_S / PROFILE_S, SATURATED_S / PROFILE_S,
 * IDLE_S / PROFILE_S; then the 2 * DCSIM_OCC_BINS * n_dc bins as stored.  A replica counts when its status is 0 and
 * PROFILE_S > 0.  Pass 1 over every column: dev_out = [4][columns] {n, sum, min, max}; the bins' sums are the pooled
 * time-weighted distributions of queue length and busy GPUs.  Pass 2 over the statistics columns only: m2 and
 * histograms, the contract of dcsim_ensemble_spread; Q_INF_MAX and Q_TRN_MAX are the integer columns.  Both on the
 * handle's stream, with device pointers. */
int dcsim_occupancy_moments(dcsim_t* h, double* dev_out);
int dcsim_occupancy_spread(dcsim_t* h, const double* dev_mean, const double* dev_lo, const double* dev_hi,
                           double* dev_m2_out, uint64_t* dev_hist_out);

/* Per-run tail latency: for EVERY replica, exact order statistics of its own finished jobs.  For a job that finished
 * (status 0 replica) with arrival instant arr (the ingress arrival, simulator_paper_multi.py:539-540), xfer_done instant
 * tx (SIM:580-588), start and finish, each one f64 subtraction:
 *   latency  = finish - start   (SIM:820: the latency_s column, the reference's p99 monitor sample)
 *   wait     = start - tx       (as dcsim_enable_job_waits)
 *   response = finish - arr     (as dcsim_enable_job_waits)
 * A group is (job type, scope): scope 0 all DCs, scope 1 + d DC d (the DC the job ran in).  Per replica and group:
 *   JOBS        jobs of the group that finished;
 *   UNFINISHED  jobs the run created (a jid, SIM:541) of that type, routed to that DC, not finished at end_time
 *               (in transfer, queued or running); summed over types and DCs: JOBS_CREATED - JOBS_FINISHED;
 *   per kind K: P50, P95, P99, P999 — the q-quantile of the group's n values is the k-th smallest, k = max(ceil(fl(n *
 *               q)), 1) with fl the f64 product (numpy.quantile(..., method="inverted_cdf")) — and MAX; NaN for an
 *               empty group.
 * Then per (kind, job type) SLA_MET: 1.0 when the run's P99 of the all-DC group is <= sla_s, else 0.0; NaN without a
 * finished job of that type, or with sla_s = +inf (no SLA).  Column of group (jt, scope), field f:
 * (jt * (n_dc + 1) + scope) * DCSIM_TAIL_GROUP_FIELDS + f, f = JOBS, UNFINISHED or DCSIM_TAIL_STAT(kind, stat); column
 * of SLA_MET: 2 * (n_dc + 1) * DCSIM_TAIL_GROUP_FIELDS + kind * 2 + jt.  Device layout [DCSIM_TAIL_COLS(n_dc)]
 * [n_replicas] doubles, replica fastest; every column of a replica whose status is not 0 is NaN. */
enum {
  DCSIM_TAIL_JOBS = 0, DCSIM_TAIL_UNFINISHED = 1,
  DCSIM_TAIL_LATENCY = 0, DCSIM_TAIL_WAIT = 1, DCSIM_TAIL_RESPONSE = 2, DCSIM_TAIL_KINDS = 3,
  DCSIM_TAIL_P50 = 0, DCSIM_TAIL_P95 = 1, DCSIM_TAIL_P99 = 2, DCSIM_TAIL_P999 = 3, DCSIM_TAIL_MAX = 4,
  DCSIM_TAIL_QUANTILES = 4, /* P50 .. P999: order statistics */
  DCSIM_TAIL_STATS = 5,
  DCSIM_TAIL_GROUP_FIELDS = 2 + DCSIM_TAIL_KINDS * DCSIM_TAIL_STATS
};
#define DCSIM_TAIL_STAT(kind, stat) (2 + (kind) * DCSIM_TAIL_STATS + (stat))
#define DCSIM_TAIL_COLS(n_dc) (2 * ((n_dc) + 1) * DCSIM_TAIL_GROUP_FIELDS + 2 * DCSIM_TAIL_KINDS)
/* Opt-in (before the first advance of a batch; stays on across dcsim_reset, cleared by it).  Each finished job stores its
 * start and finish into a per-arrival slot buffer [n_replicas][cap_arrivals][2] doubles (16 bytes per slot, NaN until
 * it finishes); the running records carry the job id (the layout job_log.csv uses).  DCSIM_E_INVALID for a NaN or
 * negative sla_s (+inf: no SLA), DCSIM_E_STATE after the first advance or on a member of a shared group, DCSIM_E_NOMEM
 * (with the byte count in dcsim_last_error) when the buffers do not fit. */
int dcsim_enable_tail_latency(dcsim_t* h, double sla_s);
/* The columns to host memory, [DCSIM_TAIL_COLS(n_dc)][n_replicas] doubles (synchronises).  The columns are made from
 * the slot buffer by one selection pass on the handle's stream, run by the first of this call, _moments or _spread
 * after the batch is done (every later advance or reset makes them stale); DCSIM_E_STATE while a replica is still
 * running.  A smaller buffer is DCSIM_E_INVALID. */
int dcsim_fetch_tail_latency(dcsim_t* h, double* out, size_t out_bytes);
/* The raw slot buffer of local replicas [first, first + count): [count][cap_arrivals][2] doubles, (start, finish) of
 * arrival slot jid - 1 (synchronises).  A range, because a large batch's buffer takes tens of GB. */
int dcsim_fetch_tail_jobs(dcsim_t* h, uint64_t first, uint64_t count, double* out, size_t out_bytes);
/* The two passes over the DCSIM_TAIL_COLS(n_dc) columns: the contract of dcsim_ensemble_moments / _spread.  A replica
 * counts in a column when its status is 0 and the value is not NaN.  JOBS, UNFINISHED and SLA_MET are integer columns. */
int dcsim_tail_latency_moments(dcsim_t* h, double* dev_out);
int dcsim_tail_latency_spread(dcsim_t* h, const double* dev_mean, const double* dev_lo, const double* dev_hi,
                              double* dev_m2_out, uint64_t* dev_hist_out);

/* Paired reductions: columns (metric, field), metric-major, over replica r's summary rows of `base` and of a variant
 * batch with the same keys (a member's dcsim_summary_device_ptr or a copy of it: [n][DCSIM_SUMMARY_K] doubles on the
 * base's device).  Replica r counts in a column when both rows have status 0 and the metric is defined in both (a
 * per-job or latency metric needs a finished job of that kind).  n_cols = (DCSIM_PAIR_DC_ENERGY_J + n_dc) *
 * DCSIM_PAIR_FIELDS.  The same two passes and contract as dcsim_ensemble_moments / _spread, on the base's stream; n
 * must be the base's replica count.  JOBS_*, UNFINISHED and their differences, and LOWER / HIGHER, are integer columns
 * (unit bins when their range allows). */
enum {
  DCSIM_PAIR_ENERGY_J = 0,         /* total energy [J] */
  DCSIM_PAIR_ENERGY_PER_JOB_J = 1, /* total energy / jobs finished */
  DCSIM_PAIR_JOBS_INF = 2,         /* inference jobs finished */
  DCSIM_PAIR_JOBS_TRN = 3,
  DCSIM_PAIR_MEAN_LAT_INF_S = 4,   /* mean latency of the finished inference jobs */
  DCSIM_PAIR_MEAN_LAT_TRN_S = 5,
  DCSIM_PAIR_UNFINISHED = 6,       /* sum over DCs of queued (both types) + running jobs at the end */
  DCSIM_PAIR_DC_ENERGY_J = 7       /* + dc: energy of each DC */
};
enum { DCSIM_PAIR_BASE = 0, DCSIM_PAIR_VARIANT = 1, DCSIM_PAIR_DIFF = 2 /* variant - base */, DCSIM_PAIR_LOWER = 3 /* 1: variant < base */,
       DCSIM_PAIR_HIGHER = 4, DCSIM_PAIR_FIELDS = 5 };
int dcsim_paired_moments(dcsim_t* base, const double* dev_variant_summary, uint64_t n, double* dev_out);
int dcsim_paired_spread(dcsim_t* base, const double* dev_variant_summary, uint64_t n, const double* dev_mean,
                        const double* dev_lo, const double* dev_hi, double* dev_m2_out, uint64_t* dev_hist_out);

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
