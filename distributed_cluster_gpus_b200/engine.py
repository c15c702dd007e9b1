"""BatchedEngine — thin owner of one ``dcsim_t`` handle (one CUDA device, one stream, R replicas)."""
import ctypes as C
import os

import numpy as np

from . import _native as N
from . import spec as S

TRACE_DTYPE = np.dtype([("t", "<f8"), ("seq", "<u4"), ("kind", "<u4")])
JOB_DTYPE = np.dtype([("jid", "<u4"), ("n_gpus", "<u4"), ("ingress", "u1"), ("jtype", "u1"), ("dc", "u1"), ("_pad0", "u1"),
                      ("_pad1", "<u4"), ("size", "<f8"), ("f_used", "<f8"), ("start_s", "<f8"), ("finish_s", "<f8")], align=True)
CLUSTER_DTYPE = np.dtype([("time_s", "<f8"), ("freq", "<f8"), ("util_gpu_time", "<f8"), ("util_begin_ts", "<f8"),
                          ("acc_job_unit", "<f8"), ("power_w", "<f8"), ("energy_j", "<f8"), ("dc", "<i4"),
                          ("busy", "<i4"), ("run_total", "<i4"), ("run_inf", "<i4"), ("q_inf", "<i4"),
                          ("q_train", "<i4")], align=True)
assert TRACE_DTYPE.itemsize == C.sizeof(S.TraceRec) and JOB_DTYPE.itemsize == C.sizeof(S.JobRec)
assert CLUSTER_DTYPE.itemsize == C.sizeof(S.ClusterRec)


LAT_BINS = 128
ENS_FIELDS = 11     # DCSIM_ENS_FIELDS (names: ensemble.FIELDS)
ENS_BINS = 1024     # DCSIM_ENS_BINS
JENS_STORED = 2     # DCSIM_JENS_STORED: jobs, lat_sum per (window, dc, jtype) and replica
JWAIT_STORED = 3    # DCSIM_JWAIT_STORED: waited, wait_sum, resp_sum per (window, dc, jtype) and replica
JRES_STORED = 3     # DCSIM_JRES_STORED: gpu_sum, freq_sum, energy_sum per (window, dc, jtype) and replica
MAX_FREQ = 16       # DCSIM_MAX_FREQ: the mix's frequency stride
JRES_EBINS = 128    # DCSIM_JRES_EBINS: quarter-octave energy-per-job bins from 1 J


def jres_mix_g(max_gpus_per_job) -> int:
    """G = DCSIM_JRES_G(max_gpus_per_job): the GPU-count rows of the (n, f) mix; the last one takes every g >= G."""
    return min(max(int(max_gpus_per_job), 1), 32)


def latency_bin_edges() -> np.ndarray:
    """Lower edges [s] of the LAT_BINS histogram bins (+ the upper edge of the last): 2^e * (1 + m/4), e from -20."""
    k = np.arange(LAT_BINS + 1)
    return np.ldexp(1.0 + (k % 4) / 4.0, k // 4 - 20)


def latency_quantiles(hist_row, qs=(0.5, 0.9, 0.99)):
    """Quantiles [s] of one histogram row, log-interpolated inside the bin that holds the quantile."""
    h = np.asarray(hist_row, dtype=np.float64)
    total = h.sum()
    if total == 0:
        return [float("nan")] * len(qs)
    edges, cum, out = latency_bin_edges(), np.cumsum(h), []
    for q in qs:
        b = int(np.searchsorted(cum, q * total, side="left"))
        b = min(b, LAT_BINS - 1)
        below = cum[b - 1] if b else 0.0
        frac = (q * total - below) / h[b] if h[b] else 0.0
        out.append(float(edges[b] * (edges[b + 1] / edges[b]) ** frac))
    return out


RNG_KINDS = {"philox": 0, "mt19937": 1}


class RecorderOverflow(RuntimeError):
    """A recorder (0 trace, 1 job log, 2 cluster log, 3 cluster-log ensemble) saw more rows (ensemble: log ticks) than its
    capacity; `.needed` says how many."""

    def __init__(self, which, needed, capacity):
        unit = "ticks" if which == 3 else "rows"
        super().__init__(f"{('trace', 'job log', 'cluster log', 'cluster ensemble')[which]} needs {needed} {unit}, "
                         f"capacity {capacity}")
        self.which, self.needed, self.capacity = which, needed, capacity


class BatchedEngine:
    """R independent replicas of one scenario on one GPU.

    Replica r uses Philox key ``base_seed + first_replica_id + r`` — the key the reference would be given as
    ``rng_seed`` — so results do not depend on how replicas are sharded over GPUs.
    """

    def __init__(self, spec: S.Spec, n_replicas: int, base_seed: int, first_replica_id: int = 0, device: int = 0,
                 cuda_stream: int = 0, _owner=None):
        self._lib = N.load()
        self._h = C.c_void_p()
        self.spec = spec
        blob = spec.to_bytes()
        self._blob = C.create_string_buffer(blob, len(blob))
        self.owner = _owner
        if _owner is None:
            self.n_replicas, self.device = int(n_replicas), int(device)
            self.keys = (base_seed + first_replica_id) & (2**64 - 1)
            N.check(self._lib.dcsim_create(self._blob, len(blob), self.n_replicas, base_seed & (2**64 - 1),
                                           first_replica_id, device, C.byref(self._h)))
        else:
            self.n_replicas, self.device = _owner.n_replicas, _owner.device
            self.keys = _owner.keys
            N.check(self._lib.dcsim_create_shared(self._blob, len(blob), _owner._h, C.byref(self._h)))
        if cuda_stream:
            self.set_stream(cuda_stream)
        self._trace_cap = self._jobs_cap = self._cluster_cap = 0
        self._ens_cap, self._ens_on = 0, False
        self._jens_windows, self._jens_bin = 0, None

    @classmethod
    def shared(cls, spec: S.Spec, owner: "BatchedEngine") -> "BatchedEngine":
        """A member of ``owner``'s group: the same replicas and keys, reading the owner's arrival lists (one pre-pass for
        the group, common random numbers).  ``spec`` must draw the same arrivals (``arrivals_compatible``); its
        ``reset(seed, first)`` forwards the owner's current keys.  The owner may be closed first."""
        return cls(spec, 0, 0, _owner=owner)

    @property
    def is_member(self) -> bool:
        return self.owner is not None

    # -- configuration ---------------------------------------------------------------------------
    def set_stream(self, cuda_stream: int):
        N.check(self._lib.dcsim_set_stream(self._h, C.c_void_p(cuda_stream)), self._h)

    def reset(self, base_seed=None, first_replica_id: int = 0):
        """All replicas back to t = 0 with new keys; allocations are kept.  A member (``shared``) takes its owner's
        current keys (``base_seed=None``); the library refuses any other keys for it."""
        if base_seed is None:
            if self.owner is None:
                raise ValueError("reset: base_seed is required for an engine that owns its keys")
            base_seed, first_replica_id = self.owner.keys, 0
        N.check(self._lib.dcsim_reset(self._h, base_seed & (2**64 - 1), first_replica_id), self._h)
        self.keys = (base_seed + first_replica_id) & (2**64 - 1)

    def set_rng(self, kind: str = "philox"):
        """Word source of the replicas' random streams: "philox" (default; key = seed) or "mt19937" (CPython's own
        generator seeded like ``random.seed(seed)``: replica r is then the STOCK reference run at rng_seed + r)."""
        if kind not in RNG_KINDS:
            raise ValueError(f"unknown rng {kind!r}; expected one of {sorted(RNG_KINDS)}")
        N.check(self._lib.dcsim_set_rng(self._h, RNG_KINDS[kind]), self._h)

    def set_trace(self, replica: int, capacity: int):
        N.check(self._lib.dcsim_set_trace(self._h, replica, capacity), self._h)
        self._trace_cap = capacity

    def set_logging(self, replica: int, job_capacity: int, cluster_capacity: int):
        N.check(self._lib.dcsim_set_logging(self._h, replica, job_capacity, cluster_capacity), self._h)
        self._jobs_cap, self._cluster_cap = job_capacity, cluster_capacity

    # -- run -------------------------------------------------------------------------------------
    def prepare(self):
        """Launches the arrival pre-pass (optional; advance() does it when needed)."""
        N.check(self._lib.dcsim_prepare(self._h), self._h)

    def advance(self, max_events_per_replica: int = 0, sync: bool = True) -> int:
        """Every replica processes up to ``max_events_per_replica`` more events (0 = to end_time).
        With ``sync`` returns the number of events this call processed; otherwise launches and returns -1."""
        if sync:
            total = C.c_uint64(0)
            N.check(self._lib.dcsim_advance(self._h, max_events_per_replica, C.byref(total)), self._h)
            return int(total.value)
        N.check(self._lib.dcsim_advance(self._h, max_events_per_replica, None), self._h)
        return -1

    def all_done(self) -> bool:
        d = C.c_int(0)
        N.check(self._lib.dcsim_all_done(self._h, C.byref(d)), self._h)
        return bool(d.value)

    def summary(self, out=None) -> np.ndarray:
        """[n_replicas, SUMMARY_K] float64; ``out`` may be a (pinned) preallocated array."""
        if out is None and hasattr(self._lib, "dcsim_fetch_summary_host"):
            # through the library's page-locked mirror (a full-rate DMA), then one host copy: the mirror is reused by
            # the next fetch on this handle, the returned array is the caller's
            p = C.POINTER(C.c_double)()
            N.check(self._lib.dcsim_fetch_summary_host(self._h, C.byref(p)), self._h)
            return _copy_rows(np.ctypeslib.as_array(p, shape=(self.n_replicas, S.SUMMARY_K)))
        if out is None:
            out = np.empty((self.n_replicas, S.SUMMARY_K), dtype=np.float64)
        N.check(self._lib.dcsim_fetch_summary(self._h, C.c_void_p(out.ctypes.data), out.nbytes), self._h)
        return out

    def fetch_summary_into(self, host_ptr: int, nbytes: int):
        N.check(self._lib.dcsim_fetch_summary(self._h, C.c_void_p(host_ptr), nbytes), self._h)

    def summary_device_ptr(self) -> int:
        p = C.c_void_p()
        N.check(self._lib.dcsim_summary_device_ptr(self._h, C.byref(p)), self._h)
        return int(p.value)

    def reduce_into(self, device_ptr: int):
        """Writes the AGG_K-vector (spec.A_*) to device memory; the caller all-reduces it."""
        N.check(self._lib.dcsim_reduce_summary(self._h, C.c_void_p(device_ptr)), self._h)

    def enable_latency_histogram(self):
        """Opt-in, before the first advance of a batch: job-latency histogram of the whole batch."""
        N.check(self._lib.dcsim_enable_latency_histogram(self._h), self._h)

    def latency_histogram(self) -> np.ndarray:
        """[2, LAT_BINS] uint64: job-latency counts of the whole batch ([0] inference, [1] training)."""
        out = np.zeros((2, LAT_BINS), dtype=np.uint64)
        N.check(self._lib.dcsim_fetch_latency_histogram(self._h, C.c_void_p(out.ctypes.data), out.nbytes), self._h)
        return out

    # -- cluster-log ensemble (ensemble.py turns it into per-tick statistics) --------------------------------------
    def enable_cluster_ensemble(self, max_ticks=None):
        """Opt-in, before the first advance of a batch (stays on across reset): every replica records the values of its
        cluster_log.csv rows at every log tick (ensemble.FIELDS).  ``max_ticks=None``: the exact tick count of the spec."""
        N.check(self._lib.dcsim_enable_cluster_ensemble(self._h, int(max_ticks or 0)), self._h)
        cap = C.c_uint32(0)
        N.check(self._lib.dcsim_cluster_ensemble_capacity(self._h, C.byref(cap)), self._h)
        self._ens_cap, self._ens_on = int(cap.value), True

    @property
    def cluster_ensemble_capacity(self) -> int:
        """Log ticks the recorder holds (0: not enabled, or a spec without a log tick: log_interval > duration)."""
        return self._ens_cap

    def _ens_check(self, rc):
        """A replica recorded more ticks than the capacity: RecorderOverflow (never a truncated ensemble)."""
        if rc == N.E_STATE and self._ens_cap and b"overflow" in (self._lib.dcsim_last_error(self._h) or b""):
            needed = int(self.summary()[:, S.S_EV_LOG].max())
            raise RecorderOverflow(3, needed, self._ens_cap)
        N.check(rc, self._h)

    def cluster_ensemble_rows(self) -> np.ndarray:
        """[ticks, FIELDS, n_dc, n_replicas] float64, ticks = the most any replica recorded; NaN where a replica did not
        reach a tick.  Raises RecorderOverflow if a replica went past the capacity.  For tests and small batches."""
        if not self._ens_on:
            raise RuntimeError("cluster ensemble not enabled (enable_cluster_ensemble)")
        ticks = min(int(self.summary()[:, S.S_EV_LOG].max()), self._ens_cap)
        out = np.empty((ticks, ENS_FIELDS, self.spec.n_dc, self.n_replicas), dtype=np.float64)
        self._ens_check(self._lib.dcsim_fetch_cluster_ensemble(self._h, C.c_void_p(out.ctypes.data), out.nbytes))
        return out

    def ensemble_moments_into(self, device_ptr: int):
        """Pass 1 on the handle's stream: [4][capacity * FIELDS * n_dc] float64 {n, sum, min, max} at ``device_ptr``."""
        self._ens_check(self._lib.dcsim_ensemble_moments(self._h, C.c_void_p(device_ptr)))

    def ensemble_spread_into(self, mean_ptr: int, lo_ptr: int, hi_ptr: int, m2_ptr: int, hist_ptr: int):
        """Pass 2 on the handle's stream: per column sum (x - mean)^2 and an ENS_BINS histogram over [lo, hi]."""
        self._ens_check(self._lib.dcsim_ensemble_spread(self._h, C.c_void_p(mean_ptr), C.c_void_p(lo_ptr), C.c_void_p(hi_ptr),
                                                        C.c_void_p(m2_ptr), C.c_void_p(hist_ptr)))

    # -- job-log ensemble (ensemble.job_ensemble turns it into per-window statistics) --------------------------------
    def enable_job_ensemble(self, bin_s=None):
        """Opt-in, before the first advance of a batch (stays on across reset): every replica sums its finished jobs and
        their latencies per finish window of ``bin_s`` seconds (None / 0: log_interval), DC and job type, plus a per-DC
        job-latency histogram."""
        if self._jens_bin != (float(bin_s) if bin_s else float(self.spec.log_interval)):
            self._jwait_on = False     # the library drops the waits recorder with the old windows, even when this fails
            self._jres_on = False      # and the job-resources recorder
        N.check(self._lib.dcsim_enable_job_ensemble(self._h, float(bin_s or 0.0)), self._h)
        w = C.c_uint32(0)
        N.check(self._lib.dcsim_job_ensemble_windows(self._h, C.byref(w)), self._h)
        self._jens_windows = int(w.value)
        self._jens_bin = float(bin_s) if bin_s else float(self.spec.log_interval)

    @property
    def job_ensemble_windows(self) -> int:
        """W, the finish windows (0: not enabled); the recorder's rows are W + 1, the last one the whole run."""
        return self._jens_windows

    @property
    def job_ensemble_bin(self):
        """The window width [s] (None: not enabled)."""
        return self._jens_bin if self._jens_windows else None

    def job_ensemble_rows(self):
        """(rows [W + 1, JENS_STORED, n_dc, 2, n_replicas] float64 {jobs, lat_sum}, hist [n_dc, 2, LAT_BINS, n_replicas]
        uint32): every replica's raw recorder.  For tests and small batches."""
        if not self._jens_windows:
            raise RuntimeError("job ensemble not enabled (enable_job_ensemble)")
        rows = np.empty((self._jens_windows + 1, JENS_STORED, self.spec.n_dc, 2, self.n_replicas), dtype=np.float64)
        hist = np.empty((self.n_replicas, self.spec.n_dc, 2, LAT_BINS), dtype=np.uint32)
        N.check(self._lib.dcsim_fetch_job_ensemble(self._h, C.c_void_p(rows.ctypes.data), rows.nbytes,
                                                   C.c_void_p(hist.ctypes.data), hist.nbytes), self._h)
        return rows, np.ascontiguousarray(np.moveaxis(hist, 0, -1))

    def job_ensemble_moments_into(self, device_ptr: int):
        """Pass 1 on the handle's stream: [4][(W + 1) * 3 * n_dc * 2] float64 {n, sum, min, max} at ``device_ptr``."""
        N.check(self._lib.dcsim_job_ensemble_moments(self._h, C.c_void_p(device_ptr)), self._h)

    def job_ensemble_spread_into(self, mean_ptr: int, lo_ptr: int, hi_ptr: int, m2_ptr: int, hist_ptr: int):
        """Pass 2 on the handle's stream: per column sum (x - mean)^2 and an ENS_BINS histogram over [lo, hi]."""
        N.check(self._lib.dcsim_job_ensemble_spread(self._h, C.c_void_p(mean_ptr), C.c_void_p(lo_ptr), C.c_void_p(hi_ptr),
                                                    C.c_void_p(m2_ptr), C.c_void_p(hist_ptr)), self._h)

    def dc_latency_histogram(self) -> np.ndarray:
        """[n_dc, 2, LAT_BINS] uint64: job-latency counts per DC and job type over the replicas with status 0."""
        out = np.zeros((self.spec.n_dc, 2, LAT_BINS), dtype=np.uint64)
        N.check(self._lib.dcsim_fetch_dc_latency_histogram(self._h, C.c_void_p(out.ctypes.data), out.nbytes), self._h)
        return out

    # -- waiting and response times (ensemble.job_waits), in the job ensemble's cells ---------------------------------
    def enable_job_waits(self):
        """Opt-in, after enable_job_ensemble and before the first advance of a batch (stays on across reset, zeroed by
        it): every finished job adds its wait (start - xfer_done) and response time (finish - arrival) to its cells of the
        job ensemble, and to per-DC wait and response histograms.  The running records then carry the job id."""
        N.check(self._lib.dcsim_enable_job_waits(self._h), self._h)
        self._jwait_on = True

    @property
    def job_waits_enabled(self) -> bool:
        return getattr(self, "_jwait_on", False) and bool(self._jens_windows)

    def job_waits_rows(self):
        """(rows [W + 1, JWAIT_STORED, n_dc, 2, n_replicas] float64 {waited, wait_sum, resp_sum}, hist [n_dc, 2 kinds,
        2, LAT_BINS, n_replicas] uint32): every replica's raw recorder.  For tests and small batches."""
        if not self.job_waits_enabled:
            raise RuntimeError("job waits not enabled (enable_job_waits)")
        rows = np.empty((self._jens_windows + 1, JWAIT_STORED, self.spec.n_dc, 2, self.n_replicas), dtype=np.float64)
        hist = np.empty((self.n_replicas, self.spec.n_dc, 2, 2, LAT_BINS), dtype=np.uint32)
        N.check(self._lib.dcsim_fetch_job_waits(self._h, C.c_void_p(rows.ctypes.data), rows.nbytes,
                                                C.c_void_p(hist.ctypes.data), hist.nbytes), self._h)
        return rows, np.ascontiguousarray(np.moveaxis(hist, 0, -1))

    def job_waits_moments_into(self, device_ptr: int):
        """Pass 1 on the handle's stream: [4][(W + 1) * 3 * n_dc * 2] float64 {n, sum, min, max} at ``device_ptr``."""
        N.check(self._lib.dcsim_job_waits_moments(self._h, C.c_void_p(device_ptr)), self._h)

    def job_waits_spread_into(self, mean_ptr: int, lo_ptr: int, hi_ptr: int, m2_ptr: int, hist_ptr: int):
        """Pass 2 on the handle's stream: per column sum (x - mean)^2 and an ENS_BINS histogram over [lo, hi]."""
        N.check(self._lib.dcsim_job_waits_spread(self._h, C.c_void_p(mean_ptr), C.c_void_p(lo_ptr), C.c_void_p(hi_ptr),
                                                 C.c_void_p(m2_ptr), C.c_void_p(hist_ptr)), self._h)

    def dc_wait_histogram(self) -> np.ndarray:
        """[n_dc, 2 kinds (wait, response), 2, LAT_BINS] uint64 over the replicas with status 0."""
        out = np.zeros((self.spec.n_dc, 2, 2, LAT_BINS), dtype=np.uint64)
        N.check(self._lib.dcsim_fetch_dc_wait_histogram(self._h, C.c_void_p(out.ctypes.data), out.nbytes), self._h)
        return out

    # -- job resources (ensemble.job_resources), in the job ensemble's cells ------------------------------------------
    def enable_job_resources(self):
        """Opt-in, after enable_job_ensemble and before the first advance of a batch (stays on across reset, zeroed by
        it): every finished job adds its GPU count, frequency and predicted energy E_pred * size to its cells of the job
        ensemble, and one count each to its DC's (n, f) mix and energy-per-job histogram.  The running records then
        carry the size and frequency."""
        N.check(self._lib.dcsim_enable_job_resources(self._h), self._h)
        self._jres_on = True

    @property
    def job_resources_enabled(self) -> bool:
        return getattr(self, "_jres_on", False) and bool(self._jens_windows)

    def job_resources_rows(self):
        """(rows [W + 1, JRES_STORED, n_dc, 2, n_replicas] float64 {gpu_sum, freq_sum, energy_sum}, mix [n_dc, 2, G,
        MAX_FREQ, n_replicas] uint32, off_level [n_dc, 2, n_replicas] uint32, hist [n_dc, 2, JRES_EBINS, n_replicas]
        uint32): every replica's raw recorder.  For tests and small batches."""
        if not self.job_resources_enabled:
            raise RuntimeError("job resources not enabled (enable_job_resources)")
        n_dc, n, G = self.spec.n_dc, self.n_replicas, jres_mix_g(self.spec.max_gpus_per_job)
        rows = np.empty((self._jens_windows + 1, JRES_STORED, n_dc, 2, n), dtype=np.float64)
        mix = np.empty((n_dc, 2, G * MAX_FREQ + 1, n), dtype=np.uint32)
        hist = np.empty((n_dc, 2, JRES_EBINS, n), dtype=np.uint32)
        N.check(self._lib.dcsim_fetch_job_resources(self._h, C.c_void_p(rows.ctypes.data), rows.nbytes,
                                                    C.c_void_p(mix.ctypes.data), mix.nbytes,
                                                    C.c_void_p(hist.ctypes.data), hist.nbytes), self._h)
        return rows, mix[:, :, :-1].reshape(n_dc, 2, G, MAX_FREQ, n), np.ascontiguousarray(mix[:, :, -1]), hist

    def job_resources_moments_into(self, device_ptr: int):
        """Pass 1 on the handle's stream: [4][(W + 1) * 6 * n_dc * 2 + n_dc * 2 * (G * MAX_FREQ + 1 + JRES_EBINS)] float64
        {n, sum, min, max} at ``device_ptr``."""
        N.check(self._lib.dcsim_job_resources_moments(self._h, C.c_void_p(device_ptr)), self._h)

    def job_resources_spread_into(self, mean_ptr: int, lo_ptr: int, hi_ptr: int, m2_ptr: int, hist_ptr: int):
        """Pass 2 on the handle's stream, over the (W + 1) * 6 * n_dc * 2 windowed columns: per column sum
        (x - mean)^2 and an ENS_BINS histogram over [lo, hi]."""
        N.check(self._lib.dcsim_job_resources_spread(self._h, C.c_void_p(mean_ptr), C.c_void_p(lo_ptr), C.c_void_p(hi_ptr),
                                                     C.c_void_p(m2_ptr), C.c_void_p(hist_ptr)), self._h)

    # -- power profile (ensemble.power_profile turns it into batch statistics) ----------------------------------------
    def enable_power_profile(self, threshold=None):
        """Opt-in, before the first advance of a batch (stays on across reset, zeroed by it): every replica records its
        cluster power step function — peak, time and energy over ``threshold`` watts (None: no threshold), per-DC peaks
        and a time-weighted power histogram (include/dcsim_b200.h DCSIM_PP_*).  Runs the event-loop instantiation with
        the recorder compiled in."""
        N.check(self._lib.dcsim_enable_power_profile(self._h, float("inf") if threshold is None else float(threshold)),
                self._h)
        self._pp_threshold = None if threshold is None else float(threshold)
        self._pp_on = True

    @property
    def power_profile_enabled(self) -> bool:
        return getattr(self, "_pp_on", False)

    @property
    def power_threshold(self):
        """The threshold [W] of the enabled profile (None: none)."""
        return getattr(self, "_pp_threshold", None)

    def power_profile_range(self) -> float:
        """hi [W]: the power histogram covers [0, hi] in PP_BINS bins (the library's bound, dcsim_power_profile_range)."""
        hi = C.c_double(0.0)
        N.check(self._lib.dcsim_power_profile_range(self._h, C.byref(hi)), self._h)
        return float(hi.value)

    def power_profile_rows(self) -> np.ndarray:
        """[PP_FIELDS + n_dc + PP_BINS, n_replicas] float64: every replica's raw profile.  For tests and small batches."""
        rows = np.empty((S.PP_FIELDS + self.spec.n_dc + S.PP_BINS, self.n_replicas), dtype=np.float64)
        N.check(self._lib.dcsim_fetch_power_profile(self._h, C.c_void_p(rows.ctypes.data), rows.nbytes), self._h)
        return rows

    def power_profile_moments_into(self, device_ptr: int):
        """Pass 1 on the handle's stream: [4][PP_FIELDS + n_dc + PP_BINS] float64 {n, sum, min, max} at ``device_ptr``."""
        N.check(self._lib.dcsim_power_profile_moments(self._h, C.c_void_p(device_ptr)), self._h)

    def power_profile_spread_into(self, mean_ptr: int, lo_ptr: int, hi_ptr: int, m2_ptr: int, hist_ptr: int):
        """Pass 2 on the handle's stream over the first PP_FIELDS + n_dc columns: sum (x - mean)^2 and an ENS_BINS
        histogram over [lo, hi]."""
        N.check(self._lib.dcsim_power_profile_spread(self._h, C.c_void_p(mean_ptr), C.c_void_p(lo_ptr), C.c_void_p(hi_ptr),
                                                     C.c_void_p(m2_ptr), C.c_void_p(hist_ptr)), self._h)

    # -- occupancy (ensemble.occupancy turns it into batch statistics) ------------------------------------------------
    def enable_occupancy(self):
        """Opt-in, before the first advance of a batch (stays on across reset, zeroed by it): every replica records, per
        DC, the time-weighted queue lengths, running jobs and busy GPUs between every two events — areas, maxima, time
        queued / saturated / idle, and queue-length and busy-GPU histograms (include/dcsim_b200.h DCSIM_OCC_*).  Runs the
        event-loop instantiation with the profile recorders compiled in."""
        N.check(self._lib.dcsim_enable_occupancy(self._h), self._h)
        self._occ_on = True

    @property
    def occupancy_enabled(self) -> bool:
        return getattr(self, "_occ_on", False)

    def occupancy_bin_widths(self) -> np.ndarray:
        """[n_dc] int32: GPUs per busy-GPU bin of each DC (1 for DCs of up to 127 GPUs)."""
        w = np.zeros(self.spec.n_dc, dtype=np.int32)
        N.check(self._lib.dcsim_occupancy_bin_widths(self._h, C.c_void_p(w.ctypes.data)), self._h)
        return w

    def occupancy_rows(self) -> np.ndarray:
        """[1 + OCC_FIELDS * n_dc + 2 * OCC_BINS * n_dc, n_replicas] float64: every replica's raw columns.  For tests
        and small batches."""
        n_dc = self.spec.n_dc
        rows = np.empty((1 + S.OCC_FIELDS * n_dc + 2 * S.OCC_BINS * n_dc, self.n_replicas), dtype=np.float64)
        N.check(self._lib.dcsim_fetch_occupancy(self._h, C.c_void_p(rows.ctypes.data), rows.nbytes), self._h)
        return rows

    def occupancy_moments_into(self, device_ptr: int):
        """Pass 1 on the handle's stream: [4][OCC_FIELDS * n_dc + 2 * OCC_BINS * n_dc] float64 {n, sum, min, max} at
        ``device_ptr``."""
        N.check(self._lib.dcsim_occupancy_moments(self._h, C.c_void_p(device_ptr)), self._h)

    def occupancy_spread_into(self, mean_ptr: int, lo_ptr: int, hi_ptr: int, m2_ptr: int, hist_ptr: int):
        """Pass 2 on the handle's stream over the first OCC_FIELDS * n_dc columns: sum (x - mean)^2 and an ENS_BINS
        histogram over [lo, hi]."""
        N.check(self._lib.dcsim_occupancy_spread(self._h, C.c_void_p(mean_ptr), C.c_void_p(lo_ptr), C.c_void_p(hi_ptr),
                                                 C.c_void_p(m2_ptr), C.c_void_p(hist_ptr)), self._h)

    # -- energy cost and carbon (ensemble.energy_cost turns it into batch statistics) --------------------------------
    def enable_energy_cost(self):
        """Opt-in, before the first advance of a batch (stays on across reset, zeroed by it): every replica records each
        DC's energy by hour of day, its cost under the DC's hourly tariff and its carbon (include/dcsim_b200.h
        DCSIM_COST_*).  Runs the event-loop instantiation with the profile recorders compiled in."""
        N.check(self._lib.dcsim_enable_energy_cost(self._h), self._h)
        self._cost_on = True

    @property
    def energy_cost_enabled(self) -> bool:
        return getattr(self, "_cost_on", False)

    def energy_cost_rows(self) -> np.ndarray:
        """[cost_cols(n_dc), n_replicas] float64: every replica's raw columns.  For tests and small batches."""
        rows = np.empty((S.cost_cols(self.spec.n_dc), self.n_replicas), dtype=np.float64)
        N.check(self._lib.dcsim_fetch_energy_cost(self._h, C.c_void_p(rows.ctypes.data), rows.nbytes), self._h)
        return rows

    def energy_cost_moments_into(self, device_ptr: int):
        """Pass 1 on the handle's stream: [4][cost_cols(n_dc)] float64 {n, sum, min, max} at ``device_ptr``."""
        N.check(self._lib.dcsim_energy_cost_moments(self._h, C.c_void_p(device_ptr)), self._h)

    def energy_cost_spread_into(self, mean_ptr: int, lo_ptr: int, hi_ptr: int, m2_ptr: int, hist_ptr: int):
        """Pass 2 on the handle's stream over every column: sum (x - mean)^2 and an ENS_BINS histogram over [lo, hi]."""
        N.check(self._lib.dcsim_energy_cost_spread(self._h, C.c_void_p(mean_ptr), C.c_void_p(lo_ptr), C.c_void_p(hi_ptr),
                                                   C.c_void_p(m2_ptr), C.c_void_p(hist_ptr)), self._h)

    # -- per-run tail latency (ensemble.tail_latency turns it into batch statistics) ----------------------------------
    def enable_tail_latency(self, sla_s=None):
        """Opt-in, before the first advance of a batch (stays on across reset, cleared by it): every finished job's start
        and finish instants are kept per arrival slot, and once the batch is done a selection pass turns them into each
        replica's exact p50 / p95 / p99 / p99.9 / max of service, wait and response time per (job type, scope), and
        whether its p99 met ``sla_s`` seconds (None: no SLA) — include/dcsim_b200.h DCSIM_TAIL_*.  The running records
        then carry the job id."""
        N.check(self._lib.dcsim_enable_tail_latency(self._h, float("inf") if sla_s is None else float(sla_s)), self._h)
        self._tail_sla = None if sla_s is None else float(sla_s)
        self._tail_on = True

    @property
    def tail_latency_enabled(self) -> bool:
        return getattr(self, "_tail_on", False)

    @property
    def tail_latency_sla(self):
        """The SLA [s] of the enabled recorder (None: none)."""
        return getattr(self, "_tail_sla", None)

    def tail_latency_rows(self) -> np.ndarray:
        """[S.tail_cols(n_dc), n_replicas] float64: every replica's columns (NaN: does not count).  Runs the selection
        pass first if the batch has not had it yet.  For tests and small batches."""
        rows = np.empty((S.tail_cols(self.spec.n_dc), self.n_replicas), dtype=np.float64)
        N.check(self._lib.dcsim_fetch_tail_latency(self._h, C.c_void_p(rows.ctypes.data), rows.nbytes), self._h)
        return rows

    def tail_latency_jobs(self, first: int = 0, count=None) -> np.ndarray:
        """[count, cap_arrivals, 2] float64: the raw slot buffer of local replicas [first, first + count) (None: to the
        last) — (start, finish) of the job of every arrival slot (jid - 1), NaN while it has not finished.  For tests."""
        cap = self.spec.cap_arrivals if self.spec.cap_arrivals > 0 else 16384
        count = self.n_replicas - first if count is None else int(count)
        out = np.empty((count, cap, 2), dtype=np.float64)
        N.check(self._lib.dcsim_fetch_tail_jobs(self._h, int(first), count, C.c_void_p(out.ctypes.data), out.nbytes),
                self._h)
        return out

    def tail_latency_moments_into(self, device_ptr: int):
        """Pass 1 on the handle's stream: [4][S.tail_cols(n_dc)] float64 {n, sum, min, max} at ``device_ptr``."""
        N.check(self._lib.dcsim_tail_latency_moments(self._h, C.c_void_p(device_ptr)), self._h)

    def tail_latency_spread_into(self, mean_ptr: int, lo_ptr: int, hi_ptr: int, m2_ptr: int, hist_ptr: int):
        """Pass 2 on the handle's stream: per column sum (x - mean)^2 and an ENS_BINS histogram over [lo, hi]."""
        N.check(self._lib.dcsim_tail_latency_spread(self._h, C.c_void_p(mean_ptr), C.c_void_p(lo_ptr), C.c_void_p(hi_ptr),
                                                    C.c_void_p(m2_ptr), C.c_void_p(hist_ptr)), self._h)

    # -- paired reductions (compare.py) ------------------------------------------------------------------------------
    def paired_moments_into(self, variant_summary_ptr: int, device_ptr: int):
        """Pass 1 on this (base) handle's stream against a variant's [n_replicas, SUMMARY_K] summaries on the device:
        [4][(PAIR_DC_ENERGY_J + n_dc) * PAIR_FIELDS] float64 {n, sum, min, max} at ``device_ptr``."""
        N.check(self._lib.dcsim_paired_moments(self._h, C.c_void_p(variant_summary_ptr), self.n_replicas,
                                               C.c_void_p(device_ptr)), self._h)

    def paired_spread_into(self, variant_summary_ptr: int, mean_ptr: int, lo_ptr: int, hi_ptr: int, m2_ptr: int,
                           hist_ptr: int):
        """Pass 2 on this handle's stream: per column sum (x - mean)^2 and an ENS_BINS histogram over [lo, hi]."""
        N.check(self._lib.dcsim_paired_spread(self._h, C.c_void_p(variant_summary_ptr), self.n_replicas,
                                              C.c_void_p(mean_ptr), C.c_void_p(lo_ptr), C.c_void_p(hi_ptr),
                                              C.c_void_p(m2_ptr), C.c_void_p(hist_ptr)), self._h)

    # -- recorders -------------------------------------------------------------------------------
    def recorder_counts(self):
        """(trace, job_log, cluster_log) rows the recorders WOULD have written: more than a recorder's capacity means
        its rows are a truncated prefix (the kernels keep counting and stop writing)."""
        out = (C.c_uint32 * 3)()
        N.check(self._lib.dcsim_recorder_counts(self._h, C.byref(out)), self._h)
        return int(out[0]), int(out[1]), int(out[2])

    def _fetch(self, fn, dtype, cap, which):
        arr = np.zeros(max(cap, 1), dtype=dtype)
        n = C.c_uint32(0)
        N.check(fn(self._h, C.c_void_p(arr.ctypes.data), cap, C.byref(n)), self._h)
        if cap and which is not None and self.recorder_counts()[which] > cap:     # never hand a silently truncated log to a caller
            raise RecorderOverflow(which, self.recorder_counts()[which], cap)
        return arr[: n.value]

    def trace(self):
        """The first `capacity` processed events of the traced replica (a debug aid: a prefix by design)."""
        return self._fetch(self._lib.dcsim_fetch_trace, TRACE_DTYPE, self._trace_cap, None)

    def job_log(self):
        return self._fetch(self._lib.dcsim_fetch_job_log, JOB_DTYPE, self._jobs_cap, 1)

    def cluster_log(self):
        return self._fetch(self._lib.dcsim_fetch_cluster_log, CLUSTER_DTYPE, self._cluster_cap, 2)

    def launch_info(self) -> dict:
        li = S.LaunchInfo()
        N.check(self._lib.dcsim_launch_info(self._h, C.byref(li)), self._h)
        return {name: int(getattr(li, name)) for name, _ in S.LaunchInfo._fields_ if not name.startswith("_")}

    def close(self):
        if getattr(self, "_h", None) is not None and self._h:
            self._lib.dcsim_destroy(self._h)
            self._h = C.c_void_p()

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def arrivals_compatible(spec_a: S.Spec, spec_b: S.Spec) -> bool:
    """True when the two specs give every replica the same arrival list (the library's dcsim_arrivals_compatible): their
    batches can share one arrival pre-pass (``BatchedEngine.shared``)."""
    lib = N.load()
    a, b = spec_a.to_bytes(), spec_b.to_bytes()
    eq = C.c_int(0)
    N.check(lib.dcsim_arrivals_compatible(a, len(a), b, len(b), C.byref(eq)))
    return bool(eq.value)


_COPY_POOL = None


def _copy_rows(src: np.ndarray) -> np.ndarray:
    """A private copy of a large row-major array, row blocks on a few threads (numpy's copy loops release the GIL):
    a single-threaded copy of the 46 MB of summaries of a 65 536-replica batch is memory-latency bound."""
    global _COPY_POOL
    n = src.shape[0]
    if src.nbytes < (8 << 20):
        return src.copy()
    if _COPY_POOL is None:
        from concurrent.futures import ThreadPoolExecutor
        _COPY_POOL = ThreadPoolExecutor(max_workers=4, thread_name_prefix="dcsim-copy")
    dst = np.empty_like(src)
    step = (n + 3) // 4
    list(_COPY_POOL.map(lambda a: np.copyto(dst[a:a + step], src[a:a + step]), range(0, n, step)))
    return dst


STATUS_NAMES = {S.ST_XFER_OVERFLOW: "in-flight transfer pool", S.ST_RUN_OVERFLOW: "running set",
                S.ST_QUEUE_OVERFLOW: "FIFO queue", S.ST_STALE_OVERFLOW: "stale-event pool",
                S.ST_RNG_RUNAWAY: "rejection-sampling runaway", S.ST_ARRIVALS_OVERFLOW: "arrival list",
                S.ST_ARRIVAL_TIE: "two arrivals at the identical instant (unused since ABI 2: ties are resolved in push order)",
                S.ST_SEQ_OVERFLOW: "more than 2^28 event pushes in one replica"}


def describe_status(bits: int) -> str:
    return ", ".join(name for bit, name in STATUS_NAMES.items() if bits & bit) or "ok"


# One idle engine is kept after run_to_completion()/release() so that the next run of the SAME scenario shape (same
# spec blob, replica count, device, stream) re-seeds the existing device allocations (dcsim_reset) instead of
# freeing and re-allocating tens of GB.  free_cached_engine() drops it.
_CACHED = {"key": None, "engine": None}
_CACHED_LOGGED = {"key": None, "engine": None}   # the one-replica companion engine of LoggedReplica


def _job_bin(sp, job_ensemble, job_ensemble_bin):
    """The job-log ensemble's resolved window width, None when it is off."""
    return float(job_ensemble_bin or sp.log_interval) if job_ensemble else None


def _pp_key(power_profile, power_threshold):
    """The power profile's threshold as the engine cache sees it: None when the profile is off, +inf for no threshold."""
    return (float("inf") if power_threshold is None else float(power_threshold)) if power_profile else None


def _cache_key(sp, n_replicas, device, cuda_stream, cluster_ensemble=False, job_bin=None, pp=None, job_waits=False,
               occupancy=False, tail=None, job_resources=False, energy_cost=False):
    # the launch overrides are read when a handle sizes its launch: a parked engine sized under others is not reused
    return (sp.to_bytes(), int(n_replicas), int(device), int(cuda_stream), os.environ.get("DCSIM_RECORDS", ""),
            os.environ.get("DCSIM_GROUP", ""), bool(cluster_ensemble), job_bin, pp, bool(job_waits and job_bin is not None),
            bool(occupancy), tail, bool(job_resources and job_bin is not None), bool(energy_cost))


def _tail_key(tail_latency, tail_sla_s):
    """The tail-latency recorder's SLA as the engine cache sees it: None when the recorder is off, +inf for no SLA."""
    return (float("inf") if tail_sla_s is None else float(tail_sla_s)) if tail_latency else None


def _drop_parked_batch_engine():
    if _CACHED["engine"] is not None:
        _CACHED["engine"].close()
    _CACHED["engine"], _CACHED["key"] = None, None


def acquire_engine(sp, n_replicas, base_seed, first_replica_id=0, device=0, cuda_stream=0, cluster_ensemble=False,
                   job_ensemble=False, job_ensemble_bin=None, power_profile=False, power_threshold=None, job_waits=False,
                   occupancy=False, tail_latency=False, tail_sla_s=None, job_resources=False, energy_cost=False):
    """A fresh batch; ``cluster_ensemble``: with the cluster-log ensemble recorder on; ``job_ensemble``: with the job-log
    ensemble recorder on, windows of ``job_ensemble_bin`` seconds (None: log_interval); ``power_profile``: with the
    power-profile recorder on, threshold ``power_threshold`` watts (None: none); ``job_waits``: with the waiting /
    response-time recorder on (it implies the job ensemble); ``occupancy``: with the occupancy recorder on;
    ``tail_latency``: with the per-run tail-latency recorder on, SLA ``tail_sla_s`` seconds (None: none);
    ``job_resources``: with the job-resources recorder on (it implies the job ensemble); ``energy_cost``: with the
    energy-cost recorder on.  A parked engine is only reused by a caller that asks for the same recorders."""
    job_bin = _job_bin(sp, job_ensemble or job_waits or job_resources, job_ensemble_bin)
    key = _cache_key(sp, n_replicas, device, cuda_stream, cluster_ensemble, job_bin, _pp_key(power_profile, power_threshold),
                     job_waits, occupancy, _tail_key(tail_latency, tail_sla_s), job_resources, energy_cost)
    if _CACHED["engine"] is not None and _CACHED["key"] == key:
        eng, _CACHED["engine"], _CACHED["key"] = _CACHED["engine"], None, None
        eng.reset(base_seed, first_replica_id)   # fresh batch: recorders may be re-targeted again
        eng.set_trace(0, 0)
        eng.set_logging(0, 0, 0)
        eng.set_rng("philox")
        return eng
    _drop_parked_batch_engine()   # (tens of GB: gone before the new batch allocates; the one-replica companion stays)
    eng = BatchedEngine(sp, n_replicas, base_seed, first_replica_id, device, cuda_stream)
    try:
        if cluster_ensemble:
            eng.enable_cluster_ensemble()
        if job_bin is not None:
            eng.enable_job_ensemble(job_bin)
        if job_waits:
            eng.enable_job_waits()
        if job_resources:
            eng.enable_job_resources()
        if power_profile:
            eng.enable_power_profile(power_threshold)
        if occupancy:
            eng.enable_occupancy()
        if tail_latency:
            eng.enable_tail_latency(tail_sla_s)
        if energy_cost:
            eng.enable_energy_cost()
    except BaseException:
        eng.close()
        raise
    return eng


def release_engine(eng, sp, device=0, cuda_stream=0):
    """Parks a finished engine for reuse (see acquire_engine); a previously parked batch engine is destroyed.  The
    parked companion of LoggedReplica is a separate slot and is left alone (closing and re-creating it would cost
    every run() its allocations)."""
    _drop_parked_batch_engine()
    _CACHED["engine"], _CACHED["key"] = eng, _cache_key(sp, eng.n_replicas, device, cuda_stream, eng.cluster_ensemble_capacity > 0,
                                                        eng.job_ensemble_bin,
                                                        _pp_key(eng.power_profile_enabled, eng.power_threshold),
                                                        eng.job_waits_enabled, eng.occupancy_enabled,
                                                        _tail_key(eng.tail_latency_enabled, eng.tail_latency_sla),
                                                        eng.job_resources_enabled, eng.energy_cost_enabled)


def free_cached_engine():
    for slot in (_CACHED, _CACHED_LOGGED):
        if slot["engine"] is not None:
            slot["engine"].close()
        slot["engine"], slot["key"] = None, None


class LoggedReplica:
    """The cluster_log.csv / job_log.csv rows of ONE replica of a batch, produced by a one-replica companion engine
    that runs the same trajectory (same spec, same key) on its own stream WHILE the batch runs.

    Switching the recorders on inside the batch makes every replica carry the job log's fields in its running-job
    records (60 instead of 40 bytes: fewer resident warps); a single warp
    next to the batch's grid costs nothing — it is launched first, is resident before the grid fills the GPU, and
    finishes long before it.  Results are identical by construction (one replica = one deterministic trajectory)."""

    def __init__(self, sp, seed, replica_id, device, job_rows, cluster_rows, rng="philox"):
        key = (sp.to_bytes(), int(device))
        if _CACHED_LOGGED["engine"] is not None and _CACHED_LOGGED["key"] == key:
            self.eng, _CACHED_LOGGED["engine"], _CACHED_LOGGED["key"] = _CACHED_LOGGED["engine"], None, None
            self.eng.reset(seed, replica_id)
        else:
            if _CACHED_LOGGED["engine"] is not None:
                _CACHED_LOGGED["engine"].close()
                _CACHED_LOGGED["engine"], _CACHED_LOGGED["key"] = None, None
            self.eng = BatchedEngine(sp, 1, seed, replica_id, device)    # its own (non-blocking) stream
        self._key = key
        self.eng.set_rng(rng)
        self.eng.set_logging(0, job_rows, cluster_rows)
        self.eng.advance(0, sync=False)                                 # in flight; the caller launches the batch now

    def collect(self):
        """(status bits, job rows, cluster rows); synchronises with the companion's stream."""
        bits = int(self.eng.summary()[0, S.S_STATUS])
        return bits, self.eng.job_log(), self.eng.cluster_log()

    def release(self, keep=True):
        if keep:
            _CACHED_LOGGED["engine"], _CACHED_LOGGED["key"] = self.eng, self._key
        else:
            self.eng.close()
        self.eng = None


def run_to_completion(spec_factory, n_replicas, base_seed, first_replica_id=0, device=0, cuda_stream=0,
                      max_retries=3, configure=None, while_running=None, cluster_ensemble=False, job_ensemble=False,
                      job_ensemble_bin=None, power_profile=False, power_threshold=None, job_waits=False,
                      occupancy=False, tail_latency=False, tail_sla_s=None, job_resources=False, energy_cost=False):
    """Runs all replicas to end_time.  A replica that overflowed a capacity is never trusted: the whole batch
    is re-run with that capacity raised (``spec_factory(caps)`` rebuilds the blob).  Returns (engine, summary);
    hand the engine back with release_engine() (reuse) or close().  ``while_running()`` is called once, after the
    kernels of the first attempt were launched and before the host waits for them (host work that can overlap).
    ``cluster_ensemble`` / ``job_ensemble``: every attempt runs with that ensemble recorder on (``job_ensemble_bin``: its
    window width, None = log_interval); ``power_profile``: with the power-profile recorder on (``power_threshold`` [W],
    None = no threshold); ``job_waits``: with the waiting / response-time recorder on (and the job ensemble);
    ``occupancy``: with the occupancy recorder on; ``tail_latency``: with the per-run tail-latency recorder on
    (``tail_sla_s``: its SLA [s], None = none), its slot buffer sized by each attempt's cap_arrivals; ``job_resources``:
    with the job-resources recorder on (and the job ensemble); ``energy_cost``: with the energy-cost recorder on."""
    caps = {}
    for attempt in range(max_retries + 1):
        sp = spec_factory(dict(caps))
        eng = acquire_engine(sp, n_replicas, base_seed, first_replica_id, device, cuda_stream, cluster_ensemble,
                             job_ensemble, job_ensemble_bin, power_profile, power_threshold, job_waits, occupancy,
                             tail_latency, tail_sla_s, job_resources, energy_cost)
        if configure:
            configure(eng)
        eng.advance(0, sync=False)
        if while_running is not None and attempt == 0:
            try:
                while_running()
            except BaseException:
                eng.close()
                raise
        summ = eng.summary()                     # synchronises with the batch's stream
        bits = int(np.bitwise_or.reduce(summ[:, S.S_STATUS].astype(np.int64)))
        if bits == 0:
            return eng, summ
        eng.close()
        raise_caps(bits, sp, caps, last_attempt=attempt == max_retries)
    raise AssertionError("unreachable")


def raise_caps(bits, sp, caps, last_attempt=False):
    """The capacity retry rule: raises in ``caps`` every capacity of ``sp`` that a replica overflowed (status ``bits``).
    RuntimeError when a status no capacity can cure is set, or on the last attempt."""
    raisable = S.ST_RUN_OVERFLOW | S.ST_XFER_OVERFLOW | S.ST_ARRIVALS_OVERFLOW | S.ST_QUEUE_OVERFLOW | S.ST_STALE_OVERFLOW
    if bits & ~raisable or last_attempt:             # a status no capacity can cure (or out of attempts): fail now
        raise RuntimeError(f"replicas stopped: {describe_status(bits)}")
    g_max = max(sp.dc[d].total_gpus for d in range(sp.n_dc))
    if bits & S.ST_RUN_OVERFLOW:
        caps["cap_run"] = g_max
    if bits & S.ST_XFER_OVERFLOW:
        caps["cap_xfer"] = 2 * sp.cap_xfer
    if bits & S.ST_ARRIVALS_OVERFLOW:
        caps["cap_arrivals"] = 2 * sp.cap_arrivals
    if bits & S.ST_QUEUE_OVERFLOW:
        caps["cap_q_inf"], caps["cap_q_trn"] = 2 * sp.cap_q_inf, 2 * sp.cap_q_trn
    if bits & S.ST_STALE_OVERFLOW:                   # cap_greedy: superseded job_finish events still in the event set
        caps["cap_stale"] = 2 * max(64, sp.cap_stale)
