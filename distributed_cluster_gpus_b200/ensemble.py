"""Batch-wide cluster-log and job-log statistics: per log tick, the mean, spread and quantiles of every DC's
cluster_log.csv columns, and per finish window the same of every DC's job counts and mean latencies, over all replicas
of the batch (all GPUs of a sharded run).

The device records, for every replica, the values its cluster_log.csv rows would hold at every log tick
(``BatchedEngine.enable_cluster_ensemble``).  Two reductions turn them into statistics per column (tick, field, DC):

  moments  n, sum, min, max              -> all-reduce (SUM for n / sum, MIN, MAX)
  spread   sum (x - mean)^2, histogram   -> all-reduce (SUM), given the GLOBAL mean, min and max

Only n, min, max and the histograms cross GPUs exactly: they, and the quantiles read off the histograms, do not depend
on the number of GPUs.  Mean and std do only up to summation order.  ``moments_rows`` / ``spread_rows`` are the numpy
mirror of the two kernels (csrc dcsim_ens_moments_kernel / dcsim_ens_spread_kernel), as ``sharding.aggregate_rows``
mirrors dcsim_reduce_kernel.

The job-log ensemble (``BatchedEngine.enable_job_ensemble``, ``job_ensemble``) runs the same two passes over columns
(row, field, DC, job type): rows are finish windows of ``bin_s`` seconds plus the whole run, fields ``JOB_FIELDS``.
"""
import csv
import math
from dataclasses import dataclass
from typing import Sequence, Tuple

import numpy as np

FIELDS = ("freq", "busy", "run_total", "run_inf", "run_train", "q_inf", "q_train", "util_avg", "acc_job_unit", "power_W",
          "energy_J")                                  # DCSIM_ENS_* order
INTEGER_FIELDS = (1, 2, 3, 4, 5, 6)                    # busy, run_*, q_*: unit-width bins, exact quantiles
BINS = 1024                                            # DCSIM_ENS_BINS
DEFAULT_QUANTILES = (0.05, 0.25, 0.5, 0.75, 0.95)
CSV_HEADER_HEAD = ["time_s", "dc", "field", "n", "mean", "std", "min"]


def tick_times(log_interval: float, n_ticks: int) -> np.ndarray:
    """Instants of the log ticks: the chain t += log_interval from 0 (SIM:157, :949), the same in every replica."""
    out, t = np.empty(n_ticks), 0.0 + log_interval
    for k in range(n_ticks):
        out[k] = t
        t = t + log_interval
    return out


def fields_from_cluster_log(cluster, total_gpus: Sequence[int]) -> np.ndarray:
    """One replica's cluster-log records (engine.CLUSTER_DTYPE, tick-major, DC order) -> [ticks, FIELDS, n_dc], each value
    derived as write_csv_logs (simcore/simulator_paper_multi.py) derives its CSV column, unrounded."""
    n_dc = len(total_gpus)
    ticks = len(cluster) // n_dc
    out = np.empty((ticks, len(FIELDS), n_dc))
    for i, r in enumerate(cluster[:ticks * n_dc]):
        k, d = divmod(i, n_dc)
        total, now = int(total_gpus[d]), float(r["time_s"])
        elapsed = max(1e-9, now - (float(r["util_begin_ts"]) or now))
        util_avg = (float(r["util_gpu_time"]) / (total * elapsed)) if total else 0.0
        out[k, :, d] = (float(r["freq"]), int(r["busy"]), int(r["run_total"]), int(r["run_inf"]),
                        int(r["run_total"]) - int(r["run_inf"]), int(r["q_inf"]), int(r["q_train"]), util_avg,
                        float(r["acc_job_unit"]), float(r["power_w"]), float(r["energy_j"]))
    return out


# ---- host mirror of the two reduction kernels ------------------------------------------------------------------------
def _valid(n_ticks: int, nlog: np.ndarray) -> np.ndarray:
    """[ticks, replicas]: replica r recorded tick k."""
    return np.arange(n_ticks)[:, None] < np.asarray(nlog)[None, :]


def moments_rows(rows: np.ndarray, nlog: np.ndarray) -> np.ndarray:
    """rows [ticks, FIELDS, n_dc, R], nlog [R] (ticks each replica recorded) -> [4, ticks * FIELDS * n_dc]
    {n, sum, min, max}; an empty column is 0, 0, +inf, -inf."""
    T, F, D, R = rows.shape
    ok = np.broadcast_to(_valid(T, nlog)[:, None, None, :], rows.shape)
    return moments_cols(rows.reshape(-1, R), ok.reshape(-1, R))


def moments_cols(x: np.ndarray, m: np.ndarray) -> np.ndarray:
    """x [columns, R] values, m [columns, R] which of them count -> [4, columns] {n, sum, min, max}."""
    out = np.empty((4, x.shape[0]))
    out[0] = m.sum(axis=1)
    out[1] = np.where(m, x, 0.0).sum(axis=1)
    out[2] = np.where(m, x, np.inf).min(axis=1)
    out[3] = np.where(m, x, -np.inf).max(axis=1)
    return out


def bin_widths(lo: np.ndarray, hi: np.ndarray, n_dc: int) -> np.ndarray:
    """Per column of the cluster-log ensemble: the histogram's bin width (0: every value in bin 0)."""
    field = (np.arange(np.asarray(lo).size) // n_dc) % len(FIELDS)
    return bin_widths_for(lo, hi, np.isin(field, INTEGER_FIELDS))


def bin_widths_for(lo: np.ndarray, hi: np.ndarray, integral: np.ndarray) -> np.ndarray:
    """Per column: the histogram's bin width given which columns are integer fields — the kernel's rule, the kernel's
    float ops."""
    lo, hi = np.asarray(lo, dtype=np.float64), np.asarray(hi, dtype=np.float64)
    with np.errstate(invalid="ignore", over="ignore"):
        span = hi - lo + 1.0
        w_int = np.where(span <= BINS, 1.0, np.ceil(span / BINS))
        w_real = (hi - lo) / BINS
        w = np.where(integral, w_int, w_real)
        return np.where(hi > lo, w, 0.0)


def bin_index(x: np.ndarray, lo, width) -> np.ndarray:
    with np.errstate(invalid="ignore", divide="ignore"):
        f = np.floor((x - lo) / np.where(width > 0, width, 1.0))
    b = np.clip(np.nan_to_num(f, nan=0.0, posinf=BINS - 1, neginf=0.0), 0, BINS - 1).astype(np.int64)
    return np.where(width > 0, b, 0)


def spread_rows(rows: np.ndarray, nlog: np.ndarray, mean: np.ndarray, lo: np.ndarray, hi: np.ndarray):
    """-> (m2 [columns] = sum (x - mean)^2, hist [columns, BINS] uint64) over the replicas that recorded each tick."""
    T, F, D, R = rows.shape
    ok = np.broadcast_to(_valid(T, nlog)[:, None, None, :], rows.shape).reshape(-1, R)
    x = rows.reshape(-1, R)
    return spread_cols(x, ok, mean, lo, hi, bin_widths(lo, hi, D))


def spread_cols(x: np.ndarray, ok: np.ndarray, mean, lo, hi, width):
    """x [columns, R], ok [columns, R], per-column mean / lo / width -> (m2 [columns], hist [columns, BINS] uint64)."""
    mean = np.asarray(mean, dtype=np.float64)
    with np.errstate(invalid="ignore"):
        m2 = np.where(ok, (x - mean[:, None]) ** 2, 0.0).sum(axis=1)
    b = bin_index(x, np.asarray(lo)[:, None], width[:, None])
    hist = np.zeros((x.shape[0], BINS), dtype=np.uint64)
    cols = np.broadcast_to(np.arange(x.shape[0])[:, None], x.shape)
    np.add.at(hist, (cols[ok], b[ok]), 1)
    return m2, hist


def hist_quantiles(hist: np.ndarray, n: np.ndarray, lo: np.ndarray, hi: np.ndarray, width: np.ndarray,
                   integral: np.ndarray, quantiles: Sequence[float]) -> np.ndarray:
    """numpy's ``inverted_cdf`` quantiles read off the histograms -> [Q, columns].  The order statistic numpy picks is
    located exactly; its value is exact for unit bins (integer fields) and the bin's centre, clamped to [min, max],
    otherwise (within one bin width)."""
    hist = np.asarray(hist, dtype=np.int64)
    cum = np.cumsum(hist, axis=1)
    n = np.asarray(n, dtype=np.float64)
    out = np.full((len(quantiles), hist.shape[0]), np.nan)
    has = n > 0
    for i, q in enumerate(quantiles):
        v = n * float(q) - 1.0                         # numpy: _inverted_cdf -> _discrete_interpolation_to_boundaries
        prev = np.floor(v)
        j = np.where(v - prev == 0, prev, prev + 1)
        j = np.clip(j, 0, np.maximum(n - 1, 0))
        b = np.argmax(cum > j[:, None], axis=1)
        with np.errstate(invalid="ignore"):
            exact = (integral & (width == 1.0)) | (width == 0)
            val = np.where(exact, lo + b * width, np.clip(lo + (b + 0.5) * width, lo, hi))
        out[i] = np.where(has, val, np.nan)
    return out


@dataclass
class EnsembleResult:
    """Per (tick, field, dc) statistics over every replica of the batch; arrays are [ticks, len(fields), n_dc]."""
    time_s: np.ndarray
    fields: Tuple[str, ...]
    n: np.ndarray
    mean: np.ndarray
    std: np.ndarray                                    # unbiased (ddof = 1); 0 for a single sample
    min: np.ndarray
    max: np.ndarray
    q: Tuple[float, ...]
    quantiles: np.ndarray                              # [Q, ticks, fields, n_dc]

    def quantile_names(self):
        return [f"p{int(round(q * 100)):02d}" for q in self.q]

    def to_csv(self, path: str, dc_names: Sequence[str]):
        """Long format: time_s,dc,field,n,mean,std,min,p05,p25,p50,p75,p95,max (energy in J, unrounded)."""
        T, F, D = self.n.shape
        with open(path, "w", newline="") as f:
            w = csv.writer(f)
            w.writerow(CSV_HEADER_HEAD + self.quantile_names() + ["max"])
            for k in range(T):
                for d in range(D):
                    for i in range(F):
                        w.writerow([repr(float(self.time_s[k])), dc_names[d], self.fields[i], int(self.n[k, i, d]),
                                    repr(float(self.mean[k, i, d])), repr(float(self.std[k, i, d])),
                                    repr(float(self.min[k, i, d]))]
                                   + [repr(float(self.quantiles[j, k, i, d])) for j in range(len(self.q))]
                                   + [repr(float(self.max[k, i, d]))])


def finalize(mom: np.ndarray, m2: np.ndarray, hist: np.ndarray, n_dc: int, log_interval: float,
             quantiles: Sequence[float] = DEFAULT_QUANTILES) -> EnsembleResult:
    """All-reduced moments [4, columns], m2 [columns] and histograms [columns, BINS] -> statistics.  Trailing ticks no
    replica recorded are dropped."""
    F = len(FIELDS)
    n_all, s, lo, hi = (np.asarray(a, dtype=np.float64) for a in mom)
    cols_per_tick = F * n_dc
    per_tick = n_all.reshape(-1, cols_per_tick).max(axis=1)
    T = int(np.nonzero(per_tick > 0)[0].max()) + 1 if np.any(per_tick > 0) else 0
    c = T * cols_per_tick
    n_all, s, lo, hi, m2 = n_all[:c], s[:c], lo[:c], hi[:c], np.asarray(m2, dtype=np.float64)[:c]
    hist = np.asarray(hist)[:c]
    with np.errstate(invalid="ignore", divide="ignore"):
        mean = np.where(n_all > 0, s / n_all, np.nan)
        std = np.where(n_all > 1, np.sqrt(m2 / (n_all - 1)), np.where(n_all == 1, 0.0, np.nan))
    empty = n_all == 0
    width = bin_widths(lo, hi, n_dc)
    integral = np.isin((np.arange(c) // n_dc) % F, INTEGER_FIELDS)
    qv = hist_quantiles(hist, n_all, lo, hi, width, integral, quantiles)
    shape = (T, F, n_dc)
    return EnsembleResult(time_s=tick_times(log_interval, T), fields=FIELDS, n=n_all.astype(np.int64).reshape(shape),
                          mean=mean.reshape(shape), std=std.reshape(shape),
                          min=np.where(empty, np.nan, lo).reshape(shape), max=np.where(empty, np.nan, hi).reshape(shape),
                          q=tuple(float(q) for q in quantiles), quantiles=qv.reshape((len(quantiles),) + shape))


# ---- the two passes with the all-reduces in between ------------------------------------------------------------------
def _allreduce(t, op):
    """In place over every rank (only when torch.distributed runs with world > 1, as sharding.allreduce_aggregate)."""
    import torch.distributed as dist
    if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
        if t.is_cuda and dist.get_backend() == "gloo":
            tmp = t.cpu()
            dist.all_reduce(tmp, op=op)
            t.copy_(tmp)
        else:
            dist.all_reduce(t, op=op)
    return t


def reduce_passes(moments_fn, spread_fn, n_dc: int, log_interval: float,
                  quantiles: Sequence[float] = DEFAULT_QUANTILES) -> EnsembleResult:
    """moments_fn() -> torch [4, columns] float64; spread_fn(mean, lo, hi) -> (m2 [columns] float64, hist [columns, BINS]
    int64), torch tensors on one device.  Runs pass 1, all-reduces it, pass 2 on the global mean / min / max, all-reduces
    that, and finalizes on the host."""
    return finalize(*two_passes(moments_fn, spread_fn), n_dc, log_interval, quantiles)


def two_passes(moments_fn, spread_fn):
    """The two passes with the all-reduces in between (see reduce_passes) -> host (moments, m2, hist)."""
    import torch
    import torch.distributed as dist
    mom = moments_fn()
    _allreduce(mom[0:2], dist.ReduceOp.SUM)
    _allreduce(mom[2], dist.ReduceOp.MIN)
    _allreduce(mom[3], dist.ReduceOp.MAX)
    n = mom[0]
    mean = torch.where(n > 0, mom[1] / n.clamp(min=1.0), torch.zeros_like(n)).contiguous()
    lo, hi = mom[2].contiguous(), mom[3].contiguous()
    m2, hist = spread_fn(mean, lo, hi)
    _allreduce(m2, dist.ReduceOp.SUM)
    _allreduce(hist, dist.ReduceOp.SUM)
    return mom.cpu().numpy(), m2.cpu().numpy(), hist.cpu().numpy()


def cluster_ensemble(engine, quantiles: Sequence[float] = DEFAULT_QUANTILES) -> EnsembleResult:
    """Statistics of the cluster-log ensemble of ``engine`` (a finished BatchedEngine with enable_cluster_ensemble()),
    over all ranks when torch.distributed runs with world > 1 (every rank calls this).  Raises RecorderOverflow if a
    replica recorded more ticks than the capacity."""
    import torch
    dev = torch.device("cuda", engine.device)
    cols = engine.cluster_ensemble_capacity * len(FIELDS) * engine.spec.n_dc

    def moments():
        out = torch.zeros((4, cols), dtype=torch.float64, device=dev)
        if cols:
            torch.cuda.synchronize(dev)                # the library runs on the handle's stream, torch on its own
            engine.ensemble_moments_into(out.data_ptr())
            torch.cuda.synchronize(dev)
        return out

    def spread(mean, lo, hi):
        m2 = torch.zeros(cols, dtype=torch.float64, device=dev)
        hist = torch.zeros((cols, BINS), dtype=torch.int64, device=dev)
        if cols:
            torch.cuda.synchronize(dev)
            engine.ensemble_spread_into(mean.data_ptr(), lo.data_ptr(), hi.data_ptr(), m2.data_ptr(), hist.data_ptr())
            torch.cuda.synchronize(dev)
        return m2, hist

    return reduce_passes(moments, spread, engine.spec.n_dc, engine.spec.log_interval, quantiles)


def cluster_ensemble_from_rows(rows: np.ndarray, nlog: np.ndarray, log_interval: float,
                               quantiles: Sequence[float] = DEFAULT_QUANTILES) -> EnsembleResult:
    """The same statistics from host rows [ticks, FIELDS, n_dc, R] through the numpy mirror (all-reduced over the ranks
    like cluster_ensemble)."""
    import torch
    n_dc = rows.shape[2]
    return reduce_passes(lambda: torch.from_numpy(moments_rows(rows, nlog)),
                         lambda mean, lo, hi: tuple(torch.from_numpy(np.ascontiguousarray(a).astype(dt)) for a, dt in
                                                    zip(spread_rows(rows, nlog, mean.numpy(), lo.numpy(), hi.numpy()),
                                                        (np.float64, np.int64))),
                         n_dc, log_interval, quantiles)


# ---- job-log ensemble ------------------------------------------------------------------------------------------------
JOB_FIELDS = ("jobs", "lat_sum", "mean_latency_s")    # DCSIM_JENS_* order
JOB_TYPES = ("inference", "training")
LAT_BINS = 128                                         # DCSIM_LAT_BINS
JOB_CSV_HEADER_HEAD = ["t0_s", "t1_s", "dc", "type", "field", "n", "mean", "std", "min"]


def job_windows(end_time: float, bin_s: float) -> int:
    """W = max(1, ceil(end_time / bin_s)), the device's f64 expression."""
    w = math.ceil(float(end_time) / float(bin_s))
    return max(1, int(w))


def job_window_index(t, bin_s: float, n_windows: int) -> np.ndarray:
    """Window of a finish instant: min(floor(t / bin_s), W - 1), the device's f64 expression."""
    return np.minimum(np.floor(np.asarray(t, dtype=np.float64) / float(bin_s)), n_windows - 1).astype(np.int64)


def latency_bin(lat) -> np.ndarray:
    """dcsim_lat_bin: 4 bins per octave from 2^-20 s, from the IEEE exponent and the top two mantissa bits."""
    hi = (np.asarray(lat, dtype=np.float64).view(np.uint64) >> np.uint64(32)).astype(np.int64)
    idx = (((hi >> 20) & 0x7FF) - (1023 - 20)) * 4 + ((hi >> 18) & 3)
    return np.clip(idx, 0, LAT_BINS - 1)


def rows_from_job_log(log, n_dc: int, bin_s: float, end_time: float):
    """One replica's job log (engine.JOB_DTYPE rows, finish order) -> what its job-log ensemble recorder holds:
    (rows [W + 1, 2, n_dc, 2] {jobs, lat_sum}, hist [n_dc, 2, LAT_BINS]); the sums run in finish order."""
    W = job_windows(end_time, bin_s)
    rows = np.zeros((W + 1, 2, n_dc, 2))
    hist = np.zeros((n_dc, 2, LAT_BINS), dtype=np.uint32)
    fin = np.asarray(log["finish_s"], dtype=np.float64)
    lat = fin - np.asarray(log["start_s"], dtype=np.float64)
    win, lb = job_window_index(fin, bin_s, W), latency_bin(lat)
    for k, d, jt, x, b in zip(win, log["dc"], log["jtype"], lat, lb):
        for row in (k, W):
            rows[row, 0, d, jt] += 1.0
            rows[row, 1, d, jt] += float(x)
        hist[d, jt, b] += 1
    return rows, hist


def _job_columns(rows: np.ndarray, status: np.ndarray):
    """rows [W + 1, 2, n_dc, 2, R] -> (x, ok) [columns, R], columns (row, JOB_FIELDS, dc, jtype) as the kernels'."""
    R = rows.shape[-1]
    jobs, lat = rows[:, 0], rows[:, 1]
    with np.errstate(invalid="ignore", divide="ignore"):
        mean = lat / jobs
    x = np.stack([jobs, lat, mean], axis=1)
    good = (np.asarray(status) == 0)[None, None, None, :]
    ok = np.stack([np.broadcast_to(good, jobs.shape), np.broadcast_to(good, jobs.shape), good & (jobs > 0)], axis=1)
    return x.reshape(-1, R), ok.reshape(-1, R)


def _job_integral(n_cols: int, n_dc: int) -> np.ndarray:
    return (np.arange(n_cols) // (2 * n_dc)) % len(JOB_FIELDS) == 0


@dataclass
class JobEnsembleResult:
    """Per (row, field, dc, jtype) statistics over every replica of the batch; arrays are [W + 1, len(fields), n_dc, 2],
    rows 0 .. W - 1 the finish windows [t0_s, t1_s), row W the whole run.  Throughput in jobs/s is ``jobs / bin_s`` (a
    window's count over its width) and needs no column of its own."""
    t0_s: np.ndarray
    t1_s: np.ndarray
    bin_s: float
    end_time: float
    fields: Tuple[str, ...]
    n: np.ndarray
    mean: np.ndarray
    std: np.ndarray                                    # unbiased (ddof = 1); 0 for a single sample
    min: np.ndarray
    max: np.ndarray
    q: Tuple[float, ...]
    quantiles: np.ndarray                              # [Q, W + 1, fields, n_dc, 2]
    pooled_mean_latency_s: np.ndarray                  # [W + 1, n_dc, 2]: sum of lat_sum / sum of jobs over the replicas
    latency_histogram: np.ndarray                      # [n_dc, 2, LAT_BINS] uint64: per-DC job latencies, whole run

    def quantile_names(self):
        return [f"p{int(round(q * 100)):02d}" for q in self.q]

    def to_csv(self, path: str, dc_names: Sequence[str]):
        """Long format: t0_s,t1_s,dc,type,field,n,mean,std,min,p05,p25,p50,p75,p95,max.  Per window, then for the whole
        run (t0_s = 0, t1_s = end_time), the rows of ``jobs`` and ``mean_latency_s`` per DC and type; then per DC and
        type one whole-run ``latency_s`` row: n = jobs, mean = the pooled mean latency, quantiles from the per-DC
        log-binned latency histogram (engine.latency_quantiles), std / min / max empty."""
        from .engine import latency_quantiles
        rows, F, D, J = self.n.shape
        keep = [self.fields.index("jobs"), self.fields.index("mean_latency_s")]
        with open(path, "w", newline="") as f:
            w = csv.writer(f)
            w.writerow(JOB_CSV_HEADER_HEAD + self.quantile_names() + ["max"])
            for k in range(rows):
                for d in range(D):
                    for jt in range(J):
                        for i in keep:
                            w.writerow([repr(float(self.t0_s[k])), repr(float(self.t1_s[k])), dc_names[d], JOB_TYPES[jt],
                                        self.fields[i], int(self.n[k, i, d, jt]), repr(float(self.mean[k, i, d, jt])),
                                        repr(float(self.std[k, i, d, jt])), repr(float(self.min[k, i, d, jt]))]
                                       + [repr(float(self.quantiles[j, k, i, d, jt])) for j in range(len(self.q))]
                                       + [repr(float(self.max[k, i, d, jt]))])
            for d in range(D):
                for jt in range(J):
                    h = self.latency_histogram[d, jt]
                    w.writerow([repr(0.0), repr(float(self.end_time)), dc_names[d], JOB_TYPES[jt], "latency_s",
                                int(h.sum()), repr(float(self.pooled_mean_latency_s[-1, d, jt])), "", ""]
                               + [repr(float(v)) for v in latency_quantiles(h, self.q)] + [""])


def job_finalize(mom, m2, hist, lat_hist, n_dc: int, bin_s: float, end_time: float,
                 quantiles: Sequence[float] = DEFAULT_QUANTILES) -> JobEnsembleResult:
    """All-reduced moments [4, columns], m2, histograms [columns, BINS] and per-DC latency histograms -> statistics."""
    F, J = len(JOB_FIELDS), 2
    n_all, s, lo, hi = (np.asarray(a, dtype=np.float64) for a in mom)
    m2 = np.asarray(m2, dtype=np.float64)
    c = n_all.size
    rows = c // (F * n_dc * J)
    with np.errstate(invalid="ignore", divide="ignore"):
        mean = np.where(n_all > 0, s / n_all, np.nan)
        std = np.where(n_all > 1, np.sqrt(m2 / (n_all - 1)), np.where(n_all == 1, 0.0, np.nan))
    empty = n_all == 0
    integral = _job_integral(c, n_dc)
    qv = hist_quantiles(np.asarray(hist), n_all, lo, hi, bin_widths_for(lo, hi, integral), integral, quantiles)
    shape = (rows, F, n_dc, J)
    s4 = s.reshape(shape)
    with np.errstate(invalid="ignore", divide="ignore"):
        pooled = np.where(s4[:, 0] > 0, s4[:, 1] / s4[:, 0], np.nan)
    W = rows - 1
    k = np.arange(W, dtype=np.float64)
    return JobEnsembleResult(t0_s=np.append(k * bin_s, 0.0), t1_s=np.append((k + 1.0) * bin_s, float(end_time)),
                             bin_s=float(bin_s), end_time=float(end_time), fields=JOB_FIELDS,
                             n=n_all.astype(np.int64).reshape(shape), mean=mean.reshape(shape), std=std.reshape(shape),
                             min=np.where(empty, np.nan, lo).reshape(shape), max=np.where(empty, np.nan, hi).reshape(shape),
                             q=tuple(float(q) for q in quantiles), quantiles=qv.reshape((len(quantiles),) + shape),
                             pooled_mean_latency_s=pooled,
                             latency_histogram=np.asarray(lat_hist).astype(np.uint64).reshape(n_dc, J, LAT_BINS))


def _job_passes(moments_fn, spread_fn, lat_hist, n_dc, bin_s, end_time, quantiles):
    """The two passes, then the per-DC latency histograms (torch int64, on the device of the passes) all-reduced."""
    import torch.distributed as dist
    mom, m2, hist = two_passes(moments_fn, spread_fn)
    lh = _allreduce(lat_hist, dist.ReduceOp.SUM).cpu().numpy()
    return job_finalize(mom, m2, hist, lh, n_dc, bin_s, end_time, quantiles)


def job_ensemble(engine, quantiles: Sequence[float] = DEFAULT_QUANTILES) -> JobEnsembleResult:
    """Statistics of the job-log ensemble of ``engine`` (a finished BatchedEngine with enable_job_ensemble()), over all
    ranks when torch.distributed runs with world > 1 (every rank calls this)."""
    import torch
    dev = torch.device("cuda", engine.device)
    n_dc = engine.spec.n_dc
    cols = (engine.job_ensemble_windows + 1) * len(JOB_FIELDS) * n_dc * 2

    def moments():
        out = torch.zeros((4, cols), dtype=torch.float64, device=dev)
        torch.cuda.synchronize(dev)                    # the library runs on the handle's stream, torch on its own
        engine.job_ensemble_moments_into(out.data_ptr())
        torch.cuda.synchronize(dev)
        return out

    def spread(mean, lo, hi):
        m2 = torch.zeros(cols, dtype=torch.float64, device=dev)
        hist = torch.zeros((cols, BINS), dtype=torch.int64, device=dev)
        torch.cuda.synchronize(dev)
        engine.job_ensemble_spread_into(mean.data_ptr(), lo.data_ptr(), hi.data_ptr(), m2.data_ptr(), hist.data_ptr())
        torch.cuda.synchronize(dev)
        return m2, hist

    lat_hist = torch.from_numpy(engine.dc_latency_histogram().astype(np.int64)).to(dev)
    return _job_passes(moments, spread, lat_hist, n_dc, engine.job_ensemble_bin,
                       engine.spec.end_time, quantiles)


def job_ensemble_from_rows(rows: np.ndarray, hist: np.ndarray, status: np.ndarray, bin_s: float, end_time: float,
                           quantiles: Sequence[float] = DEFAULT_QUANTILES) -> JobEnsembleResult:
    """The same statistics from host rows [W + 1, 2, n_dc, 2, R] and per-DC histograms [n_dc, 2, LAT_BINS, R] (the
    layout of BatchedEngine.job_ensemble_rows) through the numpy mirror; replicas with status != 0 are left out.
    All-reduced over the ranks like job_ensemble."""
    import torch
    n_dc = rows.shape[2]
    x, ok = _job_columns(rows, status)
    width_of = lambda lo, hi: bin_widths_for(lo, hi, _job_integral(x.shape[0], n_dc))  # noqa: E731
    good = np.asarray(status) == 0
    lat_hist = torch.from_numpy(np.asarray(hist)[..., good].astype(np.int64).sum(axis=-1))
    return _job_passes(lambda: torch.from_numpy(moments_cols(x, ok)),
                       lambda mean, lo, hi: tuple(torch.from_numpy(np.ascontiguousarray(a).astype(dt)) for a, dt in
                                                  zip(spread_cols(x, ok, mean.numpy(), lo.numpy(), hi.numpy(),
                                                                  width_of(lo.numpy(), hi.numpy())),
                                                      (np.float64, np.int64))),
                       lat_hist, n_dc, bin_s, end_time, quantiles)
