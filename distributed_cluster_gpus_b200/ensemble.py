"""Batch-wide cluster-log and job-log statistics: per log tick, the mean, spread and quantiles of every DC's
cluster_log.csv columns, and per finish window the same of every DC's job counts and mean latencies, over all replicas
of the batch (all GPUs of a sharded run).

The device records, for every replica, the values its cluster_log.csv rows would hold at every log tick
(``BatchedEngine.enable_cluster_ensemble``).  Two reductions turn them into statistics per column (tick, field, DC):

  moments  n, sum, min, max              -> all-reduce (SUM for n / sum, MIN, MAX)
  spread   sum (x - mean)^2, histogram   -> all-reduce (SUM), given the GLOBAL mean, min and max

Only n, min, max and the histograms cross GPUs exactly: they, and the quantiles read off the histograms, do not depend
on the number of GPUs.  Mean and std do only up to summation order.  ``moments_cols`` / ``spread_cols`` are the numpy
mirror of the two kernels (csrc dcsim_ens_moments_kernel / dcsim_ens_spread_kernel), as ``sharding.aggregate_rows``
mirrors dcsim_reduce_kernel; they run over a statistic's column view (x, ok) [columns, replicas], the values and which
of them count.  Every statistic runs its passes through ``device_passes`` or ``host_passes`` and turns the all-reduced
sums into per-column statistics with ``column_stats``.

The job-log ensemble (``BatchedEngine.enable_job_ensemble``, ``job_ensemble``) runs the same two passes over columns
(row, field, DC, job type): rows are finish windows of ``bin_s`` seconds plus the whole run, fields ``JOB_FIELDS``.
Waiting and response times (``BatchedEngine.enable_job_waits``, ``job_waits``) use the same rows and cells, fields
``WAIT_FIELDS``.
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
def moments_cols(x: np.ndarray, m: np.ndarray) -> np.ndarray:
    """x [columns, R] values, m [columns, R] which of them count -> [4, columns] {n, sum, min, max}; an empty column is
    0, 0, +inf, -inf."""
    out = np.empty((4, x.shape[0]))
    out[0] = m.sum(axis=1)
    out[1] = np.where(m, x, 0.0).sum(axis=1)
    out[2] = np.where(m, x, np.inf).min(axis=1)
    out[3] = np.where(m, x, -np.inf).max(axis=1)
    return out


def bin_widths_for(lo: np.ndarray, hi: np.ndarray, integral: np.ndarray) -> np.ndarray:
    """Per column: the histogram's bin width (0: every value in bin 0) given which columns are integer fields — the
    kernel's rule, the kernel's float ops."""
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


def spread_cols(x: np.ndarray, ok: np.ndarray, mean, lo, hi, width):
    """x [columns, R], ok [columns, R], per-column mean / lo / width -> (m2 [columns] = sum (x - mean)^2 over the values
    that count, hist [columns, BINS] uint64)."""
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
class ColumnStats:
    """Per-column statistics of the all-reduced passes; arrays are [columns], quantiles [Q, columns]."""
    n: np.ndarray
    mean: np.ndarray
    var: np.ndarray                                    # unbiased (ddof = 1); 0 for a single sample
    std: np.ndarray
    min: np.ndarray
    max: np.ndarray
    q: Tuple[float, ...]
    quantiles: np.ndarray

    def result_fields(self, shape) -> dict:
        """n, mean, std, min, max, q and quantiles with the columns laid out as ``shape``: the fields the result
        classes share."""
        return dict(n=self.n.reshape(shape), mean=self.mean.reshape(shape), std=self.std.reshape(shape),
                    min=self.min.reshape(shape), max=self.max.reshape(shape), q=self.q,
                    quantiles=self.quantiles.reshape(self.quantiles.shape[:1] + tuple(shape)))


def column_stats(mom: np.ndarray, m2: np.ndarray, hist: np.ndarray, integral: np.ndarray,
                 quantiles: Sequence[float]) -> ColumnStats:
    """All-reduced moments [4, columns], m2 [columns] and histograms [columns, BINS], and which columns are integer
    fields -> statistics; an empty column has NaN mean, std, min, max and quantiles."""
    n, s, lo, hi = (np.asarray(a, dtype=np.float64) for a in mom)
    with np.errstate(invalid="ignore", divide="ignore"):
        mean = np.where(n > 0, s / n, np.nan)
        var = np.where(n > 1, np.asarray(m2, dtype=np.float64) / (n - 1), np.where(n == 1, 0.0, np.nan))
    empty = n == 0
    qv = hist_quantiles(np.asarray(hist), n, lo, hi, bin_widths_for(lo, hi, integral), integral, quantiles)
    return ColumnStats(n=n.astype(np.int64), mean=mean, var=var, std=np.sqrt(var), min=np.where(empty, np.nan, lo),
                       max=np.where(empty, np.nan, hi), q=tuple(float(q) for q in quantiles), quantiles=qv)


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


def _cluster_columns(rows: np.ndarray, nlog: np.ndarray):
    """rows [ticks, FIELDS, n_dc, R], nlog [R] (ticks each replica recorded) -> (x, ok) [columns, R], columns
    (tick, field, dc) as the kernels'; replica r counts in the ticks it recorded."""
    R = rows.shape[-1]
    ok = np.arange(rows.shape[0])[:, None, None, None] < np.asarray(nlog)[None, None, None, :]
    return rows.reshape(-1, R), np.broadcast_to(ok, rows.shape).reshape(-1, R)


def _cluster_integral(n_cols: int, n_dc: int) -> np.ndarray:
    return np.isin((np.arange(n_cols) // n_dc) % len(FIELDS), INTEGER_FIELDS)


def finalize(mom: np.ndarray, m2: np.ndarray, hist: np.ndarray, n_dc: int, log_interval: float,
             quantiles: Sequence[float] = DEFAULT_QUANTILES) -> EnsembleResult:
    """All-reduced moments [4, columns], m2 [columns] and histograms [columns, BINS] -> statistics.  Trailing ticks no
    replica recorded are dropped."""
    F = len(FIELDS)
    mom = np.asarray(mom, dtype=np.float64)
    per_tick = mom[0].reshape(-1, F * n_dc).max(axis=1)
    T = int(np.nonzero(per_tick > 0)[0].max()) + 1 if np.any(per_tick > 0) else 0
    c = T * F * n_dc
    st = column_stats(mom[:, :c], np.asarray(m2)[:c], np.asarray(hist)[:c], _cluster_integral(c, n_dc), quantiles)
    return EnsembleResult(time_s=tick_times(log_interval, T), fields=FIELDS, **st.result_fields((T, F, n_dc)))


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


def _allreduce_sum(t) -> np.ndarray:
    import torch.distributed as dist
    return _allreduce(t, dist.ReduceOp.SUM).cpu().numpy()


def two_passes(moments_fn, spread_fn):
    """moments_fn() -> torch [4, columns] float64; spread_fn(mean, lo, hi) -> (m2 [columns] float64, hist [columns, BINS]
    int64), torch tensors on one device.  Runs pass 1, all-reduces it, pass 2 on the global mean / min / max, all-reduces
    that -> host (moments, m2, hist)."""
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


def device_passes(dev, cols: int, moments_into, spread_into, stat_cols: int = None):
    """two_passes over a device recorder of ``cols`` columns: ``moments_into(out_ptr)`` and ``spread_into(mean_ptr,
    lo_ptr, hi_ptr, m2_ptr, hist_ptr)`` (a BatchedEngine's ``*_into`` methods), the spread over the first ``stat_cols``
    columns (None: all of them)."""
    import torch
    stat_cols = cols if stat_cols is None else stat_cols

    def moments():
        out = torch.zeros((4, cols), dtype=torch.float64, device=dev)
        if cols:
            torch.cuda.synchronize(dev)                # the library runs on the handle's stream, torch on its own
            moments_into(out.data_ptr())
            torch.cuda.synchronize(dev)
        return out

    def spread(mean, lo, hi):
        m2 = torch.zeros(stat_cols, dtype=torch.float64, device=dev)
        hist = torch.zeros((stat_cols, BINS), dtype=torch.int64, device=dev)
        if cols:
            torch.cuda.synchronize(dev)
            spread_into(mean.data_ptr(), lo.data_ptr(), hi.data_ptr(), m2.data_ptr(), hist.data_ptr())
            torch.cuda.synchronize(dev)
        return m2, hist

    return two_passes(moments, spread)


def host_passes(x: np.ndarray, ok: np.ndarray, integral: np.ndarray, stat_cols: int = None):
    """two_passes through the numpy mirror of the kernels over the columns x [columns, R] (ok [columns, R]: the values
    that count), the spread over the first ``stat_cols`` columns (None: all of them), ``integral`` [stat_cols] the
    integer fields among them."""
    import torch
    c = slice(stat_cols)

    def spread(mean, lo, hi):
        lo, hi = lo.numpy()[c], hi.numpy()[c]
        m2, hist = spread_cols(x[c], ok[c], mean.numpy()[c], lo, hi, bin_widths_for(lo, hi, integral))
        return torch.from_numpy(m2.astype(np.float64)), torch.from_numpy(hist.astype(np.int64))

    return two_passes(lambda: torch.from_numpy(moments_cols(x, ok)), spread)


def cluster_ensemble(engine, quantiles: Sequence[float] = DEFAULT_QUANTILES) -> EnsembleResult:
    """Statistics of the cluster-log ensemble of ``engine`` (a finished BatchedEngine with enable_cluster_ensemble()),
    over all ranks when torch.distributed runs with world > 1 (every rank calls this).  Raises RecorderOverflow if a
    replica recorded more ticks than the capacity."""
    import torch
    dev = torch.device("cuda", engine.device)
    cols = engine.cluster_ensemble_capacity * len(FIELDS) * engine.spec.n_dc
    passes = device_passes(dev, cols, engine.ensemble_moments_into, engine.ensemble_spread_into)
    return finalize(*passes, engine.spec.n_dc, engine.spec.log_interval, quantiles)


def cluster_ensemble_from_rows(rows: np.ndarray, nlog: np.ndarray, log_interval: float,
                               quantiles: Sequence[float] = DEFAULT_QUANTILES) -> EnsembleResult:
    """The same statistics from host rows [ticks, FIELDS, n_dc, R] through the numpy mirror (all-reduced over the ranks
    like cluster_ensemble)."""
    n_dc = rows.shape[2]
    x, ok = _cluster_columns(rows, nlog)
    return finalize(*host_passes(x, ok, _cluster_integral(x.shape[0], n_dc)), n_dc, log_interval, quantiles)


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
    mom = np.asarray(mom, dtype=np.float64)
    rows = mom.shape[1] // (F * n_dc * J)
    shape = (rows, F, n_dc, J)
    st = column_stats(mom, m2, hist, _job_integral(mom.shape[1], n_dc), quantiles)
    s4 = mom[1].reshape(shape)
    with np.errstate(invalid="ignore", divide="ignore"):
        pooled = np.where(s4[:, 0] > 0, s4[:, 1] / s4[:, 0], np.nan)
    k = np.arange(rows - 1, dtype=np.float64)
    return JobEnsembleResult(t0_s=np.append(k * bin_s, 0.0), t1_s=np.append((k + 1.0) * bin_s, float(end_time)),
                             bin_s=float(bin_s), end_time=float(end_time), fields=JOB_FIELDS, **st.result_fields(shape),
                             pooled_mean_latency_s=pooled,
                             latency_histogram=np.asarray(lat_hist).astype(np.uint64).reshape(n_dc, J, LAT_BINS))


def job_ensemble(engine, quantiles: Sequence[float] = DEFAULT_QUANTILES) -> JobEnsembleResult:
    """Statistics of the job-log ensemble of ``engine`` (a finished BatchedEngine with enable_job_ensemble()), over all
    ranks when torch.distributed runs with world > 1 (every rank calls this)."""
    import torch
    dev = torch.device("cuda", engine.device)
    n_dc = engine.spec.n_dc
    cols = (engine.job_ensemble_windows + 1) * len(JOB_FIELDS) * n_dc * 2
    passes = device_passes(dev, cols, engine.job_ensemble_moments_into, engine.job_ensemble_spread_into)
    lat_hist = _allreduce_sum(torch.from_numpy(engine.dc_latency_histogram().astype(np.int64)).to(dev))
    return job_finalize(*passes, lat_hist, n_dc, engine.job_ensemble_bin, engine.spec.end_time, quantiles)


def job_ensemble_from_rows(rows: np.ndarray, hist: np.ndarray, status: np.ndarray, bin_s: float, end_time: float,
                           quantiles: Sequence[float] = DEFAULT_QUANTILES) -> JobEnsembleResult:
    """The same statistics from host rows [W + 1, 2, n_dc, 2, R] and per-DC histograms [n_dc, 2, LAT_BINS, R] (the
    layout of BatchedEngine.job_ensemble_rows) through the numpy mirror; replicas with status != 0 are left out.
    All-reduced over the ranks like job_ensemble."""
    import torch
    n_dc = rows.shape[2]
    x, ok = _job_columns(rows, status)
    passes = host_passes(x, ok, _job_integral(x.shape[0], n_dc))
    good = np.asarray(status) == 0
    lat_hist = _allreduce_sum(torch.from_numpy(np.asarray(hist)[..., good].astype(np.int64).sum(axis=-1)))
    return job_finalize(*passes, lat_hist, n_dc, bin_s, end_time, quantiles)


# ---- waiting and response times ---------------------------------------------------------------------------------------
WAIT_FIELDS = ("waited", "wait_sum", "resp_sum", "mean_wait_s", "mean_response_s")   # DCSIM_JWAIT_* order
WAIT_CSV_FIELDS = ("waited", "mean_wait_s", "mean_response_s")


def _wait_columns(rows: np.ndarray, jobs: np.ndarray, status: np.ndarray):
    """rows [W + 1, 3, n_dc, 2, R] {waited, wait_sum, resp_sum}, jobs [W + 1, n_dc, 2, R] (the job ensemble's counts) ->
    (x, ok) [columns, R], columns (row, WAIT_FIELDS, dc, jtype) as the kernels'."""
    R = rows.shape[-1]
    with np.errstate(invalid="ignore", divide="ignore"):
        x = np.concatenate([rows, rows[:, 1:3] / jobs[:, None]], axis=1)
    good = np.broadcast_to((np.asarray(status) == 0)[None, None, None, :], jobs.shape)
    has = good & (jobs > 0)
    ok = np.stack([good, good, good, has, has], axis=1)
    return x.reshape(-1, R), ok.reshape(-1, R)


def _wait_integral(n_cols: int, n_dc: int) -> np.ndarray:
    return (np.arange(n_cols) // (2 * n_dc)) % len(WAIT_FIELDS) == 0


def zero_share_quantiles(hist_row, zero_share: float, qs) -> list:
    """latency_quantiles of one wait histogram row, except that a quantile whose share lies at or below ``zero_share``
    (the jobs that did not wait: their bin 0 also holds waits below 2^-20 s) is exactly 0."""
    from .engine import latency_quantiles
    vals = latency_quantiles(hist_row, qs)
    return [0.0 if float(q) <= zero_share and np.asarray(hist_row).sum() else v for q, v in zip(qs, vals)]


@dataclass
class JobWaitsResult:
    """Per (row, field, dc, jtype) statistics over every replica of the batch; arrays are [W + 1, len(fields), n_dc, 2],
    rows as JobEnsembleResult's.  wait = start - xfer_done (the time in the DC's FIFO), response = finish - arrival."""
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
    jobs: np.ndarray                                   # [n_dc, 2]: finished jobs of the valid replicas, whole run
    waited: np.ndarray                                 # [n_dc, 2]: of them, jobs whose wait was > 0
    wait_sum: np.ndarray                               # [n_dc, 2]: their waits' sum (pooled over replicas)
    resp_sum: np.ndarray                               # [n_dc, 2]: their response times' sum
    wait_histogram: np.ndarray                         # [n_dc, 2 kinds (wait, response), 2, LAT_BINS] uint64

    def quantile_names(self):
        return [f"p{int(round(q * 100)):02d}" for q in self.q]

    def zero_wait_share(self, d: int, jt: int) -> float:
        """1 - waited / jobs of DC d and type jt (whole run, pooled): the share of jobs that did not wait."""
        return 1.0 - float(self.waited[d, jt]) / float(self.jobs[d, jt]) if self.jobs[d, jt] else float("nan")

    def wait_quantiles(self, d: int, jt: int, qs=None) -> list:
        """Quantiles [s] of the wait of DC d's jobs of type jt, pooled over the replicas (log-binned; exactly 0 at or below
        the zero-wait share)."""
        return zero_share_quantiles(self.wait_histogram[d, 0, jt], self.zero_wait_share(d, jt), self.q if qs is None else qs)

    def response_quantiles(self, d: int, jt: int, qs=None) -> list:
        from .engine import latency_quantiles
        return latency_quantiles(self.wait_histogram[d, 1, jt], self.q if qs is None else qs)

    def pooled(self, qs=(0.5, 0.95, 0.99)) -> dict:
        """Per job type over all DCs: pooled mean / quantiles of wait and response, and waited_share."""
        from .engine import latency_quantiles
        out = {}
        for jt, name in enumerate(JOB_TYPES):
            jobs, waited = float(self.jobs[:, jt].sum()), float(self.waited[:, jt].sum())
            wh, rh = self.wait_histogram[:, 0, jt].sum(axis=0), self.wait_histogram[:, 1, jt].sum(axis=0)
            share = 1.0 - waited / jobs if jobs else float("nan")
            e = {"jobs": int(jobs), "waited_share": waited / jobs if jobs else float("nan"),
                 "mean_wait_s": float(self.wait_sum[:, jt].sum()) / jobs if jobs else float("nan"),
                 "mean_response_s": float(self.resp_sum[:, jt].sum()) / jobs if jobs else float("nan")}
            for q, v in zip(qs, zero_share_quantiles(wh, share, qs)):
                e[f"p{int(round(q * 100)):02d}_wait_s"] = v
            for q, v in zip(qs, latency_quantiles(rh, qs)):
                e[f"p{int(round(q * 100)):02d}_response_s"] = v
            out[name] = e
        return out

    def to_csv(self, path: str, dc_names: Sequence[str]):
        """The job ensemble's long format (t0_s,t1_s,dc,type,field,n,mean,std,min,p05,...,p95,max).  Per window, then for
        the whole run, the rows of ``waited``, ``mean_wait_s`` and ``mean_response_s`` per DC and type; then per DC and
        type three whole-run rows: ``wait_s`` and ``response_s`` (n = jobs, mean = the pooled mean, quantiles from the
        per-DC histograms, wait quantiles exactly 0 at or below the zero-wait share; std / min / max empty) and
        ``waited_share`` (mean = waited / jobs)."""
        rows, F, D, J = self.n.shape
        keep = [self.fields.index(f) for f in WAIT_CSV_FIELDS]
        nan = float("nan")
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
            head = [repr(0.0), repr(float(self.end_time))]
            for d in range(D):
                for jt in range(J):
                    jobs = float(self.jobs[d, jt])
                    for name, s_, qv in (("wait_s", self.wait_sum, self.wait_quantiles(d, jt)),
                                         ("response_s", self.resp_sum, self.response_quantiles(d, jt))):
                        w.writerow(head + [dc_names[d], JOB_TYPES[jt], name, int(jobs),
                                           repr(float(s_[d, jt]) / jobs if jobs else nan), "", ""]
                                   + [repr(float(v)) for v in qv] + [""])
                    w.writerow(head + [dc_names[d], JOB_TYPES[jt], "waited_share", int(jobs),
                                       repr(float(self.waited[d, jt]) / jobs if jobs else nan), "", ""]
                               + [""] * len(self.q) + [""])


def waits_finalize(mom, m2, hist, wait_hist, n_dc: int, bin_s: float, end_time: float,
                   quantiles: Sequence[float] = DEFAULT_QUANTILES) -> JobWaitsResult:
    """All-reduced moments [4, columns], m2, histograms [columns, BINS] and per-DC wait / response histograms ->
    statistics."""
    F, J = len(WAIT_FIELDS), 2
    mom = np.asarray(mom, dtype=np.float64)
    rows = mom.shape[1] // (F * n_dc * J)
    shape = (rows, F, n_dc, J)
    st = column_stats(mom, m2, hist, _wait_integral(mom.shape[1], n_dc), quantiles)
    s4 = mom[1].reshape(shape)[-1]                     # whole-run sums over the valid replicas
    wh = np.asarray(wait_hist).astype(np.uint64).reshape(n_dc, 2, J, LAT_BINS)
    k = np.arange(rows - 1, dtype=np.float64)
    return JobWaitsResult(t0_s=np.append(k * bin_s, 0.0), t1_s=np.append((k + 1.0) * bin_s, float(end_time)),
                          bin_s=float(bin_s), end_time=float(end_time), fields=WAIT_FIELDS, **st.result_fields(shape),
                          jobs=wh[:, 0].sum(axis=-1), waited=s4[0], wait_sum=s4[1], resp_sum=s4[2], wait_histogram=wh)


def job_waits(engine, quantiles: Sequence[float] = DEFAULT_QUANTILES) -> JobWaitsResult:
    """Statistics of the waiting / response-time recorder of ``engine`` (a finished BatchedEngine with enable_job_waits()),
    over all ranks when torch.distributed runs with world > 1 (every rank calls this)."""
    import torch
    if not engine.job_waits_enabled:
        raise RuntimeError("job waits not enabled (enable_job_waits)")
    dev = torch.device("cuda", engine.device)
    n_dc = engine.spec.n_dc
    cols = (engine.job_ensemble_windows + 1) * len(WAIT_FIELDS) * n_dc * 2
    passes = device_passes(dev, cols, engine.job_waits_moments_into, engine.job_waits_spread_into)
    wait_hist = _allreduce_sum(torch.from_numpy(engine.dc_wait_histogram().astype(np.int64)).to(dev))
    return waits_finalize(*passes, wait_hist, n_dc, engine.job_ensemble_bin, engine.spec.end_time, quantiles)


def job_waits_from_rows(rows: np.ndarray, hist: np.ndarray, jobs: np.ndarray, status: np.ndarray, bin_s: float,
                        end_time: float, quantiles: Sequence[float] = DEFAULT_QUANTILES) -> JobWaitsResult:
    """The same statistics from host rows [W + 1, 3, n_dc, 2, R], per-DC histograms [n_dc, 2 kinds, 2, LAT_BINS, R]
    (BatchedEngine.job_waits_rows) and the job ensemble's counts [W + 1, n_dc, 2, R] (job_ensemble_rows()[0][:, 0])
    through the numpy mirror; replicas with status != 0 are left out.  All-reduced over the ranks like job_waits."""
    import torch
    n_dc = rows.shape[2]
    x, ok = _wait_columns(rows, jobs, status)
    passes = host_passes(x, ok, _wait_integral(x.shape[0], n_dc))
    good = np.asarray(status) == 0
    wait_hist = _allreduce_sum(torch.from_numpy(np.asarray(hist)[..., good].astype(np.int64).sum(axis=-1)))
    return waits_finalize(*passes, wait_hist, n_dc, bin_s, end_time, quantiles)


# ---- job resources: GPUs, frequency and predicted energy of every finished job ---------------------------------------
RES_FIELDS = ("gpu_sum", "freq_sum", "energy_sum", "mean_gpus", "mean_freq_ghz", "mean_energy_j")   # DCSIM_JRES_* order
RES_CSV_FIELDS = ("mean_gpus", "mean_freq_ghz", "mean_energy_j")
RES_EBINS = 128                                        # DCSIM_JRES_EBINS
RES_MAX_FREQ = 16                                      # DCSIM_MAX_FREQ: the mix's frequency stride
RES_OCT = (float.fromhex("0x1.306fe0a31b716p+0"), float.fromhex("0x1.6a09e667f3bcdp+0"),
           float.fromhex("0x1.ae89f995ad3aep+0"))     # DCSIM_JRES_OCT1..3: the smallest doubles >= 2^(1/4, 1/2, 3/4)


def energy_bin(e) -> np.ndarray:
    """dcsim_jres_ebin: clamp(floor(4 * log2(E)), 0, RES_EBINS - 1), decided exactly from the binary exponent and the
    significand's place among RES_OCT."""
    e = np.asarray(e, dtype=np.float64)
    m, ex = np.frexp(np.where(e >= 1.0, e, 1.0))
    m = 2.0 * m
    b = 4 * (ex.astype(np.int64) - 1) + sum((m >= t).astype(np.int64) for t in RES_OCT)
    return np.where(e >= 1.0, np.minimum(b, RES_EBINS - 1), 0)


def energy_bin_edges() -> np.ndarray:
    """Lower edges [J] of the RES_EBINS energy bins (+ the upper edge of the last): 2^(k / 4)."""
    return 2.0 ** (np.arange(RES_EBINS + 1) / 4.0)


def _res_columns(rows: np.ndarray, mix: np.ndarray, hist: np.ndarray, jobs: np.ndarray, status: np.ndarray):
    """rows [W + 1, 3, n_dc, 2, R] {gpu_sum, freq_sum, energy_sum}, mix [n_dc, 2, G * RES_MAX_FREQ + 1, R] (the stored
    layout, OFF_LEVEL last), hist [n_dc, 2, RES_EBINS, R], jobs [W + 1, n_dc, 2, R] (the job ensemble's counts) ->
    (x, ok) [columns, R] as the kernels' column source: the windowed (row, RES_FIELDS, dc, jtype) columns, then the mix
    and the energy bins as stored."""
    R = rows.shape[-1]
    with np.errstate(invalid="ignore", divide="ignore"):
        x = np.concatenate([rows, rows / jobs[:, None]], axis=1)
    good = np.broadcast_to((np.asarray(status) == 0)[None, None, None, :], jobs.shape)
    has = good & (jobs > 0)
    ok = np.stack([good, good, good, has, has, has], axis=1)
    counts = np.concatenate([np.asarray(mix).reshape(-1, R), np.asarray(hist).reshape(-1, R)]).astype(np.float64)
    x = np.concatenate([x.reshape(-1, R), counts])
    ok = np.concatenate([ok.reshape(-1, R), np.broadcast_to((np.asarray(status) == 0)[None, :], counts.shape)])
    return x, ok


def _res_integral(n_cols: int, n_dc: int) -> np.ndarray:
    return (np.arange(n_cols) // (2 * n_dc)) % len(RES_FIELDS) == 0


@dataclass
class JobResourcesResult:
    """Per (row, field, dc, jtype) statistics over every replica of the batch; arrays are [W + 1, len(fields), n_dc, 2],
    rows as JobEnsembleResult's.  Per job: g its GPU count, f its frequency [GHz] (f_used), E_job = E_pred * size its
    predicted energy [J].  Whole run, pooled over the valid replicas: ``mix`` [n_dc, 2, G, RES_MAX_FREQ] jobs per GPU
    count (row g - 1; the last row holds g >= G) and frequency level (column q: ``levels[d, q]``, NaN past the DC's
    levels), ``off_level`` [n_dc, 2] jobs whose f matched no level, ``energy_histogram`` [n_dc, 2, RES_EBINS]."""
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
    levels: np.ndarray                                 # [n_dc, RES_MAX_FREQ] frequency levels [GHz], NaN past n_freq
    jobs: np.ndarray                                   # [n_dc, 2]: finished jobs of the valid replicas, whole run
    gpu_sum: np.ndarray                                # [n_dc, 2]: their sums, pooled over replicas
    freq_sum: np.ndarray
    energy_sum: np.ndarray
    mix: np.ndarray                                    # [n_dc, 2, G, RES_MAX_FREQ] uint64
    off_level: np.ndarray                              # [n_dc, 2] uint64
    energy_histogram: np.ndarray                       # [n_dc, 2, RES_EBINS] uint64

    def quantile_names(self):
        return [f"p{int(round(q * 100)):02d}" for q in self.q]

    def mix_shares(self, d: int, jt: int) -> np.ndarray:
        """[G, RES_MAX_FREQ] share of DC d's finished jobs of type jt at each (GPU count, level); NaN without jobs."""
        total = float(self.mix[d, jt].sum() + self.off_level[d, jt])
        return self.mix[d, jt] / total if total else np.full(self.mix[d, jt].shape, np.nan)

    def mix_labels(self, d: int):
        """((g row, level column, label) for every GPU count and level of DC d), label "n{g}_f{level}" ("n{G}+" for the
        last row)."""
        G = self.mix.shape[2]
        out = []
        for gi in range(G):
            for qi in range(self.levels.shape[1]):
                if self.levels[d, qi] == self.levels[d, qi]:
                    out.append((gi, qi, f"n{gi + 1}{'+' if gi == G - 1 else ''}_f{float(self.levels[d, qi])!r}"))
        return out

    def energy_quantiles(self, d: int, jt: int, qs=None) -> list:
        """Quantiles [J] of E_job of DC d's jobs of type jt, pooled over the replicas, log-interpolated in the
        quarter-octave bin that holds each; NaN without jobs."""
        qs = self.q if qs is None else qs
        h = np.asarray(self.energy_histogram[d, jt], dtype=np.float64)
        total = h.sum()
        if total == 0:
            return [float("nan")] * len(qs)
        edges, cum, out = energy_bin_edges(), np.cumsum(h), []
        for q in qs:
            b = min(int(np.searchsorted(cum, q * total, side="left")), RES_EBINS - 1)
            below = cum[b - 1] if b else 0.0
            frac = (q * total - below) / h[b] if h[b] else 0.0
            out.append(float(edges[b] * (edges[b + 1] / edges[b]) ** frac))
        return out

    def pooled(self, qs=(0.5, 0.95, 0.99)) -> dict:
        """Per DC (index) and job type: jobs, pooled mean GPUs / frequency / energy per job, energy quantiles, and the
        (n, f) mix as shares (the occupied cells only, plus off_level)."""
        out = {}
        nan = float("nan")
        for d in range(self.jobs.shape[0]):
            row = {}
            for jt, name in enumerate(JOB_TYPES):
                jobs = float(self.jobs[d, jt])
                e = {"jobs": int(jobs), "mean_gpus": float(self.gpu_sum[d, jt]) / jobs if jobs else nan,
                     "mean_freq_ghz": float(self.freq_sum[d, jt]) / jobs if jobs else nan,
                     "mean_energy_j": float(self.energy_sum[d, jt]) / jobs if jobs else nan}
                for q, v in zip(qs, self.energy_quantiles(d, jt, qs)):
                    e[f"p{int(round(q * 100)):02d}_energy_j"] = v
                shares = self.mix_shares(d, jt)
                e["mix"] = {lab: float(shares[gi, qi]) for gi, qi, lab in self.mix_labels(d) if self.mix[d, jt, gi, qi]}
                e["off_level_share"] = float(self.off_level[d, jt]) / jobs if jobs else nan
                row[name] = e
            out[d] = row
        return out

    def to_csv(self, path: str, dc_names: Sequence[str]):
        """The job ensemble's long format (t0_s,t1_s,dc,type,field,n,mean,std,min,p05,...,p95,max).  Per window, then for
        the whole run, the rows of ``mean_gpus``, ``mean_freq_ghz`` and ``mean_energy_j`` per DC and type; then per DC
        and type the whole-run rows ``energy_j`` (n = jobs, mean = the pooled mean, quantiles from the per-DC histogram;
        std / min / max empty), one ``mix_n{g}_f{level}`` row per GPU count and level (n = jobs, mean = their share) and
        ``mix_off_level``."""
        rows, F, D, J = self.n.shape
        keep = [self.fields.index(f) for f in RES_CSV_FIELDS]
        nan = float("nan")
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
            head = [repr(0.0), repr(float(self.end_time))]
            blank = [""] * len(self.q) + [""]
            for d in range(D):
                for jt in range(J):
                    jobs = float(self.jobs[d, jt])
                    w.writerow(head + [dc_names[d], JOB_TYPES[jt], "energy_j", int(jobs),
                                       repr(float(self.energy_sum[d, jt]) / jobs if jobs else nan), "", ""]
                               + [repr(float(v)) for v in self.energy_quantiles(d, jt)] + [""])
                    shares = self.mix_shares(d, jt)
                    for gi, qi, lab in self.mix_labels(d):
                        w.writerow(head + [dc_names[d], JOB_TYPES[jt], "mix_" + lab, int(self.mix[d, jt, gi, qi]),
                                           repr(float(shares[gi, qi])), "", ""] + blank)
                    w.writerow(head + [dc_names[d], JOB_TYPES[jt], "mix_off_level", int(self.off_level[d, jt]),
                                       repr(float(self.off_level[d, jt]) / jobs if jobs else nan), "", ""] + blank)


def _res_levels(sp) -> np.ndarray:
    lv = np.full((sp.n_dc, RES_MAX_FREQ), np.nan)
    for d in range(sp.n_dc):
        lv[d, :sp.dc[d].n_freq] = [sp.dc[d].freq_levels[q] for q in range(sp.dc[d].n_freq)]
    return lv


def res_finalize(mom, m2, hist, n_dc: int, G: int, levels, bin_s: float, end_time: float,
                 quantiles: Sequence[float] = DEFAULT_QUANTILES) -> JobResourcesResult:
    """All-reduced moments [4, columns] (windowed, then the counts), m2 and histograms over the windowed columns ->
    statistics."""
    F, J = len(RES_FIELDS), 2
    mom = np.asarray(mom, dtype=np.float64)
    mix_cols = G * RES_MAX_FREQ + 1
    win = mom.shape[1] - n_dc * J * (mix_cols + RES_EBINS)
    rows = win // (F * n_dc * J)
    shape = (rows, F, n_dc, J)
    st = column_stats(mom[:, :win], np.asarray(m2)[:win], np.asarray(hist)[:win], _res_integral(win, n_dc), quantiles)
    s4 = mom[1, :win].reshape(shape)[-1]               # whole-run sums over the valid replicas
    mix = np.rint(mom[1, win:win + n_dc * J * mix_cols]).astype(np.uint64).reshape(n_dc, J, mix_cols)
    eh = np.rint(mom[1, win + n_dc * J * mix_cols:]).astype(np.uint64).reshape(n_dc, J, RES_EBINS)
    k = np.arange(rows - 1, dtype=np.float64)
    return JobResourcesResult(t0_s=np.append(k * bin_s, 0.0), t1_s=np.append((k + 1.0) * bin_s, float(end_time)),
                              bin_s=float(bin_s), end_time=float(end_time), fields=RES_FIELDS, **st.result_fields(shape),
                              levels=np.asarray(levels, dtype=np.float64), jobs=eh.sum(axis=-1), gpu_sum=s4[0],
                              freq_sum=s4[1], energy_sum=s4[2], mix=mix[:, :, :-1].reshape(n_dc, J, G, RES_MAX_FREQ),
                              off_level=mix[:, :, -1].copy(), energy_histogram=eh)


def job_resources(engine, quantiles: Sequence[float] = DEFAULT_QUANTILES) -> JobResourcesResult:
    """Statistics of the job-resources recorder of ``engine`` (a finished BatchedEngine with enable_job_resources()),
    over all ranks when torch.distributed runs with world > 1 (every rank calls this)."""
    import torch
    from .engine import jres_mix_g
    if not engine.job_resources_enabled:
        raise RuntimeError("job resources not enabled (enable_job_resources)")
    dev = torch.device("cuda", engine.device)
    sp = engine.spec
    G = jres_mix_g(sp.max_gpus_per_job)
    win = (engine.job_ensemble_windows + 1) * len(RES_FIELDS) * sp.n_dc * 2
    cols = win + sp.n_dc * 2 * (G * RES_MAX_FREQ + 1 + RES_EBINS)
    passes = device_passes(dev, cols, engine.job_resources_moments_into, engine.job_resources_spread_into, stat_cols=win)
    return res_finalize(*passes, sp.n_dc, G, _res_levels(sp), engine.job_ensemble_bin, sp.end_time, quantiles)


def job_resources_from_rows(rows: np.ndarray, mix: np.ndarray, off_level: np.ndarray, hist: np.ndarray, jobs: np.ndarray,
                            status: np.ndarray, levels, bin_s: float, end_time: float,
                            quantiles: Sequence[float] = DEFAULT_QUANTILES) -> JobResourcesResult:
    """The same statistics from host arrays in the layout of BatchedEngine.job_resources_rows — rows [W + 1, 3, n_dc, 2,
    R], mix [n_dc, 2, G, RES_MAX_FREQ, R], off_level [n_dc, 2, R], hist [n_dc, 2, RES_EBINS, R] — the job ensemble's
    counts [W + 1, n_dc, 2, R] (job_ensemble_rows()[0][:, 0]) and the levels [n_dc, RES_MAX_FREQ] (NaN past a DC's
    n_freq), through the numpy mirror of both passes; replicas with status != 0 are left out.  All-reduced over the
    ranks like job_resources."""
    n_dc, G, R = rows.shape[2], mix.shape[2], rows.shape[-1]
    stored = np.concatenate([np.asarray(mix).reshape(n_dc, 2, G * RES_MAX_FREQ, R),
                             np.asarray(off_level).reshape(n_dc, 2, 1, R)], axis=2)
    x, ok = _res_columns(rows, stored, hist, jobs, status)
    win = rows.shape[0] * len(RES_FIELDS) * n_dc * 2
    passes = host_passes(x, ok, _res_integral(win, n_dc), win)
    return res_finalize(*passes, n_dc, G, levels, bin_s, end_time, quantiles)


# ---- power profile ---------------------------------------------------------------------------------------------------
PP_FIELDS = ("profile_s", "peak_w", "t_peak_s", "over_s", "over_j", "excursions", "longest_over_s", "out_of_range")
PP_INTEGER_FIELDS = (5, 7)                             # excursions, out_of_range: unit bins, exact quantiles
PP_BINS = 1024                                         # DCSIM_PP_BINS
PP_CURVE_LEVELS = (0.5, 0.1, 0.01, 0.001)              # shares of the pooled time the CSV's power_w_time row reports
PP_CSV_HEADER = ["dc", "field", "n", "mean", "std", "min", "p05", "p25", "p50", "p75", "p95", "p99", "max"]
PP_CSV_QUANTILES = (0.05, 0.25, 0.5, 0.75, 0.95, 0.99)


def _pp_integral(n_cols: int) -> np.ndarray:
    return np.isin(np.arange(n_cols), PP_INTEGER_FIELDS)


def pp_bin_edges(hi: float) -> np.ndarray:
    """Edges of the power histogram: PP_BINS bins of hi / PP_BINS watts over [0, hi]."""
    return np.arange(PP_BINS + 1, dtype=np.float64) * (float(hi) / PP_BINS)


@dataclass
class PowerProfileResult:
    """Batch statistics of the power profile over the replicas with status 0.  ``n`` ... ``max`` and ``quantiles``
    ([Q, columns]) cover the columns ``columns`` — the per-replica fields (PP_FIELDS), then ``dc_peak_w`` per DC.
    ``duration_curve``: (bin edges [PP_BINS + 1] W, pooled seconds [PP_BINS]) summed over the replicas — how long the
    pooled simulated time spent in each power bin."""
    columns: Tuple[Tuple[str, int], ...]               # (field, dc); dc = -1 for the per-replica fields
    n: np.ndarray
    mean: np.ndarray
    std: np.ndarray                                    # unbiased (ddof = 1); 0 for a single sample
    min: np.ndarray
    max: np.ndarray
    q: Tuple[float, ...]
    quantiles: np.ndarray
    hi: float
    threshold: float                                   # +inf: none
    duration_curve: Tuple[np.ndarray, np.ndarray]
    pooled_energy_j: float                             # sum of the replicas' total energy

    def column(self, field: str, dc: int = -1) -> int:
        return self.columns.index((field, dc))

    @property
    def replicas(self) -> int:
        return int(self.n[0]) if len(self.n) else 0

    @property
    def pooled_time_s(self) -> float:
        return float(self.duration_curve[1].sum())

    @property
    def mean_power_w(self) -> float:
        """Pooled energy / pooled profile time."""
        t = self.pooled_time_s
        return self.pooled_energy_j / t if t > 0 else float("nan")

    @property
    def over_share(self) -> float:
        """Share of the pooled time above the threshold (NaN without one)."""
        if not math.isfinite(self.threshold):
            return float("nan")
        t = self.pooled_time_s
        s = float(self.mean[self.column("over_s")]) * self.replicas
        return s / t if t > 0 else float("nan")

    def time_quantiles(self, shares: Sequence[float]) -> np.ndarray:
        """The power levels exceeded for the given shares of the pooled time (0.01: the level the cluster was at or
        above for 1 % of the time), read off the pooled curve: the centre of the bin where the share is crossed, within
        one bin width."""
        edges, sec = self.duration_curve
        total = sec.sum()
        out = np.full(len(shares), np.nan)
        if total <= 0:
            return out
        above = np.cumsum(sec[::-1])[::-1]             # time at or above the bottom of each bin
        for i, s in enumerate(shares):
            k = np.nonzero(above >= float(s) * total)[0]
            b = int(k.max()) if len(k) else 0
            out[i] = 0.5 * (edges[b] + edges[b + 1])
        return out

    def to_csv(self, path: str, dc_names: Sequence[str]):
        """Long format: dc,field,n,mean,std,min,p05,p25,p50,p75,p95,p99,max — one row per field (dc empty), one per DC
        for dc_peak_w; with no threshold the threshold columns are left empty.  A last ``power_w_time`` row holds the
        pooled curve: n = replicas, mean = pooled energy / pooled time, std empty, min / max the lowest / highest occupied
        bin's centre, the quantiles the power levels exceeded for 95 / 75 / 50 / 25 / 5 / 1 % of the pooled time."""
        thr_fields = ("over_s", "over_j", "excursions", "longest_over_s")
        fmt = lambda x: repr(float(x))  # noqa: E731
        with open(path, "w", newline="") as f:
            w = csv.writer(f)
            w.writerow(PP_CSV_HEADER)
            for c, (field, d) in enumerate(self.columns):
                dc = dc_names[d] if d >= 0 else ""
                if field in thr_fields and not math.isfinite(self.threshold):
                    w.writerow([dc, field] + [""] * (len(PP_CSV_HEADER) - 2))
                    continue
                w.writerow([dc, field, int(self.n[c]), fmt(self.mean[c]), fmt(self.std[c]), fmt(self.min[c])]
                           + [fmt(self.quantiles[j, c]) for j in range(len(self.q))] + [fmt(self.max[c])])
            edges, sec = self.duration_curve
            occ = np.nonzero(sec > 0)[0]
            centre = lambda b: 0.5 * (edges[b] + edges[b + 1])  # noqa: E731
            lo = centre(occ.min()) if len(occ) else float("nan")
            hi = centre(occ.max()) if len(occ) else float("nan")
            tq = self.time_quantiles([1.0 - q for q in PP_CSV_QUANTILES])
            w.writerow(["", "power_w_time", self.replicas, fmt(self.mean_power_w), "", fmt(lo)]
                       + [fmt(v) for v in tq] + [fmt(hi)])


def pp_finalize(mom, m2, hist, n_dc: int, hi: float, threshold: float, energy: float,
                quantiles: Sequence[float] = PP_CSV_QUANTILES) -> PowerProfileResult:
    """All-reduced moments [4, PP_FIELDS + n_dc + PP_BINS], m2 and histograms over the first PP_FIELDS + n_dc columns,
    and the pooled energy -> statistics."""
    mom = np.asarray(mom, dtype=np.float64)
    c = len(PP_FIELDS) + n_dc
    st = column_stats(mom[:, :c], np.asarray(m2)[:c], np.asarray(hist)[:c], _pp_integral(c), quantiles)
    columns = tuple((f, -1) for f in PP_FIELDS) + tuple(("dc_peak_w", d) for d in range(n_dc))
    return PowerProfileResult(columns=columns, **st.result_fields((c,)), hi=float(hi), threshold=float(threshold),
                              duration_curve=(pp_bin_edges(hi), mom[1, c:c + PP_BINS].copy()), pooled_energy_j=float(energy))


def _pooled_energy(summary: np.ndarray, dev=None) -> float:
    """Total energy of the replicas with status 0, summed over the ranks (the tensor all-reduced lives on ``dev``)."""
    import torch
    from . import spec as S
    s = np.asarray(summary)
    good = s[:, S.S_STATUS] == 0
    return float(_allreduce_sum(torch.tensor([float(s[good, S.S_TOTAL_ENERGY_J].sum())], dtype=torch.float64, device=dev))[0])


def power_profile(engine, quantiles: Sequence[float] = PP_CSV_QUANTILES, summary=None) -> PowerProfileResult:
    """Statistics of the power profile of ``engine`` (a finished BatchedEngine with enable_power_profile()), over all
    ranks when torch.distributed runs with world > 1 (every rank calls this).  ``summary``: the engine's summary rows if
    the caller has them already (they give the pooled energy)."""
    import torch
    if not engine.power_profile_enabled:
        raise RuntimeError("power profile not enabled (enable_power_profile)")
    dev = torch.device("cuda", engine.device)
    n_dc = engine.spec.n_dc
    passes = device_passes(dev, len(PP_FIELDS) + n_dc + PP_BINS, engine.power_profile_moments_into,
                           engine.power_profile_spread_into, stat_cols=len(PP_FIELDS) + n_dc)
    energy = _pooled_energy(engine.summary() if summary is None else summary, dev)
    thr = engine.power_threshold
    return pp_finalize(*passes, n_dc, engine.power_profile_range(), float("inf") if thr is None else thr, energy, quantiles)


def power_profile_from_rows(rows: np.ndarray, summary: np.ndarray, hi: float, threshold=None,
                            quantiles: Sequence[float] = PP_CSV_QUANTILES) -> PowerProfileResult:
    """The same statistics from host rows [PP_FIELDS + n_dc + PP_BINS, R] (BatchedEngine.power_profile_rows) and the
    summary rows [R, SUMMARY_K] through the numpy mirror of both passes; replicas with status != 0 are left out.
    All-reduced over the ranks like power_profile."""
    from . import spec as S
    rows = np.asarray(rows, dtype=np.float64)
    n_dc = rows.shape[0] - len(PP_FIELDS) - PP_BINS
    stat_cols = len(PP_FIELDS) + n_dc
    good = np.asarray(summary)[:, S.S_STATUS] == 0
    passes = host_passes(rows, np.broadcast_to(good[None, :], rows.shape), _pp_integral(stat_cols), stat_cols)
    return pp_finalize(*passes, n_dc, hi, float("inf") if threshold is None else float(threshold), _pooled_energy(summary),
                       quantiles)


# ---- occupancy -------------------------------------------------------------------------------------------------------
# per-replica statistics of each DC's step functions (DCSIM_OCC_* order): the time averages of Qi, Qt and N, the longest
# queues, and the shares of the profile with a queue, with every GPU busy and with none busy
OCC_STATS = ("mean_q_inf", "mean_q_trn", "mean_running", "max_q_inf", "max_q_trn", "queued_share", "saturated_share",
             "idle_share")
OCC_MAX_STATS = (3, 4)                                 # the stored maxima: integer columns, not divided by profile_s
OCC_BINS = 128                                         # DCSIM_OCC_BINS
OCC_TIME_KINDS = ("queue", "busy")


def _occ_integral(n_dc: int) -> np.ndarray:
    return np.isin(np.arange(len(OCC_STATS) * n_dc) // n_dc, OCC_MAX_STATS)


def _occ_columns(rows: np.ndarray, status: np.ndarray):
    """rows [1 + 8 * n_dc + 2 * OCC_BINS * n_dc, R], status [R] -> (x, ok) [8 * n_dc + 2 * OCC_BINS * n_dc, R] as the
    kernels' column source: the stored per-DC fields over profile_s (the maxima as stored), then the bins; replica r
    counts when its status is 0 and profile_s > 0."""
    rows = np.asarray(rows, dtype=np.float64)
    profile = rows[0]
    n_dc = (rows.shape[0] - 1) // (len(OCC_STATS) + 2 * OCC_BINS)
    n_stat = len(OCC_STATS) * n_dc
    x = rows[1:].copy()
    share = ~np.isin(np.arange(n_stat) // n_dc, OCC_MAX_STATS)
    with np.errstate(invalid="ignore", divide="ignore"):
        x[:n_stat][share] = x[:n_stat][share] / profile[None, :]
    ok = (np.asarray(status) == 0) & (profile > 0)
    return x, np.broadcast_to(ok[None, :], x.shape)


@dataclass
class OccupancyResult:
    """Batch statistics of the occupancy recorder over the replicas with status 0 and a non-empty profile.  ``n`` ...
    ``max`` and ``quantiles`` ([Q, columns]) cover ``columns`` = (stat, dc) for every OCC_STATS entry and DC.
    ``queue_bins`` / ``busy_bins`` [n_dc, OCC_BINS]: pooled seconds at each queue length (the last bin: that length or
    more) and each busy-GPU bin of ``bin_widths`` GPUs, summed over the replicas."""
    columns: Tuple[Tuple[str, int], ...]
    n: np.ndarray
    mean: np.ndarray
    std: np.ndarray                                    # unbiased (ddof = 1); 0 for a single sample
    min: np.ndarray
    max: np.ndarray
    q: Tuple[float, ...]
    quantiles: np.ndarray
    queue_bins: np.ndarray
    busy_bins: np.ndarray
    bin_widths: np.ndarray

    def column(self, stat: str, dc: int) -> int:
        return self.columns.index((stat, dc))

    @property
    def replicas(self) -> int:
        return int(self.n[0]) if len(self.n) else 0

    def queue_curve(self, dc: int):
        """(queue lengths [OCC_BINS], pooled seconds at each); the last bin holds OCC_BINS - 1 jobs or more."""
        return np.arange(OCC_BINS, dtype=np.float64), self.queue_bins[dc].copy()

    def busy_curve(self, dc: int):
        """(busy GPUs at each bin's lower edge [OCC_BINS], pooled seconds in each bin); exact values when the DC's bin
        width is 1."""
        return np.arange(OCC_BINS, dtype=np.float64) * float(self.bin_widths[dc]), self.busy_bins[dc].copy()

    def time_quantiles(self, kind: str, dc: int, shares: Sequence[float]) -> np.ndarray:
        """For ``kind`` "queue" or "busy": the value the DC was at or above for each share of the pooled time (0.01: the
        queue length reached or exceeded 1 % of the time), a bin's lower edge; NaN without pooled time."""
        vals, sec = self.queue_curve(dc) if kind == "queue" else self.busy_curve(dc)
        total = sec.sum()
        out = np.full(len(shares), np.nan)
        if total <= 0:
            return out
        above = np.cumsum(sec[::-1])[::-1]             # time at or above each bin
        for i, s in enumerate(shares):
            k = np.nonzero(above >= float(s) * total)[0]
            out[i] = vals[int(k.max()) if len(k) else 0]
        return out

    def pooled(self) -> dict:
        """Per DC (index): the batch means of mean_q_inf, mean_q_trn, saturated_share and idle_share, and the queue
        length exceeded for 10 % and 1 % of the pooled time."""
        out = {}
        for d in range(self.queue_bins.shape[0]):
            row = {s: float(self.mean[self.column(s, d)]) for s in ("mean_q_inf", "mean_q_trn", "saturated_share", "idle_share")}
            p10, p1 = self.time_quantiles("queue", d, (0.1, 0.01))
            row.update(queue_len_top10pct=float(p10), queue_len_top1pct=float(p1))
            out[d] = row
        return out

    def to_csv(self, path: str, dc_names: Sequence[str]):
        """Long format: dc,field,n,mean,std,min,p05,p25,p50,p75,p95,p99,max — one row per DC and statistic, then per DC
        a ``queue_len_time`` and a ``busy_gpus_time`` row for the pooled time distributions: n = replicas, mean = the
        time-weighted mean of the bins' values, std empty, min / max the lowest / highest occupied bin, the quantiles the
        values reached or exceeded for 95 / 75 / 50 / 25 / 5 / 1 % of the pooled time."""
        fmt = lambda x: repr(float(x))  # noqa: E731
        D = self.queue_bins.shape[0]
        with open(path, "w", newline="") as f:
            w = csv.writer(f)
            w.writerow(PP_CSV_HEADER)
            for d in range(D):
                for s in OCC_STATS:
                    c = self.column(s, d)
                    w.writerow([dc_names[d], s, int(self.n[c]), fmt(self.mean[c]), fmt(self.std[c]), fmt(self.min[c])]
                               + [fmt(self.quantiles[j, c]) for j in range(len(self.q))] + [fmt(self.max[c])])
            for d in range(D):
                for kind, field in zip(OCC_TIME_KINDS, ("queue_len_time", "busy_gpus_time")):
                    vals, sec = self.queue_curve(d) if kind == "queue" else self.busy_curve(d)
                    total = sec.sum()
                    occ = np.nonzero(sec > 0)[0]
                    mean = float((vals * sec).sum() / total) if total > 0 else float("nan")
                    lo = vals[occ.min()] if len(occ) else float("nan")
                    hi = vals[occ.max()] if len(occ) else float("nan")
                    tq = self.time_quantiles(kind, d, [1.0 - q for q in PP_CSV_QUANTILES])
                    w.writerow([dc_names[d], field, self.replicas, fmt(mean), "", fmt(lo)] + [fmt(v) for v in tq] + [fmt(hi)])


def occ_finalize(mom, m2, hist, n_dc: int, widths, quantiles: Sequence[float] = PP_CSV_QUANTILES) -> OccupancyResult:
    """All-reduced moments [4, 8 * n_dc + 2 * OCC_BINS * n_dc], m2 and histograms over the first 8 * n_dc columns, and
    the busy-bin widths -> statistics."""
    mom = np.asarray(mom, dtype=np.float64)
    c = len(OCC_STATS) * n_dc
    st = column_stats(mom[:, :c], np.asarray(m2)[:c], np.asarray(hist)[:c], _occ_integral(n_dc), quantiles)
    columns = tuple((s, d) for s in OCC_STATS for d in range(n_dc))
    bins = mom[1, c:c + 2 * OCC_BINS * n_dc].reshape(2, n_dc, OCC_BINS)
    return OccupancyResult(columns=columns, **st.result_fields((c,)), queue_bins=bins[0].copy(), busy_bins=bins[1].copy(),
                           bin_widths=np.asarray(widths, dtype=np.int64))


def occupancy(engine, quantiles: Sequence[float] = PP_CSV_QUANTILES) -> OccupancyResult:
    """Statistics of the occupancy recorder of ``engine`` (a finished BatchedEngine with enable_occupancy()), over all
    ranks when torch.distributed runs with world > 1 (every rank calls this)."""
    import torch
    if not engine.occupancy_enabled:
        raise RuntimeError("occupancy not enabled (enable_occupancy)")
    dev = torch.device("cuda", engine.device)
    n_dc = engine.spec.n_dc
    stat = len(OCC_STATS) * n_dc
    passes = device_passes(dev, stat + 2 * OCC_BINS * n_dc, engine.occupancy_moments_into, engine.occupancy_spread_into,
                           stat_cols=stat)
    return occ_finalize(*passes, n_dc, engine.occupancy_bin_widths(), quantiles)


def occupancy_from_rows(rows: np.ndarray, summary: np.ndarray, widths, quantiles: Sequence[float] = PP_CSV_QUANTILES
                        ) -> OccupancyResult:
    """The same statistics from host rows [1 + 8 * n_dc + 2 * OCC_BINS * n_dc, R] (BatchedEngine.occupancy_rows), the
    summary rows [R, SUMMARY_K] and the busy-bin widths [n_dc] (BatchedEngine.occupancy_bin_widths) through the numpy
    mirror of both passes.  All-reduced over the ranks like occupancy."""
    from . import spec as S
    x, ok = _occ_columns(rows, np.asarray(summary)[:, S.S_STATUS])
    n_dc = len(widths)
    passes = host_passes(x, ok, _occ_integral(n_dc), len(OCC_STATS) * n_dc)
    return occ_finalize(*passes, n_dc, widths, quantiles)


# ---- per-run tail latency --------------------------------------------------------------------------------------------
# per replica and group (job type, scope) the columns TAIL_FIELDS, then per (kind, job type) SLA_MET (DCSIM_TAIL_*)
TAIL_KINDS = ("latency", "wait", "response")
TAIL_STATS = ("p50", "p95", "p99", "p999", "max")
TAIL_QUANTILES = (0.5, 0.95, 0.99, 0.999)              # the order statistics p50 .. p999
TAIL_FIELDS = ("jobs", "unfinished") + tuple(f"{k}_{s}_s" for k in TAIL_KINDS for s in TAIL_STATS)
TAIL_TYPES = ("inference", "training")                 # DCSIM_JT_* order
TAIL_CSV_HEADER = ["type"] + PP_CSV_HEADER
# one created job of a replica, as the tail-latency mirror takes it (finish NaN: not finished by end_time)
TAIL_JOB_DTYPE = np.dtype([("jtype", "<i4"), ("dc", "<i4"), ("arrival", "<f8"), ("xfer_done", "<f8"), ("start", "<f8"),
                           ("finish", "<f8")])


def _tail_columns(n_dc: int):
    """(type, dc, field) of every column in the kernels' order; dc = -1: all DCs."""
    cols = [(TAIL_TYPES[jt], dc, f) for jt in range(2) for dc in range(-1, n_dc) for f in TAIL_FIELDS]
    return tuple(cols + [(TAIL_TYPES[jt], -1, f"{k}_sla_met") for k in TAIL_KINDS for jt in range(2)])


def _tail_integral(n_dc: int) -> np.ndarray:
    cols = _tail_columns(n_dc)
    return np.array([f in ("jobs", "unfinished") or f.endswith("_sla_met") for _, _, f in cols])


def order_statistic(values: np.ndarray, q: float) -> float:
    """The q-quantile as the per-run tail columns define it: numpy's ``inverted_cdf``, the k-th smallest value with
    k = max(ceil(n * q), 1)."""
    return float(np.quantile(np.asarray(values, dtype=np.float64), q, method="inverted_cdf"))


def tail_rows_from_jobs(jobs: Sequence[np.ndarray], status, n_dc: int, sla_s=None) -> np.ndarray:
    """numpy mirror of the selection pass: per replica its created jobs (TAIL_JOB_DTYPE) and its status word ->
    [tail columns, R] float64 (BatchedEngine.tail_latency_rows).  Values are the f64 subtractions of the device; NaN
    where a column does not count."""
    from . import spec as S
    R = len(jobs)
    sla = math.inf if sla_s is None else float(sla_s)
    out = np.full((S.tail_cols(n_dc), R), np.nan)
    for r in range(R):
        if int(status[r]) != 0:
            continue
        j = np.asarray(jobs[r])
        fin = ~np.isnan(j["finish"])
        vals = (j["finish"] - j["start"], j["start"] - j["xfer_done"], j["finish"] - j["arrival"])
        for jt in range(2):
            for dc in range(-1, n_dc):
                sel = (j["jtype"] == jt) & ((j["dc"] == dc) if dc >= 0 else True)
                c0 = S.tail_col(n_dc, jt, 0, dc)
                out[c0 + S.TAIL_JOBS, r] = np.count_nonzero(sel & fin)
                out[c0 + S.TAIL_UNFINISHED, r] = np.count_nonzero(sel & ~fin)
                if not np.any(sel & fin):
                    continue
                for k, v in enumerate(vals):
                    x = v[sel & fin]
                    base = c0 + S.TAIL_STATS_BASE + k * len(TAIL_STATS)
                    for i, q in enumerate(TAIL_QUANTILES):
                        out[base + i, r] = order_statistic(x, q)
                    out[base + len(TAIL_QUANTILES), r] = x.max()
        if math.isfinite(sla):
            for k in range(len(TAIL_KINDS)):
                for jt in range(2):
                    if out[S.tail_col(n_dc, jt, S.TAIL_JOBS), r] > 0:
                        p99 = out[S.tail_col(n_dc, jt, S.TAIL_STATS_BASE + k * len(TAIL_STATS) + 2), r]
                        out[S.tail_sla_col(n_dc, k, jt), r] = 1.0 if p99 <= sla else 0.0
    return out


def wilson_interval(successes: float, n: float, z: float = 1.959963984540054):
    """The Wilson score interval of a binomial share (95 % by default); (NaN, NaN) without trials."""
    if n <= 0:
        return float("nan"), float("nan")
    p = successes / n
    d = 1.0 + z * z / n
    c = (p + z * z / (2.0 * n)) / d
    h = z * math.sqrt(p * (1.0 - p) / n + z * z / (4.0 * n * n)) / d
    return max(0.0, c - h), min(1.0, c + h)


@dataclass
class TailLatencyResult:
    """Batch statistics of every replica's own tail-latency columns over the replicas with status 0 (a column counts the
    replicas where it is defined: a group with a finished job; SLA_MET with an SLA).  ``n`` ... ``max`` and
    ``quantiles`` ([Q, columns]) cover ``columns`` = (type, dc, field), dc = -1 for all DCs."""
    columns: Tuple[Tuple[str, int, str], ...]
    n: np.ndarray
    mean: np.ndarray
    std: np.ndarray                                    # unbiased (ddof = 1); 0 for a single sample
    min: np.ndarray
    max: np.ndarray
    q: Tuple[float, ...]
    quantiles: np.ndarray
    sla_s: float                                       # +inf: none

    @staticmethod
    def _type(jtype) -> str:
        return TAIL_TYPES[jtype] if isinstance(jtype, (int, np.integer)) else str(jtype)

    def column(self, kind, jtype, field: str, dc: int = -1) -> int:
        """Column of ``field`` ("jobs", "unfinished", "p50" ... "max", "sla_met") of ``kind`` (TAIL_KINDS; None for jobs
        and unfinished) for job type ``jtype`` (0 / 1 or TAIL_TYPES) in DC ``dc`` (-1: all DCs)."""
        if kind is None:
            name = field
        elif field == "sla_met":
            name = f"{kind}_sla_met"
        else:
            name = f"{kind}_{field}_s"
        return self.columns.index((self._type(jtype), dc, name))

    def sla_attainment(self, kind, jtype) -> dict:
        """The share of runs (status 0, with a finished job of the type) whose p99 of ``kind`` met the SLA, with its 95 %
        Wilson interval; NaN without an SLA or such runs."""
        c = self.column(kind, jtype, "sla_met")
        runs = int(self.n[c])
        met = float(self.mean[c]) * runs if runs else 0.0
        lo, hi = wilson_interval(round(met), runs) if math.isfinite(self.sla_s) else (float("nan"), float("nan"))
        share = met / runs if runs and math.isfinite(self.sla_s) else float("nan")
        return {"share": share, "ci95_lo": lo, "ci95_hi": hi, "runs": runs, "met": int(round(met))}

    def pooled(self) -> dict:
        """{job type: {kind: ...}}: the SLA attainment (share, 95 % interval, runs) and the mean / p05 / p50 / p95 over
        the runs of the per-run p99 (the quantiles read off the batch histogram, within one bin width)."""
        out = {jt: {} for jt in TAIL_TYPES}
        qi = {q: self.q.index(q) for q in (0.05, 0.5, 0.95) if q in self.q}
        for jt in TAIL_TYPES:
            for kind in TAIL_KINDS:
                c = self.column(kind, jt, "p99")
                row = {"sla_s": self.sla_s if math.isfinite(self.sla_s) else None,
                       "sla_attainment": self.sla_attainment(kind, jt), "runs": int(self.n[c]),
                       "p99_mean_s": float(self.mean[c])}
                for q, i in qi.items():
                    row[f"p99_p{int(round(q * 100)):02d}_s"] = float(self.quantiles[i, c])
                out[jt][kind] = row
        return out

    def to_csv(self, path: str, dc_names: Sequence[str]):
        """Long format: type,dc,field,n,mean,std,min,p05,p25,p50,p75,p95,p99,max — one row per (type, scope, field),
        dc empty for all DCs, then the *_sla_met rows (left empty without an SLA)."""
        fmt = lambda x: repr(float(x))  # noqa: E731
        with open(path, "w", newline="") as f:
            w = csv.writer(f)
            w.writerow(TAIL_CSV_HEADER)
            for c, (jt, d, field) in enumerate(self.columns):
                dc = dc_names[d] if d >= 0 else ""
                if field.endswith("_sla_met") and not math.isfinite(self.sla_s):
                    w.writerow([jt, dc, field] + [""] * (len(TAIL_CSV_HEADER) - 3))
                    continue
                w.writerow([jt, dc, field, int(self.n[c]), fmt(self.mean[c]), fmt(self.std[c]), fmt(self.min[c])]
                           + [fmt(self.quantiles[j, c]) for j in range(len(self.q))] + [fmt(self.max[c])])


def tail_finalize(mom, m2, hist, n_dc: int, sla_s: float, quantiles: Sequence[float] = PP_CSV_QUANTILES
                  ) -> TailLatencyResult:
    """All-reduced moments, m2 and histograms over the tail columns -> statistics."""
    cols = _tail_columns(n_dc)
    st = column_stats(np.asarray(mom, dtype=np.float64), np.asarray(m2), np.asarray(hist), _tail_integral(n_dc), quantiles)
    return TailLatencyResult(columns=cols, **st.result_fields((len(cols),)), sla_s=float(sla_s))


def tail_latency(engine, quantiles: Sequence[float] = PP_CSV_QUANTILES) -> TailLatencyResult:
    """Statistics of the per-run tail-latency columns of ``engine`` (a finished BatchedEngine with
    enable_tail_latency()), over all ranks when torch.distributed runs with world > 1 (every rank calls this)."""
    import torch
    from . import spec as S
    if not engine.tail_latency_enabled:
        raise RuntimeError("tail latency not enabled (enable_tail_latency)")
    dev = torch.device("cuda", engine.device)
    n_dc = engine.spec.n_dc
    passes = device_passes(dev, S.tail_cols(n_dc), engine.tail_latency_moments_into, engine.tail_latency_spread_into)
    sla = engine.tail_latency_sla
    return tail_finalize(*passes, n_dc, math.inf if sla is None else sla, quantiles)


def tail_latency_from_rows(rows: np.ndarray, status, sla_s=None, quantiles: Sequence[float] = PP_CSV_QUANTILES
                           ) -> TailLatencyResult:
    """The same statistics from host columns [tail columns, R] (BatchedEngine.tail_latency_rows) and the replicas'
    status words through the numpy mirror of both passes.  All-reduced over the ranks like tail_latency."""
    from . import spec as S
    rows = np.asarray(rows, dtype=np.float64)
    n_dc = (rows.shape[0] - 2 * len(TAIL_KINDS)) // (2 * S.TAIL_GROUP_FIELDS) - 1
    ok = (np.asarray(status)[None, :] == 0) & ~np.isnan(rows)
    passes = host_passes(rows, ok, _tail_integral(n_dc))
    return tail_finalize(*passes, n_dc, math.inf if sla_s is None else float(sla_s), quantiles)


def tail_latency_from_jobs(jobs: Sequence[np.ndarray], status, n_dc: int, sla_s=None,
                           quantiles: Sequence[float] = PP_CSV_QUANTILES) -> TailLatencyResult:
    """The numpy mirror end to end: per replica its created jobs (TAIL_JOB_DTYPE) and status word -> the per-run
    columns with np.quantile(..., method="inverted_cdf") -> batch statistics through host_passes."""
    return tail_latency_from_rows(tail_rows_from_jobs(jobs, status, n_dc, sla_s), status, sla_s, quantiles)


# ---- energy cost and carbon ------------------------------------------------------------------------------------------
COST_FIELDS = ("energy_j", "cost_usd", "carbon_g")    # per DC and for the cluster (DCSIM_COST_*)
COST_CSV_HEADER = ["dc", "field", "carbon_g_per_kwh"] + PP_CSV_HEADER[2:]
J_PER_KWH = 3.6e6


def _cost_columns(n_dc: int):
    """(field, dc, hour) of every stored column in the recorder's order; dc = -1: the cluster, hour = -1: none."""
    cols = [("hour_j", d, h) for d in range(n_dc) for h in range(24)]
    cols += [(f, d, -1) for f in COST_FIELDS for d in range(n_dc)]
    return tuple(cols + [(f, -1, -1) for f in COST_FIELDS])


@dataclass
class EnergyCostResult:
    """Batch statistics of the energy-cost recorder over the replicas with status 0.  ``n`` ... ``max`` and ``quantiles``
    ([Q, columns]) cover ``columns`` = (field, dc, hour): the 24 hourly energies of each DC, energy, cost and carbon per
    DC, then the cluster totals (dc = -1).  ``sum`` [columns]: the pooled sums over those replicas.  ``price_kwh``
    [n_dc, 24] and ``carbon_intensity`` [n_dc] are the tables the columns were priced with."""
    columns: Tuple[Tuple[str, int, int], ...]
    n: np.ndarray
    mean: np.ndarray
    std: np.ndarray                                    # unbiased (ddof = 1); 0 for a single sample
    min: np.ndarray
    max: np.ndarray
    q: Tuple[float, ...]
    quantiles: np.ndarray
    sum: np.ndarray
    price_kwh: np.ndarray
    carbon_intensity: np.ndarray

    def column(self, field: str, dc: int = -1, hour: int = -1) -> int:
        """Column of ``field`` (COST_FIELDS, or "hour_j" with an ``hour``) of DC ``dc`` (-1: the cluster)."""
        return self.columns.index((field, dc, hour))

    @property
    def replicas(self) -> int:
        return int(self.n[-1]) if len(self.n) else 0

    def hourly(self, dc: int) -> dict:
        """DC ``dc``'s 24 hourly energy bands over the replicas: {"mean", "std", "min", "max": [24], "quantiles":
        [Q, 24]} [J], hour of day 0 .. 23."""
        c = [self.column("hour_j", dc, h) for h in range(24)]
        return {"mean": self.mean[c], "std": self.std[c], "min": self.min[c], "max": self.max[c],
                "quantiles": self.quantiles[:, c]}

    def pooled(self) -> dict:
        """The pooled energy [kWh], cost [USD] and carbon [g] of every replica that counts, and the effective USD/kWh
        (pooled cost over pooled kWh) and g/kWh, per DC (index) and for the cluster (key "cluster")."""
        def one(dc):
            kwh = float(self.sum[self.column("energy_j", dc)]) / J_PER_KWH
            usd = float(self.sum[self.column("cost_usd", dc)])
            g = float(self.sum[self.column("carbon_g", dc)])
            return {"energy_kwh": kwh, "cost_usd": usd, "carbon_g": g,
                    "usd_per_kwh": usd / kwh if kwh > 0 else float("nan"), "g_per_kwh": g / kwh if kwh > 0 else float("nan")}
        out = {d: one(d) for d in range(len(self.carbon_intensity))}
        out["cluster"] = one(-1)
        out["replicas"] = self.replicas
        return out

    def to_csv(self, path: str, dc_names: Sequence[str]):
        """Long format: dc,field,carbon_g_per_kwh,n,mean,std,min,p05,p25,p50,p75,p95,p99,max — per DC energy_j, cost_usd,
        carbon_g and hour_j_00 .. hour_j_23 with the DC's carbon intensity (0 for a DC the carbon map leaves out), then
        the cluster's energy_j, cost_usd and carbon_g (dc and carbon_g_per_kwh empty)."""
        fmt = lambda x: repr(float(x))  # noqa: E731
        D = len(self.carbon_intensity)
        rows = [r for d in range(D) for r in [(d, (f, d, -1), f) for f in COST_FIELDS]
                + [(d, ("hour_j", d, h), f"hour_j_{h:02d}") for h in range(24)]]
        rows += [(-1, (f, -1, -1), f) for f in COST_FIELDS]
        with open(path, "w", newline="") as fh:
            w = csv.writer(fh)
            w.writerow(COST_CSV_HEADER)
            for d, key, name in rows:
                c = self.columns.index(key)
                head = [dc_names[d], name, fmt(self.carbon_intensity[d])] if d >= 0 else ["", name, ""]
                w.writerow(head + [int(self.n[c]), fmt(self.mean[c]), fmt(self.std[c]), fmt(self.min[c])]
                           + [fmt(self.quantiles[j, c]) for j in range(len(self.q))] + [fmt(self.max[c])])


def cost_finalize(mom, m2, hist, n_dc: int, price_kwh, carbon_intensity, quantiles: Sequence[float] = PP_CSV_QUANTILES
                  ) -> EnergyCostResult:
    """All-reduced moments, m2 and histograms over the energy-cost columns -> statistics."""
    cols = _cost_columns(n_dc)
    mom = np.asarray(mom, dtype=np.float64)
    st = column_stats(mom, np.asarray(m2), np.asarray(hist), np.zeros(len(cols), dtype=bool), quantiles)
    return EnergyCostResult(columns=cols, **st.result_fields((len(cols),)), sum=mom[1].copy(),
                            price_kwh=np.asarray(price_kwh, dtype=np.float64).reshape(n_dc, 24),
                            carbon_intensity=np.asarray(carbon_intensity, dtype=np.float64).reshape(n_dc))


def _cost_tables(sp):
    return ([[sp.dc[d].price_kwh[h] for h in range(24)] for d in range(sp.n_dc)],
            [sp.dc[d].carbon_intensity for d in range(sp.n_dc)])


def energy_cost(engine, quantiles: Sequence[float] = PP_CSV_QUANTILES) -> EnergyCostResult:
    """Statistics of the energy-cost recorder of ``engine`` (a finished BatchedEngine with enable_energy_cost()), over
    all ranks when torch.distributed runs with world > 1 (every rank calls this)."""
    import torch
    from . import spec as S
    if not engine.energy_cost_enabled:
        raise RuntimeError("energy cost not enabled (enable_energy_cost)")
    dev = torch.device("cuda", engine.device)
    n_dc = engine.spec.n_dc
    passes = device_passes(dev, S.cost_cols(n_dc), engine.energy_cost_moments_into, engine.energy_cost_spread_into)
    return cost_finalize(*passes, n_dc, *_cost_tables(engine.spec), quantiles)


def energy_cost_from_rows(rows: np.ndarray, status, price_kwh, carbon_intensity,
                          quantiles: Sequence[float] = PP_CSV_QUANTILES) -> EnergyCostResult:
    """The same statistics from host columns [cost columns, R] (BatchedEngine.energy_cost_rows), the replicas' status
    words and the tables ([n_dc, 24] USD/kWh, [n_dc] gCO2/kWh) through the numpy mirror of both passes.  All-reduced
    over the ranks like energy_cost."""
    rows = np.asarray(rows, dtype=np.float64)
    n_dc = (rows.shape[0] - 3) // 27
    ok = np.broadcast_to((np.asarray(status) == 0)[None, :], rows.shape)
    passes = host_passes(rows, ok, np.zeros(rows.shape[0], dtype=bool))
    return cost_finalize(*passes, n_dc, price_kwh, carbon_intensity, quantiles)
