"""Batch-wide cluster-log statistics: per log tick, the mean, spread and quantiles of every DC's cluster_log.csv
columns over all replicas of the batch (all GPUs of a sharded run).

The device records, for every replica, the values its cluster_log.csv rows would hold at every log tick
(``BatchedEngine.enable_cluster_ensemble``).  Two reductions turn them into statistics per column (tick, field, DC):

  moments  n, sum, min, max              -> all-reduce (SUM for n / sum, MIN, MAX)
  spread   sum (x - mean)^2, histogram   -> all-reduce (SUM), given the GLOBAL mean, min and max

Only n, min, max and the histograms cross GPUs exactly: they, and the quantiles read off the histograms, do not depend
on the number of GPUs.  Mean and std do only up to summation order.  ``moments_rows`` / ``spread_rows`` are the numpy
mirror of the two kernels (csrc dcsim_ens_moments_kernel / dcsim_ens_spread_kernel), as ``sharding.aggregate_rows``
mirrors dcsim_reduce_kernel.
"""
import csv
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
    x = rows.reshape(-1, R)
    m = ok.reshape(-1, R)
    out = np.empty((4, x.shape[0]))
    out[0] = m.sum(axis=1)
    out[1] = np.where(m, x, 0.0).sum(axis=1)
    out[2] = np.where(m, x, np.inf).min(axis=1)
    out[3] = np.where(m, x, -np.inf).max(axis=1)
    return out


def bin_widths(lo: np.ndarray, hi: np.ndarray, n_dc: int) -> np.ndarray:
    """Per column: the histogram's bin width (0: every value in bin 0) — the kernel's rule, the kernel's float ops."""
    lo, hi = np.asarray(lo, dtype=np.float64), np.asarray(hi, dtype=np.float64)
    field = (np.arange(lo.size) // n_dc) % len(FIELDS)
    integral = np.isin(field, INTEGER_FIELDS)
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
    mean = np.asarray(mean, dtype=np.float64)
    with np.errstate(invalid="ignore"):
        m2 = np.where(ok, (x - mean[:, None]) ** 2, 0.0).sum(axis=1)
    width = bin_widths(lo, hi, D)
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
    return finalize(mom.cpu().numpy(), m2.cpu().numpy(), hist.cpu().numpy(), n_dc, log_interval, quantiles)


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
