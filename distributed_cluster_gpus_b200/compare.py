"""Policy comparisons on common random numbers: several variants of one scenario run on the same replica keys, and
statistics of the per-replica difference ``variant - baseline`` are reduced on the device.

Arrivals do not depend on the policy: variants whose specs draw the same arrivals (``engine.arrivals_compatible``, the
library's one rule) share ONE arrival pre-pass (``BatchedEngine.shared``), so replica r of each sees the same jobs at the
same instants.  Variants that change the arrivals (``eco_route`` routes without a random draw, other rates ...) run
their own pre-pass; they are still paired with the baseline by replica key.

Per variant and metric the two reduction passes of ``ensemble.two_passes`` run over columns (metric, field), fields
``PAIR_FIELDS``: base, variant, diff = variant - base, lower = (variant < base), higher = (variant > base).  A replica
counts when both runs ended with status 0 and the metric is defined in both.  ``paired_from_summaries`` is the numpy
mirror of the two kernels (csrc dcsim_ens_pair_src).
"""
import csv
import functools
from dataclasses import dataclass
from typing import Callable, Dict, Sequence, Tuple

import numpy as np

from . import ensemble as EN
from . import spec as S

METRICS = ("energy_j", "energy_per_job_j", "jobs_inf", "jobs_trn", "mean_latency_inf_s", "mean_latency_trn_s",
           "unfinished")                                # DCSIM_PAIR_* order, then dc_energy_j per DC
DC_METRIC = "dc_energy_j"
INTEGER_METRICS = (2, 3, 6)                             # jobs_inf, jobs_trn, unfinished: unit bins, exact quantiles
PAIR_FIELDS = ("base", "variant", "diff", "lower", "higher")
BASE, VARIANT, DIFF, LOWER, HIGHER = range(5)
CSV_HEADER = ["variant", "baseline", "metric", "dc", "n", "base_mean", "variant_mean", "diff_mean", "diff_std",
              "diff_ci95_lo", "diff_ci95_hi", "rel_change", "rel_ci95_lo", "rel_ci95_hi", "frac_lower", "frac_higher"]


def metric_names(n_dc: int) -> Tuple[str, ...]:
    return METRICS + (DC_METRIC,) * n_dc


def n_columns(n_dc: int) -> int:
    return (len(METRICS) + n_dc) * len(PAIR_FIELDS)


def _integral(n_dc: int) -> np.ndarray:
    col = np.arange(n_columns(n_dc))
    return (col % len(PAIR_FIELDS) >= LOWER) | np.isin(col // len(PAIR_FIELDS), INTEGER_METRICS)


# ---- numpy mirror of the column source ------------------------------------------------------------------------------
def _metric_values(s: np.ndarray, n_dc: int):
    """summary rows [R, SUMMARY_K] -> (values [M, R], defined [M, R]) with the kernel's float operations."""
    R = s.shape[0]
    fin, fin_i, fin_t = s[:, S.S_JOBS_FINISHED], s[:, S.S_FIN_INF], s[:, S.S_FIN_TRN]
    ones = np.ones(R, dtype=bool)
    with np.errstate(invalid="ignore", divide="ignore"):
        vals = [s[:, S.S_TOTAL_ENERGY_J], s[:, S.S_TOTAL_ENERGY_J] / fin, fin_i, fin_t, s[:, S.S_LAT_SUM_INF] / fin_i,
                s[:, S.S_LAT_SUM_TRN] / fin_t]
    ok = [ones, fin > 0, ones, ones, fin_i > 0, fin_t > 0]
    u = np.zeros(R)
    for d in range(n_dc):
        g = S.S_DC0 + d * S.S_DC_STRIDE
        u = u + (s[:, g + S.SD_Q_INF] + s[:, g + S.SD_Q_TRN] + s[:, g + S.SD_RUNNING])
    vals.append(u)
    ok.append(ones)
    for d in range(n_dc):
        vals.append(s[:, S.S_DC0 + d * S.S_DC_STRIDE + S.SD_ENERGY_J])
        ok.append(ones)
    return np.stack(vals), np.stack(ok)


def pair_columns(base: np.ndarray, variant: np.ndarray, n_dc: int):
    """-> (x, ok) [columns, R], columns (metric, PAIR_FIELDS) metric-major as the kernels'."""
    vb, okb = _metric_values(base, n_dc)
    vv, okv = _metric_values(variant, n_dc)
    both = (base[:, S.S_STATUS] == 0)[None, :] & (variant[:, S.S_STATUS] == 0)[None, :] & okb & okv
    with np.errstate(invalid="ignore"):               # undefined values (NaN) are masked out by ok
        x = np.stack([vb, vv, vv - vb, (vv < vb).astype(np.float64), (vv > vb).astype(np.float64)], axis=1)
    ok = np.broadcast_to(both[:, None, :], x.shape)
    R = base.shape[0]
    return np.ascontiguousarray(x.reshape(-1, R)), np.ascontiguousarray(ok.reshape(-1, R))


# ---- statistics ---------------------------------------------------------------------------------------------------
@dataclass
class PairedStats:
    """One variant against the baseline; arrays are [metrics] (``metric_names(n_dc)``), quantiles [Q, metrics]."""
    metrics: Tuple[str, ...]
    n: np.ndarray                  # replicas that count (both ran cleanly, the metric defined in both)
    base_mean: np.ndarray
    variant_mean: np.ndarray
    diff_mean: np.ndarray
    diff_std: np.ndarray           # unbiased (ddof = 1) std of variant - base; 0 for a single sample
    diff_ci95_lo: np.ndarray       # diff_mean -+ 1.96 diff_std / sqrt(n)
    diff_ci95_hi: np.ndarray
    rel_change: np.ndarray         # variant_mean / base_mean - 1
    rel_ci95_lo: np.ndarray        # delta method with cov(base, variant) = (var_b + var_v - var_d) / 2
    rel_ci95_hi: np.ndarray
    frac_lower: np.ndarray         # share of the replicas where variant < base
    frac_higher: np.ndarray
    var_ratio: np.ndarray          # var_d / (var_b + var_v): < 1 when pairing narrowed the CI of the difference
    q: Tuple[float, ...]
    diff_quantiles: np.ndarray     # [Q, metrics] (numpy inverted_cdf, read off the histogram)
    moments: np.ndarray            # the all-reduced passes: [4, columns] {n, sum, min, max}
    m2: np.ndarray                 # [columns]
    hist: np.ndarray               # [columns, ensemble.BINS]


def paired_finalize(mom, m2, hist, n_dc: int, quantiles: Sequence[float] = EN.DEFAULT_QUANTILES) -> PairedStats:
    """All-reduced moments [4, columns], m2 [columns] and histograms [columns, BINS] -> PairedStats."""
    F = len(PAIR_FIELDS)
    mom = np.asarray(mom, dtype=np.float64)
    m2 = np.asarray(m2, dtype=np.float64)
    st = EN.column_stats(mom, m2, hist, _integral(n_dc), quantiles)
    M = st.n.size // F
    mean, var = st.mean.reshape(M, F), st.var.reshape(M, F)
    n = st.n.reshape(M, F)[:, DIFF]
    mb, mv, md = mean[:, BASE], mean[:, VARIANT], mean[:, DIFF]
    vb, vv, vd = var[:, BASE], var[:, VARIANT], var[:, DIFF]
    sd = st.std.reshape(M, F)[:, DIFF]
    with np.errstate(invalid="ignore", divide="ignore"):
        half = np.where(n > 1, 1.96 * sd / np.sqrt(np.maximum(n, 1)), 0.0)
        rel = mv / mb - 1.0
        cov = (vb + vv - vd) / 2.0
        var_rel = (vv / mb ** 2 - 2.0 * mv * cov / mb ** 3 + mv ** 2 * vb / mb ** 4) / np.maximum(n, 1)
        rel_half = np.where(n > 1, 1.96 * np.sqrt(np.maximum(var_rel, 0.0)), 0.0)
        var_ratio = vd / (vb + vv)
    qv = st.quantiles.reshape(len(quantiles), M, F)
    return PairedStats(metrics=metric_names(n_dc), n=n, base_mean=mb, variant_mean=mv, diff_mean=md,
                       diff_std=sd, diff_ci95_lo=md - half, diff_ci95_hi=md + half, rel_change=rel,
                       rel_ci95_lo=rel - rel_half, rel_ci95_hi=rel + rel_half, frac_lower=mean[:, LOWER],
                       frac_higher=mean[:, HIGHER], var_ratio=var_ratio, q=st.q,
                       diff_quantiles=qv[:, :, DIFF], moments=mom, m2=m2, hist=np.asarray(hist))


def paired_from_summaries(base: np.ndarray, variant: np.ndarray, quantiles: Sequence[float] = EN.DEFAULT_QUANTILES,
                          n_dc: int = None) -> PairedStats:
    """The same statistics from host summary rows [R, SUMMARY_K] of the two runs (the same replica keys, row r = replica
    r) through the numpy mirror of both passes, all-reduced over the ranks like ``compare_variants``.  ``n_dc``: the
    scenario's DC count (None: the DC groups that are not all zero in either run)."""
    base, variant = np.asarray(base, dtype=np.float64), np.asarray(variant, dtype=np.float64)
    if n_dc is None:
        groups = np.abs(np.concatenate([base, variant]))[:, S.S_DC0:].reshape(-1, S.MAX_DC, S.S_DC_STRIDE)
        used = np.nonzero(groups.sum(axis=(0, 2)) > 0)[0]
        n_dc = int(used.max()) + 1 if used.size else 1
    x, ok = pair_columns(base, variant, n_dc)
    return paired_finalize(*EN.host_passes(x, ok, _integral(n_dc)), n_dc, quantiles)


@dataclass
class PairedComparison:
    """Every variant against the baseline on the same replica keys."""
    baseline: str
    variants: Tuple[str, ...]            # the compared variants (the baseline excluded), in the caller's order
    n_dc: int
    stats: Dict[str, PairedStats]
    shared_arrivals: Dict[str, bool]     # True: the variant ran on the baseline's own arrival lists (one pre-pass)
    summaries: Dict[str, np.ndarray]     # every variant's (and the baseline's) [replicas, SUMMARY_K] rows of this rank

    def quantile_names(self):
        q = next(iter(self.stats.values())).q if self.stats else EN.DEFAULT_QUANTILES
        return [f"diff_p{int(round(x * 100)):02d}" for x in q]

    def rows(self, dc_names: Sequence[str]):
        """One dict per (variant, metric[, dc]) with the CSV's columns."""
        out = []
        for v in self.variants:
            st = self.stats[v]
            for i, m in enumerate(st.metrics):
                dc = dc_names[i - len(METRICS)] if i >= len(METRICS) else ""
                row = {"variant": v, "baseline": self.baseline, "metric": m, "dc": dc, "n": int(st.n[i])}
                for k in CSV_HEADER[5:]:
                    row[k] = float(getattr(st, k)[i])
                for j, name in enumerate(self.quantile_names()):
                    row[name] = float(st.diff_quantiles[j, i])
                row["var_ratio"] = float(st.var_ratio[i])
                row["shared_arrivals"] = bool(self.shared_arrivals[v])
                out.append(row)
        return out

    def to_csv(self, path: str, dc_names: Sequence[str]):
        """Long format, one row per variant, metric (and DC for dc_energy_j): ``CSV_HEADER``, diff_p05 ... diff_p95,
        var_ratio, shared_arrivals.  Floats unrounded (repr)."""
        header = CSV_HEADER + self.quantile_names() + ["var_ratio", "shared_arrivals"]
        with open(path, "w", newline="") as f:
            w = csv.writer(f)
            w.writerow(header)
            for row in self.rows(dc_names):
                w.writerow([repr(row[k]) if isinstance(row[k], float) else row[k] for k in header])


# ---- running the variants -------------------------------------------------------------------------------------------
class _DeviceArray:
    """A raw device pointer seen through __cuda_array_interface__ (for a device-to-device copy into a torch tensor)."""

    def __init__(self, ptr, shape):
        self.__cuda_array_interface__ = {"shape": tuple(shape), "typestr": "<f8", "data": (int(ptr), False), "version": 2}


def _status_bits(summ) -> int:
    return int(np.bitwise_or.reduce(summ[:, S.S_STATUS].astype(np.int64))) if len(summ) else 0


def _keep(eng, dev):
    """The engine's summaries: (a device copy as a torch tensor, host rows).  Synchronises."""
    import torch
    host = eng.summary()
    t = torch.as_tensor(_DeviceArray(eng.summary_device_ptr(), (eng.n_replicas, S.SUMMARY_K)), device=dev).clone()
    torch.cuda.synchronize(dev)
    return t, host


def _run_group(names, factories, n_replicas, seed, first_replica_id, device, rng, max_retries, dev):
    """Runs the group's owner (names[0]) to completion, then every member on the owner's arrival lists, one at a time.
    The arrival-list and transfer-ring overflows are raised in the shared list headers: they rebuild the owner, and the
    members take the owner's cap_arrivals and cap_xfer.  -> (owner engine, {name: (device tensor, host rows)})."""
    from .engine import BatchedEngine, describe_status, raise_caps
    caps = {}
    for attempt in range(max_retries + 1):
        sp = factories[names[0]](dict(caps))
        owner = BatchedEngine(sp, n_replicas, seed, first_replica_id, device)
        try:
            owner.set_rng(rng)
            owner.advance(0, sync=False)
            bits = _status_bits(owner.summary())
            if bits:
                raise_caps(bits, sp, caps, last_attempt=attempt == max_retries)
                owner.close()
                continue
            kept = {names[0]: _keep(owner, dev)}
        except BaseException:
            owner.close()
            raise
        break
    try:
        for name in names[1:]:
            mcaps = {"cap_arrivals": sp.cap_arrivals, "cap_xfer": sp.cap_xfer}
            for attempt in range(max_retries + 1):
                msp = factories[name](dict(mcaps))
                with BatchedEngine.shared(msp, owner) as m:
                    m.advance(0, sync=False)
                    bits = _status_bits(m.summary())
                    if not bits:
                        kept[name] = _keep(m, dev)
                        break
                if bits & (S.ST_ARRIVALS_OVERFLOW | S.ST_XFER_OVERFLOW):   # flags of the shared headers, clean for the owner
                    raise RuntimeError(f"{name}: {describe_status(bits)} on a group whose owner ran cleanly")
                raise_caps(bits, msp, mcaps, last_attempt=attempt == max_retries)
    except BaseException:
        owner.close()
        raise
    return owner, kept


def compare_variants(variants: Dict[str, Callable], baseline: str, n_replicas: int, seed: int, first_replica_id: int = 0,
                     device: int = 0, rng: str = "philox", quantiles: Sequence[float] = EN.DEFAULT_QUANTILES,
                     max_retries: int = 3) -> PairedComparison:
    """Runs every variant (``name -> spec_factory(caps)``, as ``engine.run_to_completion`` takes) on replicas
    [first_replica_id, first_replica_id + n_replicas) with keys seed + replica id, and reduces each against
    ``baseline``.  Variants whose arrivals are compatible with a group's owner join that group (one pre-pass); the
    baseline owns the first group.  Capacity retries follow run_to_completion: an overflow of a member's running set,
    queues or stale events re-creates that member alone (still shared); an arrival-list or transfer-ring overflow, which
    the pre-pass raises in the group's shared list headers, rebuilds the owner with a doubled cap_arrivals / cap_xfer
    (and its members take the owner's values).  Under torch.distributed every rank runs its shard and the reductions are all-reduced."""
    import torch
    from .engine import arrivals_compatible
    if baseline not in variants:
        raise ValueError(f"baseline {baseline!r} is not one of the variants {sorted(variants)}")
    names = [baseline] + [k for k in variants if k != baseline]
    first = {k: variants[k]({}) for k in names}
    n_dc = first[baseline].n_dc
    if any(sp.n_dc != n_dc for sp in first.values()):
        raise ValueError("compare_variants: every variant must have the baseline's data centres")
    groups = []
    for k in names:
        for g in groups:
            if arrivals_compatible(first[g[0]], first[k]):
                g.append(k)
                break
        else:
            groups.append([k])
    dev = torch.device("cuda", device)
    kept, base = {}, None
    try:
        for g in groups[1:] + groups[:1]:       # the baseline's group last: only its owner stays for the reductions
            owner, got = _run_group(g, variants, n_replicas, seed, first_replica_id, device, rng, max_retries, dev)
            kept.update(got)
            if g[0] == baseline:
                base = owner
            else:
                owner.close()
        stats = {}
        for v in names[1:]:
            stats[v] = _paired_on_device(base, kept[v][0], n_dc, dev, quantiles)
    finally:
        if base is not None:
            base.close()
    return PairedComparison(baseline=baseline, variants=tuple(names[1:]), n_dc=n_dc, stats=stats,
                            shared_arrivals={v: v in groups[0] for v in names[1:]},
                            summaries={k: kept[k][1] for k in names})


def _paired_on_device(base, variant_summary, n_dc, dev, quantiles):
    """The two passes of the paired kernels on the base engine's stream, all-reduced over the ranks."""
    vptr = variant_summary.data_ptr()
    passes = EN.device_passes(dev, n_columns(n_dc), functools.partial(base.paired_moments_into, vptr),
                              functools.partial(base.paired_spread_into, vptr))
    return paired_finalize(*passes, n_dc, quantiles)
