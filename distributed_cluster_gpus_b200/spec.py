"""Scenario flattening: the reference's dataclasses -> the ``dcsim_spec_t`` blob of include/dcsim_b200.h.

Everything static is resolved here, once, on the host:
  * WAN transfer times per (ingress, DC, job type)  — the reference runs Dijkstra per arrival (SIM:487);
  * (n*, f*) winners of the grid searches          — the reference re-runs them per job (SIM:608, :628, :894);
  * hourly price per DC                             — SIM:986-1005;
  * capacities of the per-replica device structures.
"""
import ctypes as C
import math
import random as _random
from typing import Dict, Optional

from .simcore import arrivals as _arrivals
from .simcore.policy import POLICY_NAMES
from .simcore.policy_paper import best_energy_freq, best_nf_grid

MAX_DC, MAX_ING, MAX_FREQ, HOURS = 8, 8, 16, 24
SPEC_MAGIC = 0x3130304244435344
ABI_VERSION = 2

JT_NAMES = ("inference", "training")
ARR_MODES = {"off": 0, "poisson": 1, "sinusoid": 2}
POLICY_IDS = {"energy_aware": 0, "perf_first": 1}
ALGO_IDS = {"default_policy": 0, "joint_nf": 1, "carbon_cost": 2, "eco_route": 3, "debug": 4, "bandit": 5,
            "cap_uniform": 6, "cap_greedy": 7}
ROUTE_RANDOM, ROUTE_ECO = 0, 1
START_POLICY, START_NF_LUT, START_BANDIT = 0, 1, 2

# summary layout (include/dcsim_b200.h)
S_STATUS, S_EVENTS, S_JOBS_FINISHED, S_JOBS_CREATED, S_TOTAL_ENERGY_J, S_LAT_SUM = 0, 1, 2, 3, 4, 5
S_LAT_SUM_INF, S_FIN_INF, S_LAT_SUM_TRN, S_FIN_TRN, S_RNG_WORDS, S_LAST_T, S_SEQ = 6, 7, 8, 9, 10, 11, 12
S_EV_ARRIVAL, S_EV_XFER, S_EV_FINISH, S_EV_LOG, S_DONE, S_MAX_XFER, S_MAX_RUN, S_MAX_Q = 13, 14, 15, 16, 17, 18, 19, 20
S_UTIL_BEGIN = 21
S_DC0, S_DC_STRIDE = 24, 8
SUMMARY_K = 24 + 8 * MAX_DC
SD_ENERGY_J, SD_UTIL_GPU_TIME, SD_ACC_JOB_UNIT, SD_BUSY, SD_CURRENT_FREQ, SD_Q_INF, SD_Q_TRN, SD_RUNNING = range(8)
ST_XFER_OVERFLOW, ST_RUN_OVERFLOW, ST_QUEUE_OVERFLOW, ST_STALE_OVERFLOW, ST_RNG_RUNAWAY = 1, 2, 4, 8, 16
ST_ARRIVALS_OVERFLOW, ST_ARRIVAL_TIE, ST_SEQ_OVERFLOW = 32, 64, 128
A_REPLICAS, A_FAILED, A_EVENTS, A_JOBS, A_ENERGY, A_ENERGY_SQ, A_LAT_SUM, A_MEANLAT_SUM, A_MEANLAT_SQ, A_RNG_WORDS = range(10)
A_RUNNING = 11
AGG_K = 16
# power-profile columns (DCSIM_PP_*): the fields, then DC_PEAK_W per DC, then PP_BINS histogram bins
PP_PROFILE_S, PP_PEAK_W, PP_T_PEAK_S, PP_OVER_S, PP_OVER_J, PP_EXCURSIONS, PP_LONGEST_OVER_S, PP_OUT_OF_RANGE = range(8)
PP_FIELDS, PP_BINS = 8, 1024
# occupancy columns (DCSIM_OCC_*): PROFILE_S, then per DC the fields (column 1 + field * n_dc + dc), then per DC
# OCC_BINS queue-length bins, then per DC OCC_BINS busy-GPU bins
OCC_Q_INF_AREA, OCC_Q_TRN_AREA, OCC_RUN_AREA, OCC_Q_INF_MAX, OCC_Q_TRN_MAX, OCC_QUEUED_S, OCC_SATURATED_S, OCC_IDLE_S = range(8)
OCC_FIELDS, OCC_BINS = 8, 128
# per-run tail latency columns (DCSIM_TAIL_*): per group (job type, scope: all DCs, then DC 0 ...) the fields JOBS,
# UNFINISHED, then per kind the statistics; after the groups SLA_MET per (kind, job type)
TAIL_JOBS, TAIL_UNFINISHED, TAIL_STATS_BASE = 0, 1, 2
TAIL_KINDS = ("latency", "wait", "response")
TAIL_STATS = ("p50", "p95", "p99", "p999", "max")
TAIL_QUANTILES = (0.5, 0.95, 0.99, 0.999)
TAIL_GROUP_FIELDS = 2 + len(TAIL_KINDS) * len(TAIL_STATS)


def tail_cols(n_dc: int) -> int:
    return 2 * (n_dc + 1) * TAIL_GROUP_FIELDS + 2 * len(TAIL_KINDS)


# energy-cost columns (DCSIM_COST_*): HOUR_J per (dc, hour), then ENERGY_J, COST_USD and CARBON_G per DC, then the three
# cluster totals
COST_WORK_DOUBLES = 3  # the recorder's working row per replica and DC


def cost_hour_j(n_dc: int, dc: int, hour: int) -> int:
    return dc * HOURS + hour


def cost_energy_j(n_dc: int, dc: int) -> int:
    return HOURS * n_dc + dc


def cost_usd(n_dc: int, dc: int) -> int:
    return (HOURS + 1) * n_dc + dc


def cost_carbon_g(n_dc: int, dc: int) -> int:
    return (HOURS + 2) * n_dc + dc


def cost_totals(n_dc: int):
    """(TOTAL_J, TOTAL_USD, TOTAL_G) columns."""
    base = (HOURS + 3) * n_dc
    return base, base + 1, base + 2


def cost_cols(n_dc: int) -> int:
    return (HOURS + 3) * n_dc + 3


def cost_bytes_per_replica(n_dc: int) -> int:
    """Device bytes per replica of the energy-cost recorder: its columns and its working rows."""
    return 8 * (cost_cols(n_dc) + COST_WORK_DOUBLES * n_dc)


def tail_col(n_dc: int, jt: int, field: int, dc: int = -1) -> int:
    """Column of group (jt, dc) (dc = -1: all DCs) and field (TAIL_JOBS, TAIL_UNFINISHED or TAIL_STATS_BASE + kind * 5 +
    stat)."""
    return (jt * (n_dc + 1) + dc + 1) * TAIL_GROUP_FIELDS + field


def tail_sla_col(n_dc: int, kind: int, jt: int) -> int:
    return 2 * (n_dc + 1) * TAIL_GROUP_FIELDS + kind * 2 + jt


class Coeffs(C.Structure):
    _fields_ = [("alpha_p", C.c_double), ("beta_p", C.c_double), ("gamma_p", C.c_double),
                ("alpha_t", C.c_double), ("beta_t", C.c_double), ("gamma_t", C.c_double)]


class NF(C.Structure):
    _fields_ = [("n", C.c_int32), ("_pad", C.c_int32), ("f", C.c_double)]


class DCSpec(C.Structure):
    _fields_ = [("total_gpus", C.c_int32), ("power_gating", C.c_int32), ("n_freq", C.c_int32), ("_pad", C.c_int32),
                ("p_idle", C.c_double), ("p_peak", C.c_double), ("p_sleep", C.c_double), ("alpha", C.c_double),
                ("default_freq", C.c_double), ("freq_levels", C.c_double * MAX_FREQ),
                ("carbon_intensity", C.c_double), ("price_kwh", C.c_double * HOURS),
                ("coeffs", Coeffs * 2), ("nf_xfer", (NF * HOURS) * 2), ("nf_deq", NF * 2),
                ("eco_e_unit", C.c_double * 2)]


class Arrival(C.Structure):
    _fields_ = [("mode", C.c_int32), ("_pad", C.c_int32), ("rate", C.c_double), ("amp", C.c_double),
                ("period", C.c_double)]


class Spec(C.Structure):
    _fields_ = [("magic", C.c_uint64), ("abi_version", C.c_uint32), ("spec_bytes", C.c_uint32),
                ("n_dc", C.c_int32), ("n_ing", C.c_int32), ("algo", C.c_int32), ("policy_name", C.c_int32),
                ("max_gpus_per_job", C.c_int32), ("inf_priority", C.c_int32),
                ("train_scale_out_low_freq", C.c_int32), ("num_fixed_gpus", C.c_int32),
                ("route_rule", C.c_int32), ("xfer_rule", C.c_int32), ("deq_rule", C.c_int32),
                ("control_lower_idle", C.c_int32),
                ("dvfs_low", C.c_double), ("dvfs_high", C.c_double), ("fixed_freq", C.c_double),
                ("end_time", C.c_double), ("log_interval", C.c_double), ("power_cap", C.c_double),
                ("pareto_xm", C.c_double), ("pareto_inv_alpha", C.c_double), ("lognorm_mu", C.c_double),
                ("lognorm_sigma", C.c_double), ("lognorm_floor", C.c_double), ("uniform_floor", C.c_double),
                ("nv_magicconst", C.c_double), ("two_pi", C.c_double),
                ("arr", Arrival * 2),
                ("transfer_s", ((C.c_double * 2) * MAX_DC) * MAX_ING),
                ("net_lat_s", (C.c_double * MAX_DC) * MAX_ING),
                ("dc", DCSpec * MAX_DC),
                ("cap_xfer", C.c_int32), ("cap_run", C.c_int32), ("cap_q_inf", C.c_int32),
                ("cap_q_trn", C.c_int32), ("cap_stale", C.c_int32), ("cap_arrivals", C.c_int32)]

    def to_bytes(self) -> bytes:
        return bytes(memoryview(self).cast("B"))


class TraceRec(C.Structure):
    _fields_ = [("t", C.c_double), ("seq", C.c_uint32), ("kind", C.c_uint32)]


class JobRec(C.Structure):
    _fields_ = [("jid", C.c_uint32), ("n_gpus", C.c_uint32), ("ingress", C.c_uint8), ("jtype", C.c_uint8),
                ("dc", C.c_uint8), ("_pad0", C.c_uint8), ("_pad1", C.c_uint32), ("size", C.c_double),
                ("f_used", C.c_double), ("start_s", C.c_double), ("finish_s", C.c_double)]


class ClusterRec(C.Structure):
    _fields_ = [("time_s", C.c_double), ("freq", C.c_double), ("util_gpu_time", C.c_double),
                ("util_begin_ts", C.c_double), ("acc_job_unit", C.c_double), ("power_w", C.c_double),
                ("energy_j", C.c_double), ("dc", C.c_int32), ("busy", C.c_int32), ("run_total", C.c_int32),
                ("run_inf", C.c_int32), ("q_inf", C.c_int32), ("q_train", C.c_int32)]


class LaunchInfo(C.Structure):
    _fields_ = [("warps_per_cta", C.c_int32), ("ctas", C.c_int32), ("smem_bytes_per_cta", C.c_int32),
                ("regs_per_thread", C.c_int32), ("resident_warps_per_sm", C.c_int32), ("sm_count", C.c_int32),
                ("cap_xfer", C.c_int32), ("cap_run", C.c_int32), ("cap_q_inf", C.c_int32), ("cap_q_trn", C.c_int32),
                ("kernel_launches", C.c_int32), ("arrivals_prepass", C.c_int32),
                ("hbm_bytes_state", C.c_uint64), ("hbm_bytes_queues", C.c_uint64), ("hbm_bytes_arrivals", C.c_uint64),
                ("staging_mode", C.c_int32), ("state_block_bytes", C.c_int32), ("staged_bytes_per_replica", C.c_int32),
                ("lanes_per_replica", C.c_int32)]


def _price_for(energy_price, dc_name: str, hour: int) -> float:
    """SIM:986-1005 for a given hour."""
    ep = energy_price or {}
    if ep and all(isinstance(k, int) for k in ep.keys()):
        return float(ep.get(hour, 0.0))
    per_dc = ep.get(dc_name) if isinstance(ep, dict) else None
    if isinstance(per_dc, dict):
        return float(per_dc.get(hour, 0.0))
    return 0.0


def net_tuple(graph, src: str, dst: str, jtype: str):
    """(Lnet_s, bottleneck, cost, transfer_s) per SIM:482-496."""
    lnet_s, _path, bottleneck, cost = graph.shortest_path_latency(src, dst)
    data_gb = 0.05 if jtype == "inference" else 5.0
    xfer_s = data_gb / bottleneck if (bottleneck and bottleneck > 0.0) else 0.0
    return lnet_s, bottleneck, cost, lnet_s + xfer_s


def _poisson_cap(mean: float, floor: int, slack_sigmas: float = 8.0) -> int:
    return int(max(floor, math.ceil(mean + slack_sigmas * math.sqrt(max(mean, 1.0)) + floor / 2)))


def flatten(ingresses, dcs, graph, arrival_inf, arrival_train, coeffs_map, policy, *,
            carbon_intensity: Optional[Dict[str, float]] = None, energy_price=None,
            sim_duration: float = 3600.0, log_interval: float = 10.0, algo: str = "default_policy",
            power_cap: float = 0.0, num_fixed_gpus: int = 1, fixed_freq=None,
            caps: Optional[Dict[str, int]] = None) -> Spec:
    """Build the spec blob.  Raises the reference's own exception types for the reference's own error cases."""
    if algo == "chsac_af":
        raise NotImplementedError("algo=chsac_af (online torch SAC agent, SIM:555-573) is outside the batched path")
    if algo not in ALGO_IDS:
        raise ValueError(f"unknown algo {algo!r}")
    if policy.name not in POLICY_NAMES:
        raise ValueError("Unknown policy name")                      # policy.py:41
    n_dc, n_ing = len(dcs), len(ingresses)
    if not 1 <= n_dc <= MAX_DC or not 1 <= n_ing <= MAX_ING:
        raise ValueError(f"batched engine supports 1..{MAX_DC} DCs and 1..{MAX_ING} ingresses (got {n_dc}, {n_ing})")
    if not (log_interval > 0.0):
        raise ZeroDivisionError("float modulo")                      # finish_time % log_interval, SIM:711
    carbon = carbon_intensity or {}

    sp = Spec()
    sp.magic, sp.abi_version, sp.spec_bytes = SPEC_MAGIC, ABI_VERSION, C.sizeof(Spec)
    sp.n_dc, sp.n_ing = n_dc, n_ing
    sp.algo, sp.policy_name = ALGO_IDS[algo], POLICY_IDS[policy.name]
    sp.max_gpus_per_job = int(policy.max_gpus_per_job)
    sp.inf_priority = int(bool(policy.inf_priority))
    sp.train_scale_out_low_freq = int(bool(policy.train_scale_out_low_freq))
    sp.num_fixed_gpus = int(num_fixed_gpus)
    sp.route_rule = ROUTE_ECO if algo == "eco_route" else ROUTE_RANDOM
    sp.xfer_rule = {"joint_nf": START_NF_LUT, "carbon_cost": START_NF_LUT, "debug": START_NF_LUT,
                    "bandit": START_BANDIT}.get(algo, START_POLICY)
    sp.deq_rule = {"joint_nf": START_NF_LUT, "carbon_cost": START_NF_LUT, "bandit": START_BANDIT}.get(algo, START_POLICY)
    sp.control_lower_idle = int(power_cap > 0 and algo in ("eco_route", "carbon_cost"))      # SIM:221-225
    sp.dvfs_low, sp.dvfs_high = float(policy.dvfs_low), float(policy.dvfs_high)
    sp.fixed_freq = float(fixed_freq) if fixed_freq else 0.0
    sp.end_time, sp.log_interval, sp.power_cap = float(sim_duration), float(log_interval), float(power_cap)

    sp.pareto_xm = float(_arrivals.PARETO_XM)
    sp.pareto_inv_alpha = 1 / _arrivals.PARETO_ALPHA
    sp.lognorm_mu = math.log(_arrivals.LOGNORM_MEDIAN)
    sp.lognorm_sigma = _arrivals.LOGNORM_SIGMA
    sp.lognorm_floor = _arrivals.LOGNORM_FLOOR
    sp.uniform_floor = _arrivals.UNIFORM_FLOOR
    sp.nv_magicconst = _random.NV_MAGICCONST
    sp.two_pi = 2 * math.pi

    for k, arr in enumerate((arrival_inf, arrival_train)):
        if arr.mode not in ARR_MODES:
            raise ValueError("Unknown mode")                         # arrivals.py:33,48
        if arr.mode == "sinusoid" and not (arr.rate > 0 and arr.period > 0):
            raise ZeroDivisionError("sinusoid arrivals need rate > 0 and period > 0 (arrivals.py:44 divides by max_rate)")
        if arr.mode == "sinusoid" and abs(arr.amp) > 1.0:
            raise ValueError("sinusoid arrivals with |amp| > 1 never terminate in the reference "
                             "(arrivals.py:41-45 keeps redrawing while lambda(t) is clipped to 0)")
        a = sp.arr[k]
        a.mode, a.rate, a.amp, a.period = ARR_MODES[arr.mode], float(arr.rate), float(arr.amp), float(arr.period)

    dc_names = list(dcs)
    max_transfer = 0.0
    for i, ing in enumerate(ingresses.values()):
        for d, name in enumerate(dc_names):
            for jt, jname in enumerate(JT_NAMES):
                lnet, _bn, _cost, transfer = net_tuple(graph, ing.name, name, jname)
                sp.transfer_s[i][d][jt] = transfer
                sp.net_lat_s[i][d] = lnet
                if math.isfinite(transfer):
                    max_transfer = max(max_transfer, transfer)

    n_min_start = int(policy.max_gpus_per_job)
    for d, name in enumerate(dc_names):
        dc = dcs[name]
        levels = list(dc.freq_levels)
        if not 1 <= len(levels) <= MAX_FREQ:
            raise ValueError(f"DC {name}: 1..{MAX_FREQ} freq_levels supported")
        if dc.default_freq not in levels:
            raise AssertionError("default_freq must be one of freq_levels")  # models.py:75
        if int(dc.total_gpus) > 65535:
            raise ValueError(f"DC {name}: at most 65535 GPUs per data centre (a running record packs the job's GPU count into 16 bits)")
        o = sp.dc[d]
        o.total_gpus, o.power_gating, o.n_freq = int(dc.total_gpus), int(bool(dc.power_gating)), len(levels)
        gt = dc.gpu_type
        o.p_idle, o.p_peak, o.p_sleep, o.alpha = float(gt.p_idle), float(gt.p_peak), float(gt.p_sleep), float(gt.alpha)
        o.default_freq = float(dc.default_freq)
        for k, f in enumerate(levels):
            o.freq_levels[k] = float(f)
        o.carbon_intensity = float(carbon.get(name, 0.0))
        for h in range(HOURS):
            o.price_kwh[h] = _price_for(energy_price, name, h)
        for jt, jname in enumerate(JT_NAMES):
            p_c, t_c = coeffs_map[(name, jname)]
            c = o.coeffs[jt]
            c.alpha_p, c.beta_p, c.gamma_p = p_c.alpha_p, p_c.beta_p, p_c.gamma_p
            c.alpha_t, c.beta_t, c.gamma_t = t_c.alpha_t, t_c.beta_t, t_c.gamma_t
            n_e, f_e, _t, _p, e_unit = best_nf_grid(policy.max_gpus_per_job, levels, p_c, t_c, objective="energy")
            o.eco_e_unit[jt] = e_unit
            if algo == "joint_nf":
                for h in range(HOURS):
                    o.nf_xfer[jt][h].n, o.nf_xfer[jt][h].f = n_e, f_e
                o.nf_deq[jt].n, o.nf_deq[jt].f = n_e, f_e
                n_min_start = min(n_min_start, n_e)
            elif algo == "carbon_cost":
                ci = o.carbon_intensity
                n_c, f_c, *_ = best_nf_grid(policy.max_gpus_per_job, levels, p_c, t_c, objective="carbon",
                                            carbon_intensity=ci)
                for h in range(HOURS):
                    price = o.price_kwh[h]
                    if price > 0.0:
                        n_h, f_h, *_ = best_nf_grid(policy.max_gpus_per_job, levels, p_c, t_c, objective="cost",
                                                    price_kwh=price)
                    else:
                        n_h, f_h = n_c, f_c
                    o.nf_xfer[jt][h].n, o.nf_xfer[jt][h].f = n_h, f_h
                    n_min_start = min(n_min_start, n_h)
                o.nf_deq[jt].n, o.nf_deq[jt].f = n_c, f_c
                n_min_start = min(n_min_start, n_c)
            elif algo == "debug":
                n_dbg = int(num_fixed_gpus)
                f_dbg = float(fixed_freq) if fixed_freq else best_energy_freq(n_dbg, levels, p_c, t_c)
                for h in range(HOURS):
                    o.nf_xfer[jt][h].n, o.nf_xfer[jt][h].f = n_dbg, f_dbg
                n_min_start = min(n_min_start, max(1, n_dbg))

    # ---- capacities --------------------------------------------------------------------------------
    peak = [a.peak_rate() if a.mode == "sinusoid" else (a.rate if a.mode == "poisson" else 0.0)
            for a in (arrival_inf, arrival_train)]
    peak = [max(0.0, p) for p in peak]
    inflight = n_ing * (peak[0] + peak[1]) * max_transfer
    cap_xfer = -(-_poisson_cap(inflight, 16) // 8) * 8
    g_max = max(int(dc.total_gpus) for dc in dcs.values())
    cap_run = min(g_max, -(-g_max // max(1, n_min_start)) + 8)
    share = 1.0 if algo == "eco_route" else 1.0 / n_dc   # eco_route may send a whole class to one DC
    cap_q = [_poisson_cap(n_ing * p * float(sim_duration) * share, 32) for p in peak]
    sp.cap_xfer, sp.cap_run, sp.cap_q_inf, sp.cap_q_trn = cap_xfer, max(1, cap_run), cap_q[0], cap_q[1]
    # cap_greedy: every DVFS step of a running job leaves one superseded job_finish event behind (SIM:330-338)
    n_freq_max = max(len(list(dc.freq_levels)) for dc in dcs.values())
    sp.cap_stale = min(512, max(64, n_dc * max(1, cap_run) * max(1, n_freq_max - 1) // 4)) if algo == "cap_greedy" else 0
    sp.cap_arrivals = _poisson_cap(n_ing * (peak[0] + peak[1]) * float(sim_duration), 64)
    for key, val in (caps or {}).items():
        if key not in ("cap_xfer", "cap_run", "cap_q_inf", "cap_q_trn", "cap_stale", "cap_arrivals"):
            raise ValueError(f"unknown capacity {key!r}")
        setattr(sp, key, int(val))
    return sp


def full_run_capacity(sp: Spec, dcs) -> Dict[str, int]:
    """Worst-case running-set capacity (every job on one GPU), used when a replica reports RUN overflow."""
    return {"cap_run": max(int(dc.total_gpus) for dc in dcs.values())}
