"""Drop-in for the reference's ``MultiIngressPaperSimulator`` (simcore/simulator_paper_multi.py:24-55, 412).

Same constructor arguments, same ``run()``, same result carriers — the ``DataCenter`` objects are mutated in
place and ``cluster_log.csv`` / ``job_log.csv`` are written with the reference's columns and number formats —
but ``run()`` executes ``replicas`` independent trajectories on an H100 through the C-ABI of
include/dcsim_b200.h.  Replica ``r`` is the trajectory the reference would produce for ``rng_seed + r`` when its
``random`` module is backed by the Philox stream of oracle/philox_random.py.  Replica 0 fills the DataCenters and
the CSVs; all replicas are available as ``self.summary`` ([replicas, spec.SUMMARY_K]).

Not on this path (raises): ``algo="chsac_af"`` / ``elastic_scaling`` (online torch agent mutating across events,
SIM:555-573).
"""
import csv
import os
from typing import Dict, Optional, Tuple, Union

import numpy as np

from .. import spec as S
from ..engine import RECORDERS, RNG_KINDS, LoggedReplica, RecorderOverflow, release_engine, run_to_completion
from .arrivals import ArrivalConfig
from .models import DataCenter
from .network import Graph, Ingress
from .policy import PolicyConfig
from .policy_paper import energy_tuple
from .router import RouterPolicy

CLUSTER_HEADER = ["time_s", "dc", "freq", "busy", "free", "run_total", "run_inf", "run_train", "q_inf", "q_train",
                  "util_inst", "util_avg", "acc_job_unit", "power_W", "energy_kJ"]
JOB_HEADER = ["jid", "ingress", "type", "size", "dc", "f_used", "n_gpus", "net_lat_s", "start_s", "finish_s",
              "latency_s", "preempt_count", "T_pred", "P_pred", "E_pred"]


class MultiIngressPaperSimulator:
    def __init__(self,
                 ingresses: Dict[str, Ingress],
                 dcs: Dict[str, DataCenter],
                 graph: Graph,
                 arrival_inf: ArrivalConfig,
                 arrival_train: ArrivalConfig,
                 router_policy: RouterPolicy,
                 coeffs_map: Dict[Tuple, Tuple],
                 logger,
                 carbon_intensity: Optional[Dict[str, float]] = None,
                 energy_price: Optional[Union[Dict[int, float], Dict[str, Dict[int, float]]]] = None,
                 policy: PolicyConfig = None,
                 sim_duration: float = 3600.0,
                 log_interval: float = 10.0,
                 log_path: str = None,
                 rng_seed: int = 42,
                 algo: str = "default_policy",
                 elastic_scaling: bool = False,
                 power_cap: float = 0.0,
                 energy_budget_j: float = 0.0,
                 sla_p99_ms: float = 500.0,
                 control_interval: float = 5.0,
                 show_progress: bool = True,
                 upgr_batch: int = 256, upgr_warmup: int = 1000, upgr_buffer: int = 200000,
                 num_fixed_gpus=1, fixed_freq=None,
                 # --- batched-engine additions (keyword only in spirit; defaults reproduce one trajectory) ---
                 replicas: int = 1, device: int = 0, first_replica_id: int = 0, write_logs: bool = True,
                 cuda_stream: int = 0, keep_engine: bool = True, rng: str = "philox", cluster_ensemble: bool = False,
                 job_ensemble: bool = False, job_ensemble_bin: Optional[float] = None, power_profile: bool = False,
                 power_threshold: Optional[float] = None, job_waits: bool = False, occupancy: bool = False,
                 tail_latency: bool = False, job_resources: bool = False, energy_cost: bool = False):
        self.ingresses, self.dcs, self.graph = ingresses, dcs, graph
        self.arr_inf, self.arr_trn = arrival_inf, arrival_train
        self.router_policy = router_policy          # stored, never consulted — as in the reference (SIM:65)
        self.coeffs_map = coeffs_map
        self.carbon = carbon_intensity or {}
        self.energy_price = energy_price or {}
        self.policy = policy or PolicyConfig(name="energy_aware")
        self.logger = logger
        self.end_time = sim_duration
        self.log_interval = log_interval
        self.rng_seed = int(rng_seed)
        self.algo = algo
        self.power_cap = power_cap
        self.energy_budget_j, self.sla_p99_ms, self.control_interval = energy_budget_j, sla_p99_ms, control_interval
        self.num_fixed_gpus, self.fixed_freq = num_fixed_gpus, fixed_freq
        self.show_progress = bool(show_progress)
        self.replicas, self.device, self.first_replica_id = int(replicas), int(device), int(first_replica_id)
        self.write_logs, self.cuda_stream = bool(write_logs), int(cuda_stream)
        self.keep_engine = bool(keep_engine)   # park the device allocations for the next run of the same shape
        if rng not in RNG_KINDS:
            raise ValueError(f"unknown rng {rng!r}; expected one of {sorted(RNG_KINDS)}")
        self.rng = rng                         # "mt19937": the stock reference's own generator (random.seed, SIM:71)
        if algo == "chsac_af" or elastic_scaling and algo == "chsac_af":
            raise NotImplementedError("algo=chsac_af is outside the batched path (SIM:555-573)")
        self.cluster_log_path, self.job_log_path = "cluster_log.csv", "job_log.csv"
        if log_path:
            os.makedirs(log_path, exist_ok=True)
            self.cluster_log_path = os.path.join(log_path, "cluster_log.csv")
            self.job_log_path = os.path.join(log_path, "job_log.csv")
        self.now = 0.0
        self.summary: Optional[np.ndarray] = None
        self.latency_histogram: Optional[np.ndarray] = None
        self.launch_info: Optional[dict] = None
        # The batch recorders (engine.RECORDERS), each off unless asked for.  After run(), the attribute of the same name
        # holds its statistics over all replicas (of all ranks when torch.distributed runs: every rank's run() takes part
        # in the all-reduces), None when it is off:
        #   cluster_ensemble  per-tick statistics of every DC's cluster-log columns, ensemble.EnsembleResult
        #   job_ensemble      per finish window of job_ensemble_bin seconds (None: log_interval) and for the whole run,
        #                     every DC's job counts and mean latencies, ensemble.JobEnsembleResult
        #   power_profile     the cluster power step function: peak, time and energy over power_threshold watts (None: no
        #                     threshold), per-DC peaks and the pooled power-duration curve, ensemble.PowerProfileResult
        #   job_waits         per finish window and for the whole run, every job's wait (start - xfer_done) and response
        #                     time (finish - arrival), ensemble.JobWaitsResult
        #   occupancy         every DC's time-weighted queue lengths, running jobs and busy GPUs between events,
        #                     ensemble.OccupancyResult
        #   tail_latency      every run's own exact p50 / p95 / p99 / p99.9 / max of service, wait and response time per
        #                     job type and DC, and the share of runs whose p99 met sla_p99_ms, ensemble.TailLatencyResult
        #   job_resources     per finish window and for the whole run, every finished job's GPU count, frequency and
        #                     predicted energy E_pred * size, the pooled (n, f) mix and energy-per-job quantiles,
        #                     ensemble.JobResourcesResult
        #   energy_cost       every DC's energy by hour of day, its cost under the DC's hourly tariff and its carbon,
        #                     ensemble.EnergyCostResult
        # job_waits and job_resources run the job ensemble's recorder too (its windows and job counts).
        self._recorders = dict(cluster_ensemble=bool(cluster_ensemble), job_ensemble=bool(job_ensemble),
                               job_ensemble_bin=job_ensemble_bin, power_profile=bool(power_profile),
                               power_threshold=power_threshold, job_waits=bool(job_waits), occupancy=bool(occupancy),
                               tail_latency=bool(tail_latency), job_resources=bool(job_resources),
                               energy_cost=bool(energy_cost))
        for name in RECORDERS:
            setattr(self, name, None)
        self._spec = self._flatten({})              # validates now, like the reference's constructor would fail now

    # ------------------------------------------------------------------------------------------------
    def _flatten(self, caps):
        return S.flatten(self.ingresses, self.dcs, self.graph, self.arr_inf, self.arr_trn, self.coeffs_map, self.policy,
                         carbon_intensity=self.carbon, energy_price=self.energy_price, sim_duration=self.end_time,
                         log_interval=self.log_interval, algo=self.algo, power_cap=self.power_cap,
                         num_fixed_gpus=self.num_fixed_gpus, fixed_freq=self.fixed_freq, caps=caps)

    def run(self):
        n_ticks = int(self.end_time / self.log_interval) + 2
        expected_jobs = 0.0
        for arr in (self.arr_inf, self.arr_trn):
            if arr.mode != "off":
                expected_jobs += len(self.ingresses) * max(0.0, arr.rate) * (1.0 + abs(arr.amp)) * self.end_time
        job_cap = int(expected_jobs * 1.2 + 10 * expected_jobs ** 0.5 + 64)
        cluster_cap = n_ticks * len(self.dcs)

        # The CSV rows of replica 0 come from a one-replica companion engine running beside the batch (LoggedReplica):
        # recorders inside a big batch cost every replica occupancy.  A batch of one simply logs itself.
        companion = None
        in_batch_log = self.write_logs and self.replicas == 1
        if self.write_logs and not in_batch_log:
            companion = LoggedReplica(self._spec, self.rng_seed, self.first_replica_id, self.device, job_cap, cluster_cap, self.rng)

        def configure(eng):
            eng.set_rng(self.rng)
            eng.enable_latency_histogram()
            if in_batch_log:
                eng.set_logging(0, job_cap, cluster_cap)

        early = {}

        def while_running():
            # the companion's single replica is done long before the batch: fetch its rows and write the CSV files
            # while the GPU is still busy with the batch
            if companion is not None:
                try:
                    bits, jobs, cluster = companion.collect()
                except RecorderOverflow:
                    early["bits"] = -1               # a recorder was too small: replica 0 is logged again below
                    return
                early["bits"] = bits
                if bits == 0:
                    self._write_csvs(jobs, cluster)
                    early["written"] = True

        try:
            eng, summ = run_to_completion(self._flatten, self.replicas, self.rng_seed, self.first_replica_id, self.device,
                                          self.cuda_stream, configure=configure, while_running=while_running,
                                          tail_sla_s=float(self.sla_p99_ms) / 1000.0, **self._recorders)
        except BaseException:
            if companion is not None:
                companion.release(keep=False)
            raise
        try:
            self.summary = summ
            self.latency_histogram = eng.latency_histogram()     # [2, 128] job-latency counts of the whole batch
            self.launch_info = eng.launch_info()
            from .. import ensemble
            for name in RECORDERS:
                if self._recorders[name]:
                    compute = getattr(ensemble, name)
                    setattr(self, name, compute(eng, summary=summ) if name == "power_profile" else compute(eng))
            self._store_replica0(summ[0])
            if in_batch_log:
                try:
                    self._write_csvs(eng.job_log(), eng.cluster_log())
                except RecorderOverflow:
                    self._log_one_replica(eng.spec, job_cap * 2, cluster_cap * 2)
            elif companion is not None:
                if not early.get("written") or eng.spec.to_bytes() != self._spec.to_bytes():
                    # the batch (or the companion) needed larger capacities: log replica 0 again under the final spec
                    companion.release(keep=False)
                    companion = None
                    self._log_one_replica(eng.spec, job_cap, cluster_cap)
        except BaseException:
            eng.close()
            if companion is not None:
                companion.release(keep=False)
            raise
        if companion is not None:
            companion.release(keep=self.keep_engine)
        if self.keep_engine:
            release_engine(eng, eng.spec, self.device, self.cuda_stream)   # next run of this shape re-seeds it
        else:
            eng.close()
        return self

    # ------------------------------------------------------------------------------------------------
    def _store_replica0(self, row):
        """Replica 0 -> the caller's DataCenter objects, as the reference leaves them after run() (SIM:469-475,
        models.py:93-106).  What cannot be materialised — the Job objects still queued or running — is represented by
        its COUNT: `len(dc.q_inf)`, `len(dc.q_train)` and `len(dc.running_jobs)` are right, the elements are
        placeholders (None / jid-less keys); the same counts are also plain attributes (q_inf_len, q_train_len,
        running_count)."""
        self.now = float(row[S.S_LAST_T])
        any_event = row[S.S_EVENTS] > 0
        for d, dc in enumerate(self.dcs.values()):
            g = row[S.S_DC0 + d * S.S_DC_STRIDE: S.S_DC0 + (d + 1) * S.S_DC_STRIDE]
            dc.energy_joules = float(g[S.SD_ENERGY_J])
            dc.util_gpu_time = float(g[S.SD_UTIL_GPU_TIME])
            dc.accumulated_job_unit = float(g[S.SD_ACC_JOB_UNIT])
            dc.busy_gpus = int(g[S.SD_BUSY])
            dc.current_freq = float(g[S.SD_CURRENT_FREQ])
            dc.last_energy_time = self.end_time                       # accrue_energy(end_time) always stamps it
            dc.util_last_ts = self.end_time if any_event else 0.0     # SIM:471-474: untouched (0.0) without events
            dc.util_begin_ts = float(row[S.S_UTIL_BEGIN])             # instant of the first processed event
            dc.q_inf_len, dc.q_train_len, dc.running_count = int(g[S.SD_Q_INF]), int(g[S.SD_Q_TRN]), int(g[S.SD_RUNNING])
            dc.q_inf = [None] * dc.q_inf_len
            dc.q_train = [None] * dc.q_train_len
            dc.running_jobs = {-(i + 1): None for i in range(dc.running_count)}

    def _log_one_replica(self, spec, job_cap, cluster_cap):
        """Replica 0's CSV rows from a one-replica engine of its own; a recorder that turns out too small is
        re-run at the size the device counted (never a silently truncated file)."""
        from ..engine import RecorderOverflow
        for _ in range(4):
            def configure_one(e, jc=job_cap, cc=cluster_cap):
                e.set_rng(self.rng)
                e.set_logging(0, jc, cc)
            one, _s = run_to_completion(lambda caps: spec, 1, self.rng_seed, self.first_replica_id, self.device, 0,
                                        configure=configure_one)
            try:
                jobs, cluster = one.job_log(), one.cluster_log()
            except RecorderOverflow as e:
                if e.which == 1:
                    job_cap = e.needed + 64
                else:
                    cluster_cap = e.needed + 64
                continue
            finally:
                one.close()
            self._write_csvs(jobs, cluster)
            return
        raise RuntimeError("could not size the log recorders")

    def _write_csvs(self, jobs, cluster):
        write_csv_logs(jobs, cluster, self.dcs, list(self.ingresses), self.coeffs_map, self._spec.net_lat_s,
                       self.cluster_log_path, self.job_log_path)


def write_csv_logs(jobs, cluster, dcs, ingress_names, coeffs_map, net_lat_s, cluster_log_path, job_log_path):
    """cluster_log.csv / job_log.csv with the reference's columns and number formats from the engine's unrounded
    records (engine.CLUSTER_DTYPE / JOB_DTYPE).  Rows appear in the reference's order: cluster rows per log tick in
    DC order (SIM:932), job rows in finish order (SIM:814)."""
    dc_names = list(dcs)
    with open(cluster_log_path, "w", newline="") as f:       # SIM:413-418, 944-948
        w = csv.writer(f)
        w.writerow(CLUSTER_HEADER)
        for r in cluster:
            dc = dcs[dc_names[int(r["dc"])]]
            total = dc.total_gpus
            busy = int(r["busy"])
            util_inst = (busy / total) if total else 0.0
            now = float(r["time_s"])
            elapsed = max(1e-9, now - (float(r["util_begin_ts"]) or now))
            util_avg = (float(r["util_gpu_time"]) / (total * elapsed)) if total else 0.0
            w.writerow([f"{now:.3f}", dc.name, f"{float(r['freq']):.2f}", busy, total - busy,
                        int(r["run_total"]), int(r["run_inf"]), int(r["run_total"]) - int(r["run_inf"]),
                        int(r["q_inf"]), int(r["q_train"]), f"{util_inst:.4f}", f"{util_avg:.4f}",
                        f"{float(r['acc_job_unit']):.4f}", f"{float(r['power_w']):.2f}",
                        f"{float(r['energy_j']) / 1000.0:.4f}"])
    with open(job_log_path, "w", newline="") as f:           # SIM:419-421, 814-823
        w = csv.writer(f)
        w.writerow(JOB_HEADER)
        for r in jobs:
            dc_name, ing_name = dc_names[int(r["dc"])], ingress_names[int(r["ingress"])]
            jtype = S.JT_NAMES[int(r["jtype"])]
            p_c, t_c = coeffs_map[(dc_name, jtype)]
            n, f_used = int(r["n_gpus"]), float(r["f_used"])
            t_pred, p_pred, e_pred = energy_tuple(n, f_used, p_c, t_c)
            net_lat = float(net_lat_s[int(r["ingress"])][int(r["dc"])])
            start, finish = float(r["start_s"]), float(r["finish_s"])
            w.writerow([int(r["jid"]), ing_name, jtype, f"{float(r['size']):.4f}", dc_name, f"{f_used:.3f}", n,
                        f"{net_lat:.4f}", f"{start:.6f}", f"{finish:.6f}", f"{(finish - start):.6f}", "0",
                        f"{t_pred:.6f}", f"{p_pred:.2f}", f"{e_pred:.2f}"])
