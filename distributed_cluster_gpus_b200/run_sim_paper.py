"""CLI drop-in for the reference's run_sim_paper.py (flags :18-112 unchanged; batched-engine flags additive).

    python -m distributed_cluster_gpus_b200.run_sim_paper --duration 120 --inf-mode sinusoid --inf-rate 10 \\
        --n-dc 4 --gpus-per-dc 64 --replicas 65536 --log-path out/
"""
import argparse
import json
import os

import numpy as np

from . import spec as S
from .configs.paper_config import (build_arrivals, build_carbon_intensity, build_energy_price, build_policy,
                                   build_router_policy, build_scenario)
from .simcore.logger_config import get_logger
from .simcore.simulator_paper_multi import MultiIngressPaperSimulator
from .simcore.validators import validate_gpus

ALGOS = ["default_policy", "cap_uniform", "cap_greedy", "joint_nf", "bandit", "carbon_cost", "eco_route", "chsac_af",
         "debug"]
# every batch recorder (engine.RECORDERS, in its order) -> the dest of the --X-csv flag that turns it on and names its
# file
RECORDER_CSV = {"cluster_ensemble": "ensemble_csv", "job_ensemble": "job_ensemble_csv",
                "power_profile": "power_profile_csv", "job_waits": "job_waits_csv", "occupancy": "occupancy_csv",
                "tail_latency": "tail_latency_csv", "job_resources": "job_resources_csv", "energy_cost": "energy_cost_csv"}
_ENSEMBLES_REFUSED = ("--ensemble-csv / --job-ensemble-csv / --job-waits-csv are not available with --compare-algos "
                      "(run each algo on its own for its cluster-log and job-log ensembles and its waiting times)")
# why --compare-algos refuses a recorder's flag (the power profile's also refuses --power-threshold), in the order the
# flags are checked
_COMPARE_REFUSALS = {
    "power_profile": "--power-profile-csv / --power-threshold are not available with --compare-algos (run each algo on "
                     "its own)",
    "occupancy": "--occupancy-csv is not available with --compare-algos (run each algo on its own for its occupancy)",
    "tail_latency": "--tail-latency-csv is not available with --compare-algos (run each algo on its own for its per-run "
                    "tail latency)",
    "job_resources": "--job-resources-csv is not available with --compare-algos (run each algo on its own for its GPU, "
                     "frequency and energy-per-job statistics)",
    "energy_cost": "--energy-cost-csv is not available with --compare-algos (run each algo on its own for its electricity "
                   "cost and carbon)",
    "cluster_ensemble": _ENSEMBLES_REFUSED, "job_ensemble": _ENSEMBLES_REFUSED, "job_waits": _ENSEMBLES_REFUSED}


def parse_args(argv=None):
    p = argparse.ArgumentParser(description="Geo GPU simulator (paper-style, multi-ingress) — H100 batched engine",
                                formatter_class=argparse.ArgumentDefaultsHelpFormatter)
    p.add_argument("--duration", type=float, default=180.0, help="simulated seconds")
    p.add_argument("--policy", type=str, default="energy_aware", choices=["energy_aware", "perf_first"])
    p.add_argument("--log-interval", type=float, default=5.0)
    p.add_argument("--log-path", type=str, default=None)
    p.add_argument("--seed", type=int, default=123)
    p.add_argument("--progress", default=True, help="accepted for compatibility; the batched run has no progress bar")
    p.add_argument("--inf-mode", type=str, default="sinusoid", choices=["poisson", "sinusoid", "off"])
    p.add_argument("--inf-rate", type=float, default=6.0)
    p.add_argument("--inf-amp", type=float, default=0.6)
    p.add_argument("--inf-period", type=float, default=300.0)
    p.add_argument("--trn-mode", type=str, default="poisson", choices=["poisson", "sinusoid", "off"])
    p.add_argument("--trn-rate", type=float, default=0.3)
    p.add_argument("--algo", type=str, default="default_policy", choices=ALGOS)
    p.add_argument("--elastic-scaling", type=bool, default=False)
    p.add_argument("--power-cap", type=float, default=0.0)
    p.add_argument("--control-interval", type=float, default=5.0)
    p.add_argument("--eco-objective", type=str, default="energy", choices=["energy", "carbon", "cost"],
                   help="parsed and ignored, as in the reference (never forwarded: SIM:1016)")
    p.add_argument("--num_fixed_gpus", type=int, default=1)
    p.add_argument("--fixed_freq", type=float, default=None)
    p.add_argument("--upgr-buffer", type=int, default=200_000)
    p.add_argument("--upgr-batch", type=int, default=256)
    p.add_argument("--upgr-warmup", type=int, default=1_000)
    p.add_argument("--upgr-device", type=str, default="cuda", choices=["cuda", "cpu"])
    p.add_argument("--sla_p99_ms", type=float, default=500.0)
    p.add_argument("--energy_budget_j", type=float, default=None)
    # --- batched engine ---
    p.add_argument("--replicas", type=int, default=1, help="independent Monte-Carlo replicas (seed, seed+1, ...)")
    p.add_argument("--device", type=int, default=0, help="CUDA device ordinal")
    p.add_argument("--rng", choices=["philox", "mt19937"], default="philox",
                   help="mt19937 = CPython's own generator: replica r reproduces the stock reference at --seed + r")
    p.add_argument("--n-dc", type=int, default=8, help="keep the first N data centres of build_dcs()")
    p.add_argument("--gpus-per-dc", type=int, default=None, help="override total_gpus of every kept DC")
    p.add_argument("--freq-levels", type=str, default=None, help="comma-separated DVFS levels, e.g. 0.5,0.8,1.0")
    p.add_argument("--summary-json", type=str, default=None, help="write per-batch statistics to this file")
    p.add_argument("--ensemble-csv", type=str, default=None, metavar="PATH",
                   help="write per-tick statistics of every DC's cluster-log columns over all replicas (mean, std, min, "
                        "p05/p25/p50/p75/p95, max; long format) to this file")
    p.add_argument("--job-ensemble-csv", type=str, default=None, metavar="PATH",
                   help="write, per finish window and for the whole run, statistics of every DC's job counts and mean "
                        "latencies per job type over all replicas (long format), and per-DC latency quantiles, to this file")
    p.add_argument("--job-ensemble-bin", type=float, default=None, metavar="SECONDS",
                   help="finish-window width of --job-ensemble-csv, --job-waits-csv and --job-resources-csv (default: "
                        "--log-interval)")
    p.add_argument("--job-waits-csv", type=str, default=None, metavar="PATH",
                   help="write, per finish window and for the whole run, statistics of every DC's jobs that waited, mean "
                        "wait (start - xfer_done) and mean response time (finish - arrival) per job type over all "
                        "replicas (the --job-ensemble-csv format), and per-DC wait and response quantiles, to this file")
    p.add_argument("--job-resources-csv", type=str, default=None, metavar="PATH",
                   help="write, per finish window and for the whole run, statistics of every DC's mean GPUs, mean "
                        "frequency and mean predicted energy (E_pred * size) per finished job and job type over all "
                        "replicas (the --job-ensemble-csv format), per-DC energy-per-job quantiles and the pooled "
                        "(GPU count, frequency) mix, to this file")
    p.add_argument("--occupancy-csv", type=str, default=None, metavar="PATH",
                   help="write batch statistics of every DC's time-averaged queue lengths and running jobs, longest "
                        "queues and shares of time queued / saturated / idle, measured between every two events, and "
                        "the pooled queue-length and busy-GPU time distributions, to this file")
    p.add_argument("--tail-latency-csv", type=str, default=None, metavar="PATH",
                   help="write batch statistics of every run's own exact p50 / p95 / p99 / p99.9 / max of service, "
                        "wait and response time per job type and DC, its finished and unfinished jobs, and whether its "
                        "p99 met --sla_p99_ms, to this file")
    p.add_argument("--energy-cost-csv", type=str, default=None, metavar="PATH",
                   help="write batch statistics of every DC's energy, electricity cost under its hourly tariff and "
                        "carbon, the 24 hourly energy bands per DC, and the cluster totals over all replicas, to this "
                        "file")
    p.add_argument("--power-profile-csv", type=str, default=None, metavar="PATH",
                   help="write batch statistics of every replica's cluster power over time — peak, time and energy over "
                        "--power-threshold, longest excursion, per-DC peaks — and the pooled power-duration curve's "
                        "quantiles (long format) to this file")
    p.add_argument("--power-threshold", type=float, default=None, metavar="W",
                   help="threshold of --power-profile-csv (default: --power-cap when it is > 0, else none)")
    p.add_argument("--compare-algos", type=str, default=None, metavar="A,B,...",
                   help="run every listed algo on the scenario of the other flags, on the same replica keys, and compare "
                        "each with the FIRST (the baseline) replica by replica; algos that draw the same arrivals share "
                        "one arrival pre-pass.  cluster_log.csv / job_log.csv are not written in this mode")
    p.add_argument("--compare-csv", type=str, default=None, metavar="PATH",
                   help="with --compare-algos: write the paired statistics (long format, one row per algo and metric) "
                        "to this file")
    p.add_argument("--gpus", type=int, default=1,
                   help="shard the replicas over this many GPUs of the node (one process per GPU; the only collective is "
                        "the all-reduce of the end-of-run statistics over NCCL).  Under torchrun the world size wins.")
    return p.parse_args(argv)


def build_simulator(args, replicas=None, first_replica_id=0, device=None, write_logs=True):
    """argparse namespace -> configured (not yet run) simulator: run_sim_paper.py:115-159 of the reference.
    `replicas` / `first_replica_id` / `device` / `write_logs` describe this process's shard of the batch."""
    levels = [float(x) for x in args.freq_levels.split(",")] if args.freq_levels else None
    ingresses, dcs, graph, coeffs = build_scenario(args.n_dc, args.gpus_per_dc, levels)
    for m in validate_gpus((dc.gpu_type for dc in dcs.values()), strict=False):
        print("[GPU VALIDATION]", m)
    arrival_inf, arrival_trn = build_arrivals(inf_mode=args.inf_mode, inf_rate=args.inf_rate, inf_amp=args.inf_amp,
                                              inf_period=args.inf_period, trn_mode=args.trn_mode,
                                              trn_rate=args.trn_rate)
    if args.log_path:
        norm = os.path.normpath(args.log_path)
        out_dir = os.path.join(norm, args.algo) if os.sep not in norm else norm
    else:
        out_dir = os.getcwd()
    sim = MultiIngressPaperSimulator(
        ingresses=ingresses, dcs=dcs, graph=graph, arrival_inf=arrival_inf, arrival_train=arrival_trn,
        router_policy=build_router_policy(), coeffs_map=coeffs, carbon_intensity=build_carbon_intensity(),
        energy_price=build_energy_price(), policy=build_policy(name=args.policy), sim_duration=args.duration,
        log_interval=args.log_interval, log_path=out_dir, rng_seed=args.seed, algo=args.algo,
        elastic_scaling=(args.elastic_scaling == "True"), power_cap=args.power_cap,
        control_interval=args.control_interval, show_progress=args.progress,
        energy_budget_j=args.energy_budget_j, sla_p99_ms=args.sla_p99_ms, upgr_batch=args.upgr_batch,
        upgr_warmup=args.upgr_warmup, upgr_buffer=args.upgr_buffer, num_fixed_gpus=args.num_fixed_gpus,
        fixed_freq=args.fixed_freq, logger=get_logger(log_dir=out_dir),
        replicas=args.replicas if replicas is None else replicas, first_replica_id=first_replica_id,
        device=args.device if device is None else device, write_logs=write_logs, rng=args.rng,
        job_ensemble_bin=args.job_ensemble_bin, power_threshold=power_threshold(args),
        **{name: getattr(args, dest) is not None for name, dest in RECORDER_CSV.items()})
    return sim


def power_threshold(args):
    """--power-threshold, else --power-cap when it is > 0, else None (no threshold)."""
    if args.power_threshold is not None:
        return float(args.power_threshold)
    return float(args.power_cap) if args.power_cap > 0 else None


def _launch_workers(args, argv):
    """--gpus N outside torchrun: one worker process per GPU through torch's own launcher (rendezvous on 127.0.0.1)."""
    import subprocess
    import sys
    cmd = [sys.executable, "-m", "torch.distributed.run", "--standalone", "--nnodes=1", f"--nproc-per-node={args.gpus}",
           "--local-addr", "127.0.0.1", "-m", "distributed_cluster_gpus_b200.run_sim_paper"] + list(argv if argv is not None else sys.argv[1:])
    return subprocess.run(cmd, check=False).returncode


def main(argv=None):
    args = parse_args(argv)
    world, rank = int(os.environ.get("WORLD_SIZE", "1")), int(os.environ.get("RANK", "0"))
    if world == 1 and args.gpus > 1:            # not under a launcher yet: become one
        rc = _launch_workers(args, argv)
        if rc != 0:
            raise SystemExit(rc)
        return None
    if args.compare_algos:
        return _main_compare(args, world, rank)
    if world > 1:
        return _main_sharded(args, world, rank)
    sim = build_simulator(args)
    sim.run()
    _write_ensemble(args, sim)
    stats = batch_statistics(sim.summary)
    _add_latency_quantiles(stats, sim.latency_histogram)
    _add_recorders(stats, sim)
    _report(args, stats)
    return sim


def _write_ensemble(args, sim):
    for name, dest in RECORDER_CSV.items():
        if getattr(args, dest):
            getattr(sim, name).to_csv(getattr(args, dest), [dc.name for dc in sim.dcs.values()])


def _add_recorders(stats, sim):
    """The batch recorders' figures for --summary-json, each only when its recorder ran."""
    _add_power_profile(stats, sim.power_profile)
    _add_job_waits(stats, sim.job_waits)
    _add_occupancy(stats, sim.occupancy, sim)
    _add_tail_latency(stats, sim.tail_latency)
    _add_job_resources(stats, sim.job_resources, sim)
    _add_energy_cost(stats, sim.energy_cost, sim)


def _add_power_profile(stats, res):
    """The batch figures of the power profile for --summary-json."""
    if res is None:
        return
    col = lambda f: res.column(f)  # noqa: E731
    thr = res.threshold if np.isfinite(res.threshold) else None
    out = {"replicas": res.replicas, "threshold_w": thr, "hi_w": res.hi, "mean_power_w": res.mean_power_w,
           "peak_w_mean": float(res.mean[col("peak_w")]), "peak_w_max": float(res.max[col("peak_w")]),
           "power_w_exceeded_50_10_1_0.1pct": [float(v) for v in res.time_quantiles([0.5, 0.1, 0.01, 0.001])]}
    if thr is not None:
        out.update({"over_s_mean": float(res.mean[col("over_s")]), "over_j_mean": float(res.mean[col("over_j")]),
                    "excursions_mean": float(res.mean[col("excursions")]),
                    "longest_over_s_max": float(res.max[col("longest_over_s")]), "over_share": res.over_share})
    stats["power_profile"] = out


def _add_job_waits(stats, res):
    """Per job type, pooled over DCs and replicas, for --summary-json: mean / p50 / p95 / p99 of wait and response
    time, and the share of jobs that waited."""
    if res is not None:
        stats["job_waits"] = res.pooled()


def _add_occupancy(stats, res, sim):
    """Per DC, for --summary-json: the batch means of mean_q_inf, mean_q_trn, saturated_share and idle_share, and the
    pooled queue length reached for 10 % and 1 % of the time."""
    if res is not None:
        names = [dc.name for dc in sim.dcs.values()]
        stats["occupancy"] = {names[d]: v for d, v in res.pooled().items()}


def _add_tail_latency(stats, res):
    """Per job type and kind, for --summary-json: the share of runs whose p99 met the SLA (95 % Wilson interval) and
    the mean / p05 / p50 / p95 over the runs of the per-run p99."""
    if res is not None:
        stats["tail_latency"] = res.pooled()


def _add_energy_cost(stats, res, sim):
    """For --summary-json: pooled energy [kWh], cost [USD], carbon [g] and the effective USD/kWh and g/kWh, per DC and
    for the cluster, and the batch mean / min / max of each run's cluster cost and carbon."""
    if res is None:
        return
    names = [dc.name for dc in sim.dcs.values()]
    pooled = res.pooled()
    out = {"replicas": pooled["replicas"], "cluster": pooled["cluster"],
           "dc": {names[d]: dict(pooled[d], carbon_g_per_kwh=float(res.carbon_intensity[d])) for d in range(len(names))}}
    for f in ("cost_usd", "carbon_g"):
        c = res.column(f)
        out[f"run_{f}"] = {"mean": float(res.mean[c]), "min": float(res.min[c]), "max": float(res.max[c])}
    stats["energy_cost"] = out


def _add_job_resources(stats, res, sim):
    """Per DC and job type, for --summary-json: pooled jobs, mean GPUs / frequency / predicted energy per job, energy
    quantiles and the (GPU count, frequency) mix as shares."""
    if res is not None:
        names = [dc.name for dc in sim.dcs.values()]
        stats["job_resources"] = {names[d]: v for d, v in res.pooled().items()}


def _add_latency_quantiles(stats, hist):
    from .engine import latency_quantiles
    for jt, name in enumerate(("inference", "training")):        # job-level quantiles over the whole batch
        p50, p90, p99 = latency_quantiles(hist[jt])
        stats[f"job_latency_s_{name}_p50_p90_p99"] = [p50, p90, p99]


def _report(args, stats):
    if args.summary_json:
        with open(args.summary_json, "w") as f:
            json.dump(stats, f, indent=1)
    print(f"Done. ({args.algo}) Logs: cluster_log.csv, job_log.csv  | replicas={stats['replicas']} "
          f"events={stats['events_total']:.0f} mean energy={stats['energy_j_mean']:.6g} J "
          f"(+-{stats['energy_j_ci95']:.3g}) mean latency={stats['mean_latency_s_mean']:.6g} s")


def _main_sharded(args, world, rank):
    """One rank of a replica-sharded run (torchrun / --gpus N): replicas [first, first + count) of the batch on GPU
    LOCAL_RANK, keys from the GLOBAL replica id (results do not depend on N), then ONE all-reduce of the 16-double
    aggregate (+ the 2 x 128 latency histogram) over NCCL; rank 0 — the owner of replica 0 — writes the CSVs and the
    statistics.  Replaces the single-process flow of run_sim_paper.py:117-160 of the reference."""
    import torch
    import torch.distributed as dist
    from . import sharding
    backend = os.environ.get("DCSIM_DIST_BACKEND", "nccl")     # "gloo": several ranks may share a GPU (tests on a 1-GPU box)
    local = int(os.environ.get("LOCAL_RANK", str(rank))) % max(1, torch.cuda.device_count())
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local) if backend == "nccl" else torch.device("cpu")
    if not dist.is_initialized():
        if backend == "nccl":
            dist.init_process_group("nccl", device_id=dev)
        else:
            dist.init_process_group(backend)
    first, count = sharding.shard(args.replicas, rank, world)
    for dest in RECORDER_CSV.values():
        if getattr(args, dest) and count == 0:
            raise SystemExit(f"--{dest.replace('_', '-')} needs at least one replica per rank")
    sim = build_simulator(args, replicas=max(count, 1), first_replica_id=first, device=local, write_logs=(rank == 0))
    sim.run()                                                   # (the ensemble's all-reduces run inside, on every rank)
    if rank == 0:
        _write_ensemble(args, sim)
    summ = sim.summary if count > 0 else sim.summary[:0]
    agg = torch.from_numpy(sharding.aggregate_rows(summ)).to(dev)
    hist = torch.from_numpy(sim.latency_histogram.astype(np.int64) if count > 0 else np.zeros((2, 128), np.int64)).to(dev)
    sharding.allreduce_aggregate(agg)
    dist.all_reduce(hist, op=dist.ReduceOp.SUM)
    # per-replica energies / mean latencies for the percentile rows: gathered (8 bytes per replica and column)
    e = summ[:, S.S_TOTAL_ENERGY_J]
    fin = summ[:, S.S_JOBS_FINISHED]
    ml = np.divide(summ[:, S.S_LAT_SUM], fin, out=np.zeros_like(fin), where=fin > 0)
    width = -(-args.replicas // world)
    mine = torch.full((2, width), float("nan"), dtype=torch.float64, device=dev)
    mine[0, :count] = torch.from_numpy(np.ascontiguousarray(e)).to(dev)
    mine[1, :count] = torch.from_numpy(np.ascontiguousarray(ml)).to(dev)
    everyone = [torch.empty_like(mine) for _ in range(world)]
    dist.all_gather(everyone, mine)
    stats = None
    if rank == 0:
        cols = torch.cat(everyone, dim=1).cpu().numpy()
        keep = ~np.isnan(cols[0])
        stats = sharding.finalize(agg.cpu().numpy())
        n = stats["replicas"]
        ci = lambda var: float(1.96 * np.sqrt(var / n)) if n > 1 else 0.0  # noqa: E731
        stats = {"replicas": n, "gpus": world, "failed": stats["failed"], "events_total": stats["events"],
                 "jobs_finished_total": stats["jobs_finished"], "energy_j_mean": stats["energy_j_mean"],
                 "energy_j_ci95": ci(stats["energy_j_var"]),
                 "energy_j_p05_p50_p95": [float(q) for q in np.percentile(cols[0][keep], [5, 50, 95])],
                 "mean_latency_s_mean": stats["mean_latency_s_mean"], "mean_latency_s_ci95": ci(stats["mean_latency_s_var"]),
                 "mean_latency_s_p05_p50_p95": [float(q) for q in np.percentile(cols[1][keep], [5, 50, 95])]}
        _add_latency_quantiles(stats, hist.cpu().numpy().astype(np.uint64))
        _add_recorders(stats, sim)
        _report(args, stats)
    dist.barrier()
    dist.destroy_process_group()
    sim.batch_stats = stats
    return sim


def _main_compare(args, world, rank):
    """--compare-algos A,B,...: every algo on the same scenario and replica keys (compare.compare_variants), paired with
    the first.  Single-process or one rank of --gpus N (replicas sharded by global id; rank 0 writes)."""
    from . import compare
    algos = [a.strip() for a in args.compare_algos.split(",") if a.strip()]
    if len(algos) < 2 or len(set(algos)) != len(algos):
        raise SystemExit("--compare-algos needs at least two distinct algos")
    unknown = [a for a in algos if a not in ALGOS]
    if unknown:
        raise SystemExit(f"--compare-algos: unknown algo(s) {unknown}; choose from {ALGOS}")
    for name, why in _COMPARE_REFUSALS.items():
        if getattr(args, RECORDER_CSV[name]) or name == "power_profile" and args.power_threshold is not None:
            raise SystemExit(why)
    dist = None
    first, count, device = 0, args.replicas, args.device
    if world > 1:
        import torch
        import torch.distributed as dist
        from . import sharding
        backend = os.environ.get("DCSIM_DIST_BACKEND", "nccl")
        device = int(os.environ.get("LOCAL_RANK", str(rank))) % max(1, torch.cuda.device_count())
        torch.cuda.set_device(device)
        if not dist.is_initialized():
            if backend == "nccl":
                dist.init_process_group("nccl", device_id=torch.device("cuda", device))
            else:
                dist.init_process_group(backend)
        first, count = sharding.shard(args.replicas, rank, world)
        if count == 0:
            raise SystemExit("--compare-algos needs at least one replica per rank")
    sims = {a: build_simulator(argparse.Namespace(**dict(vars(args), algo=a)), replicas=count, first_replica_id=first,
                               device=device, write_logs=False) for a in algos}
    res = compare.compare_variants({a: sims[a]._flatten for a in algos}, algos[0], count, args.seed, first, device, rng=args.rng)
    dc_names = [dc.name for dc in sims[algos[0]].dcs.values()]
    per_algo = {}
    for a in algos:
        summ = res.summaries[a]
        if dist is not None:                                   # every rank's rows, in global replica order
            import torch
            width = -(-args.replicas // world)
            mine = torch.full((width, S.SUMMARY_K), float("nan"), dtype=torch.float64)
            mine[:count] = torch.from_numpy(summ)
            gathered = [torch.empty_like(mine) for _ in range(world)]
            if backend == "gloo":
                dist.all_gather(gathered, mine)
            else:
                dev = torch.device("cuda", device)
                gathered = [g.to(dev) for g in gathered]
                dist.all_gather(gathered, mine.to(dev))
            rows = torch.cat(gathered).cpu().numpy()
            summ = rows[~np.isnan(rows[:, S.S_STATUS])]
        per_algo[a] = batch_statistics(summ)
    if rank == 0:
        if args.compare_csv:
            res.to_csv(args.compare_csv, dc_names)
        if args.summary_json:
            with open(args.summary_json, "w") as f:
                json.dump({"baseline": algos[0], "algos": per_algo, "comparison": res.rows(dc_names)}, f, indent=1)
        for a in algos:
            st = per_algo[a]
            print(f"Done. ({a}) replicas={st['replicas']} events={st['events_total']:.0f} mean energy="
                  f"{st['energy_j_mean']:.6g} J (+-{st['energy_j_ci95']:.3g}) mean latency={st['mean_latency_s_mean']:.6g} s")
        for a in algos[1:]:
            st = res.stats[a]
            print(f"  {a} - {algos[0]}: energy {st.diff_mean[0]:+.6g} J [{st.diff_ci95_lo[0]:+.4g}, {st.diff_ci95_hi[0]:+.4g}] "
                  f"({100 * st.rel_change[0]:+.3f} %), var_ratio {st.var_ratio[0]:.3g}, shared arrivals "
                  f"{res.shared_arrivals[a]}")
    if dist is not None:
        dist.barrier()
        dist.destroy_process_group()
    return res


def batch_statistics(summary: np.ndarray) -> dict:
    """Cross-replica statistics the single-trajectory reference cannot give."""
    e = summary[:, S.S_TOTAL_ENERGY_J]
    fin = summary[:, S.S_JOBS_FINISHED]
    ml = np.divide(summary[:, S.S_LAT_SUM], fin, out=np.zeros_like(fin), where=fin > 0)
    n = len(e)
    ci = lambda x: float(1.96 * x.std(ddof=1) / np.sqrt(n)) if n > 1 else 0.0  # noqa: E731
    return {"replicas": int(n), "events_total": float(summary[:, S.S_EVENTS].sum()),
            "jobs_finished_total": float(fin.sum()), "energy_j_mean": float(e.mean()), "energy_j_ci95": ci(e),
            "energy_j_p05_p50_p95": [float(q) for q in np.percentile(e, [5, 50, 95])],
            "mean_latency_s_mean": float(ml.mean()), "mean_latency_s_ci95": ci(ml),
            "mean_latency_s_p05_p50_p95": [float(q) for q in np.percentile(ml, [5, 50, 95])]}


if __name__ == "__main__":
    main()
