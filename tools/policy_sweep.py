#!/usr/bin/env python
"""BASELINE.json config 4: the policy sweep — 4 DC x 64 sim-GPUs, freq_levels {0.5, 0.8, 1.0}, every algo / policy
variant on the device path, N seeds each — with the cross-replica statistics a single-trajectory simulator cannot
give (mean, 95 % CI, quantiles of total energy and mean job latency).  Under torchrun the seeds of every variant are
sharded over the ranks and the 16-double aggregates are all-reduced.

    python tools/policy_sweep.py --seeds 32768 > policy_sweep.json
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402

from distributed_cluster_gpus_b200 import scenarios as SC, sharding, spec as S  # noqa: E402
from distributed_cluster_gpus_b200.engine import BatchedEngine, latency_quantiles  # noqa: E402

VARIANTS = [("default_policy", "energy_aware", {}), ("default_policy", "perf_first", {}), ("joint_nf", "energy_aware", {}),
            ("carbon_cost", "energy_aware", {}), ("eco_route", "energy_aware", {}), ("bandit", "energy_aware", {}),
            ("cap_greedy", "energy_aware", {"power_cap": 20000.0})] + \
           [("debug", "energy_aware", {"num_fixed_gpus": n}) for n in (1, 2, 4, 8)]

ap = argparse.ArgumentParser()
ap.add_argument("--seeds", type=int, default=32768)
ap.add_argument("--duration", type=float, default=120.0)
args = ap.parse_args()
world, rank = int(os.environ.get("WORLD_SIZE", "1")), int(os.environ.get("RANK", "0"))
torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", "0")))
if world > 1:
    dist.init_process_group("nccl")
first, count = sharding.shard(args.seeds, rank, world)
rows = []
for algo, policy, extra in VARIANTS:
    sc = SC.scenario(f"sweep_{algo}_{policy}", 4, 64, SC.SIN10, SC.POI(1.0), args.duration, SC.FREQ3, algo=algo, policy=policy, **extra)
    t0 = time.perf_counter()
    with BatchedEngine(SC.to_spec(sc), count, 123, first, torch.cuda.current_device()) as eng:
        eng.enable_latency_histogram()
        eng.advance(0)
        summ = eng.summary()
        hist = torch.from_numpy(eng.latency_histogram().astype(np.int64)).cuda()
    if world > 1:
        dist.all_reduce(hist)
    hist = hist.cpu().numpy()
    vec = torch.from_numpy(sharding.aggregate_rows(summ)).cuda()
    sharding.allreduce_aggregate(vec)
    st = sharding.finalize(vec.cpu().numpy())
    n = st["replicas"]
    fin = np.maximum(summ[:, S.S_JOBS_FINISHED], 1)
    row = {"algo": algo, "policy": policy, **extra, "seeds": n, "failed": st["failed"], "events": st["events"],
           "energy_MJ_mean": st["energy_j_mean"] / 1e6, "energy_MJ_ci95": 1.96 * (st["energy_j_var"] / n) ** 0.5 / 1e6,
           "mean_job_latency_s_mean": st["mean_latency_s_mean"],
           "mean_job_latency_s_ci95": 1.96 * (st["mean_latency_s_var"] / n) ** 0.5,
           "jobs_finished_per_replica": st["jobs_finished"] / n,
           "job_latency_s_inference_p50_p90_p99": latency_quantiles(hist[0]),
           "job_latency_s_training_p50_p90_p99": latency_quantiles(hist[1]),
           "rank0_energy_MJ_p05_p50_p95": [float(q) / 1e6 for q in np.percentile(summ[:, S.S_TOTAL_ENERGY_J], [5, 50, 95])],
           "rank0_latency_s_p05_p50_p95": [float(q) for q in np.percentile(summ[:, S.S_LAT_SUM] / fin, [5, 50, 95])],
           "wall_s": time.perf_counter() - t0}
    rows.append(row)
    if rank == 0:
        print(json.dumps(row), flush=True)
if world > 1:
    dist.destroy_process_group()
