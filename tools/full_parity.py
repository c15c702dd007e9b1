#!/usr/bin/env python
"""Full-batch parity: EVERY replica of the bench workload (default 65 536 x cfg3, 120 s) from the CUDA kernel
against the oracle run on all host cores.  Prints one JSON line.

    python tools/full_parity.py [--replicas 65536] [--scenario cfg3_4x64_sinusoid_120s]
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))
import numpy as np  # noqa: E402

from distributed_cluster_gpus_b200 import scenarios as SC, spec as S  # noqa: E402
from distributed_cluster_gpus_b200.engine import BatchedEngine  # noqa: E402
import oracle_lib  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--replicas", type=int, default=65536)
ap.add_argument("--scenario", default="cfg3_4x64_sinusoid_120s")
ap.add_argument("--seed", type=int, default=123)
args = ap.parse_args()
sc = SC.BY_NAME[args.scenario]
sp = SC.to_spec(sc)
t0 = time.time()
with BatchedEngine(sp, args.replicas, args.seed) as eng:
    ev = eng.advance(0)
    got = eng.summary()
t_gpu = time.time() - t0
t0 = time.time()
want, ev_o = oracle_lib.run_batch(sp.to_bytes(), args.replicas, args.seed, 0, oracle_lib.RNG_PHILOX, os.cpu_count() or 1)
t_cpu = time.time() - t0
count_cols = [S.S_STATUS, S.S_EVENTS, S.S_JOBS_FINISHED, S.S_JOBS_CREATED, S.S_RNG_WORDS, S.S_SEQ, S.S_DONE]
forks = int(np.count_nonzero(np.any(got[:, count_cols] != want[:, count_cols], axis=1)))
fin = np.maximum(want[:, S.S_JOBS_FINISHED], 1)
rel = lambda a, b: float(np.max(np.abs(a - b) / np.maximum(np.abs(b), 1e-300)))  # noqa: E731
out = {"scenario": sc["name"], "replicas": args.replicas, "events": int(ev), "events_oracle": int(ev_o),
       "replicas_with_any_count_mismatch": forks,
       "max_rel_err_total_energy": rel(got[:, S.S_TOTAL_ENERGY_J], want[:, S.S_TOTAL_ENERGY_J]),
       "max_rel_err_mean_latency": rel(got[:, S.S_LAT_SUM] / fin, want[:, S.S_LAT_SUM] / fin),
       "replicas_bit_identical_energy": int(np.count_nonzero(got[:, S.S_TOTAL_ENERGY_J] == want[:, S.S_TOTAL_ENERGY_J])),
       "tolerance": 1e-9, "gpu_wall_s_incl_alloc": t_gpu, "oracle_wall_s": t_cpu, "host_threads": os.cpu_count()}
print(json.dumps(out))
sys.exit(0 if forks == 0 and out["max_rel_err_total_energy"] <= 1e-9 and out["max_rel_err_mean_latency"] <= 1e-9 else 1)
