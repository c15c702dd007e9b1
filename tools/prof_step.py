#!/usr/bin/env python
"""One scenario, a few batches: the command ncu wraps for launch lists and `--set full` captures.

    python tools/prof_step.py cfg3_4x64_sinusoid_120s 65536 [batches]
Prints events per batch (the denominator of per-event profiler figures)."""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from distributed_cluster_gpus_b200 import scenarios as SC, spec as S  # noqa: E402
from distributed_cluster_gpus_b200.engine import BatchedEngine  # noqa: E402

name, reps = sys.argv[1], int(sys.argv[2])
batches = int(sys.argv[3]) if len(sys.argv) > 3 else 2
with BatchedEngine(SC.to_spec(SC.BY_NAME[name]), reps, 123) as e:
    for it in range(batches):
        e.reset(123 + it * reps, 0)
        n = e.advance(0)
    s = e.summary()
    print(json.dumps({"scenario": name, "replicas": reps, "events_per_batch": int(n),
                      "arrivals_per_batch": int(s[:, S.S_EV_ARRIVAL].sum()), "launch": e.launch_info()}))
