"""Per-run tail latency through the numpy mirror pinned byte for byte (tests/golden/tail/tail_latency_*.csv, checked by
tests/test_tail_latency.py): ensemble.tail_latency_from_jobs on small seeded inputs, written with
TailLatencyResult.to_csv (floats as repr, so the files are bit-exact).

The inputs cover ragged job counts (0 to 60 created jobs), unfinished jobs, replicas with a status != 0, exact-zero
waits, empty groups (a DC no training job reached) and a run without an SLA (its *_sla_met rows stay empty).

    python tests/golden/make_golden_tail_csv.py
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
from distributed_cluster_gpus_b200 import ensemble as EN  # noqa: E402

OUT_DIR = os.path.join(HERE, "tail")
DC_NAMES = ["dc-a", "dc-b", "dc-c"]


def _replica_jobs(rng, n_dc, n_jobs, unfinished_share):
    """n_jobs created jobs of one replica (EN.TAIL_JOB_DTYPE): training jobs never reach the last DC."""
    j = np.zeros(n_jobs, dtype=EN.TAIL_JOB_DTYPE)
    j["jtype"] = (rng.random(n_jobs) < 0.3).astype(np.int32)
    j["dc"] = np.where(j["jtype"] == 1, rng.integers(0, max(n_dc - 1, 1), n_jobs), rng.integers(0, n_dc, n_jobs))
    j["arrival"] = rng.uniform(0.0, 60.0, n_jobs)
    j["xfer_done"] = j["arrival"] + rng.uniform(0.0, 0.2, n_jobs)
    wait = np.where(rng.random(n_jobs) < 0.6, 0.0, rng.lognormal(-1.0, 1.5, n_jobs))
    j["start"] = j["xfer_done"] + wait
    j["finish"] = j["start"] + rng.lognormal(-1.5, 1.0, n_jobs)
    j["finish"][rng.random(n_jobs) < unfinished_share] = np.nan
    j["start"][np.isnan(j["finish"])] = np.nan
    return j


def _inputs(seed, n_dc, counts, status, sla_s):
    rng = np.random.default_rng(seed)
    jobs = [_replica_jobs(rng, n_dc, n, 0.15) for n in counts]
    return (jobs, np.asarray(status), n_dc), {"sla_s": sla_s}


def cases():
    """name -> (args, kwargs) of ensemble.tail_latency_from_jobs."""
    return {
        # ragged counts, two bad-status replicas, DC c without training jobs, SLA 0.5 s
        "mixed": _inputs(31, 3, [60, 0, 17, 3, 41, 9, 1], [0, 0, 0, 4, 0, 0, 16], 0.5),
        # no SLA: the *_sla_met rows stay empty
        "no_sla": _inputs(32, 2, [12, 25, 30], [0, 0, 0], None),
        # every replica failed: every column empty
        "no_replica": _inputs(33, 2, [6, 4], [1, 2], 0.5),
    }


def main():
    os.makedirs(OUT_DIR, exist_ok=True)
    for name, (args, kw) in cases().items():
        EN.tail_latency_from_jobs(*args, **kw).to_csv(os.path.join(OUT_DIR, f"tail_latency_{name}.csv"), DC_NAMES[:args[2]])


if __name__ == "__main__":
    main()
