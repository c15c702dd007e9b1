"""Waiting and response times through the numpy mirror pinned byte for byte (tests/golden/waits/*.csv, checked by
tests/test_job_waits.py): ensemble.job_waits_from_rows on small seeded inputs, written with JobWaitsResult.to_csv
(floats as repr, so the files are bit-exact).

The inputs cover ragged job counts, replicas with a status != 0, all-zero waits (every quantile of wait_s exactly 0), a
mix of zero and positive waits (the quantiles at or below the zero-wait share exactly 0) and empty cells.

    python tests/golden/make_golden_waits.py
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
from distributed_cluster_gpus_b200 import ensemble as EN  # noqa: E402

OUT_DIR = os.path.join(HERE, "waits")
DC_NAMES = ["dc-a", "dc-b", "dc-c"]
BIN_S, END = 10.0, 30.0


def _replica_jobs(rng, n_dc, n_jobs, zero_share):
    """n_jobs jobs of one replica: (dc, jtype, finish, wait, resp), a share of them with wait exactly 0."""
    d = rng.integers(0, n_dc, n_jobs)
    jt = (rng.random(n_jobs) < 0.3).astype(np.int64)
    fin = rng.uniform(0.0, END, n_jobs)
    wait = np.where(rng.random(n_jobs) < zero_share, 0.0, rng.lognormal(-1.0, 1.5, n_jobs))
    resp = wait + rng.lognormal(0.0, 1.0, n_jobs) + 0.05
    return d, jt, fin, wait, resp


def _inputs(seed, n_dc, counts, zero_share, status):
    """What the device recorders of len(counts) replicas hold (finish-order sums, as the device adds them)."""
    rng = np.random.default_rng(seed)
    W, R = EN.job_windows(END, BIN_S), len(counts)
    rows = np.zeros((W + 1, 3, n_dc, 2, R))
    jobs = np.zeros((W + 1, n_dc, 2, R))
    hist = np.zeros((n_dc, 2, 2, EN.LAT_BINS, R), dtype=np.uint32)
    for r, n in enumerate(counts):
        d, jt, fin, wait, resp = _replica_jobs(rng, n_dc, n, zero_share)
        order = np.argsort(fin, kind="stable")
        for i in order:
            k = int(EN.job_window_index(fin[i], BIN_S, W))
            for row in (k, W):
                jobs[row, d[i], jt[i], r] += 1.0
                rows[row, 0, d[i], jt[i], r] += 1.0 if wait[i] > 0.0 else 0.0
                rows[row, 1, d[i], jt[i], r] += wait[i]
                rows[row, 2, d[i], jt[i], r] += resp[i]
            hist[d[i], 0, jt[i], EN.latency_bin(wait[i]), r] += 1
            hist[d[i], 1, jt[i], EN.latency_bin(resp[i]), r] += 1
    return (rows, hist, jobs, np.asarray(status), BIN_S, END), {}


def cases():
    """name -> (args, kwargs) of ensemble.job_waits_from_rows."""
    return {
        # ragged counts (0 to 40 jobs), two bad-status replicas, DC c of type training mostly empty
        "mixed": _inputs(21, 3, [40, 0, 17, 3, 25, 9, 1], 0.45, [0, 0, 0, 4, 0, 0, 16]),
        # nobody waited: every wait_s quantile is exactly 0, waited is 0 everywhere
        "all_zero_waits": _inputs(22, 2, [12, 5, 30], 1.0, [0, 0, 0]),
        # every replica failed: every column empty
        "no_replica": _inputs(23, 2, [6, 4], 0.5, [1, 2]),
    }


def main():
    os.makedirs(OUT_DIR, exist_ok=True)
    for name, (args, kw) in cases().items():
        n_dc = args[0].shape[2]
        EN.job_waits_from_rows(*args, **kw).to_csv(os.path.join(OUT_DIR, f"job_waits_{name}.csv"), DC_NAMES[:n_dc])


if __name__ == "__main__":
    main()
