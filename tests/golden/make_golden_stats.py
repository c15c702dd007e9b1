"""Batch statistics of the numpy mirrors pinned byte for byte (tests/golden/stats/*.csv, checked by
tests/test_batch_stats_pinned.py): the cluster-log ensemble, the job-log ensemble, the power profile and the paired
comparison on small seeded inputs, each written with its own to_csv (floats as repr, so the files are bit-exact).

The inputs cover ragged log counts, replicas with a status != 0, an integer field spread over more than BINS values,
empty and single-sample columns, and power profiles with and without a threshold.

    python tests/golden/make_golden_stats.py
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
from distributed_cluster_gpus_b200 import compare as CP, ensemble as EN, spec as S  # noqa: E402

OUT_DIR = os.path.join(HERE, "stats")
DC_NAMES = ["dc-a", "dc-b", "dc-c"]


def _cluster(path):
    rng = np.random.default_rng(11)
    T, n_dc, R = 4, 2, 7
    rows = rng.normal(100.0, 30.0, size=(T, len(EN.FIELDS), n_dc, R))
    rows[:, 1] = rng.integers(0, 3000, size=(T, n_dc, R))             # busy: an integer field over > BINS values
    rows[:, 2:7] = rng.integers(0, 40, size=(T, 5, n_dc, R))
    nlog = np.array([3, 1, 2, 0, 2, 2, 1])                            # ragged; tick 2 has one sample, tick 3 none
    for r in range(R):
        rows[nlog[r]:, :, :, r] = np.nan                                # what the device holds for unrecorded ticks
    EN.cluster_ensemble_from_rows(rows, nlog, 5.0).to_csv(path, DC_NAMES[:n_dc])


def _job(path):
    rng = np.random.default_rng(12)
    W, n_dc, R = 3, 2, 6
    jobs = rng.integers(0, 2500, size=(W, n_dc, 2, R)).astype(np.float64)    # > BINS distinct counts
    jobs[:, 1, 1] = 0.0                                                 # dc 1 training: no jobs, empty latency column
    jobs[0, 0, 1] = 0.0
    jobs[0, 0, 1, 2] = 3.0                                              # window 0, dc 0 training: one sample
    lat = jobs * rng.uniform(0.5, 4.0, size=jobs.shape)
    rows = np.zeros((W + 1, 2, n_dc, 2, R))
    rows[:W, 0], rows[:W, 1] = jobs, lat
    rows[W] = rows[:W].sum(axis=0)
    hist = rng.integers(0, 50, size=(n_dc, 2, EN.LAT_BINS, R)).astype(np.uint32)
    status = np.array([0, 0, 0, 4, 0, 1])
    EN.job_ensemble_from_rows(rows, hist, status, 7.0, 20.0).to_csv(path, DC_NAMES[:n_dc])


def _power(path, threshold, good):
    rng = np.random.default_rng(13)
    n_dc, R = 3, 9
    nf = len(EN.PP_FIELDS)
    rows = np.zeros((nf + n_dc + EN.PP_BINS, R))
    rows[:nf] = rng.uniform(0.0, 500.0, size=(nf, R))
    rows[S.PP_EXCURSIONS] = rng.integers(0, 4000, size=R)              # > BINS values
    rows[S.PP_OUT_OF_RANGE] = rng.integers(0, 3, size=R)
    rows[nf:nf + n_dc] = rng.uniform(1000.0, 9000.0, size=(n_dc, R))
    rows[nf + n_dc:] = rng.uniform(0.0, 2.0, size=(EN.PP_BINS, R)) * (rng.random((EN.PP_BINS, R)) < 0.1)
    summary = np.zeros((R, S.SUMMARY_K))
    summary[:, S.S_TOTAL_ENERGY_J] = rng.uniform(1e5, 2e5, size=R)
    summary[~good, S.S_STATUS] = 2.0
    EN.power_profile_from_rows(rows, summary, 12000.0, threshold).to_csv(path, DC_NAMES[:n_dc])


def _summaries(rng, R, n_dc):
    s = np.zeros((R, S.SUMMARY_K))
    s[:, S.S_TOTAL_ENERGY_J] = rng.uniform(1e5, 2e5, size=R)
    s[:, S.S_FIN_INF] = rng.integers(0, 3000, size=R)                  # > BINS values of jobs_inf and its difference
    s[:, S.S_FIN_TRN] = rng.integers(0, 5, size=R)
    s[:, S.S_JOBS_FINISHED] = s[:, S.S_FIN_INF] + s[:, S.S_FIN_TRN]
    s[:, S.S_LAT_SUM_INF] = s[:, S.S_FIN_INF] * rng.uniform(0.1, 2.0, size=R)
    s[:, S.S_LAT_SUM_TRN] = s[:, S.S_FIN_TRN] * rng.uniform(5.0, 50.0, size=R)
    for d in range(n_dc):
        g = S.S_DC0 + d * S.S_DC_STRIDE
        s[:, g + S.SD_Q_INF] = rng.integers(0, 9, size=R)
        s[:, g + S.SD_RUNNING] = rng.integers(0, 9, size=R)
        s[:, g + S.SD_ENERGY_J] = rng.uniform(1e4, 6e4, size=R)
        s[:, g + S.SD_CURRENT_FREQ] = 1.0
    return s


def _paired(path, n_dc, degenerate):
    rng = np.random.default_rng(14 + degenerate)
    R = 8
    base, var = _summaries(rng, R, 3), _summaries(rng, R, 3)
    base[2, S.S_STATUS], var[5, S.S_STATUS] = 4.0, 1.0
    if degenerate:
        base[:, S.S_FIN_TRN] = 0.0                                      # mean_latency_trn: one replica defined in both
        base[0, S.S_FIN_TRN], base[0, S.S_LAT_SUM_TRN] = 1.0, 30.0
        var[:, S.S_JOBS_FINISHED] = 0.0                                 # energy_per_job: no replica defined
    st = CP.paired_from_summaries(base, var, n_dc=n_dc)
    names = DC_NAMES[:st.metrics.count(CP.DC_METRIC)]
    CP.PairedComparison(baseline="base", variants=("var",), n_dc=len(names), stats={"var": st},
                        shared_arrivals={"var": True}, summaries={}).to_csv(path, names)


CASES = {
    "cluster_ensemble.csv": _cluster,
    "job_ensemble.csv": _job,
    "power_profile_threshold.csv": lambda p: _power(p, 6000.0, np.array([1, 1, 0, 1, 1, 1, 0, 1, 1], dtype=bool)),
    "power_profile_no_threshold.csv": lambda p: _power(p, None, np.array([1, 1, 0, 1, 1, 1, 0, 1, 1], dtype=bool)),
    "power_profile_one_replica.csv": lambda p: _power(p, 6000.0, np.arange(9) == 4),
    "power_profile_no_replica.csv": lambda p: _power(p, None, np.zeros(9, dtype=bool)),
    "paired.csv": lambda p: _paired(p, 3, False),
    "paired_degenerate.csv": lambda p: _paired(p, None, True),
}


def write_all(out_dir):
    os.makedirs(out_dir, exist_ok=True)
    for name, fn in CASES.items():
        fn(os.path.join(out_dir, name))


if __name__ == "__main__":
    write_all(OUT_DIR)
    print("wrote", ", ".join(CASES), "to", OUT_DIR)
