"""Job-log ensemble on the CPU: the recorder of the device source (host build, tests/hostemu) against every
replica's oracle job log, the window rule, the numpy mirror of the reductions against numpy, the CSV, and the two-rank
all-reduce (gloo) against one rank."""
import os
import sys

import numpy as np
import pytest
import torch.distributed as dist
import torch.multiprocessing as mp

import hostemu_lib as H
from conftest import ROOT
from distributed_cluster_gpus_b200 import ensemble as EN, scenarios as SC, spec as S

FIXTURES = ["cfg3_4x64_sinusoid_120s", "sweep_joint_nf", "cap_greedy_4x64", "ragged_3dc_12_5_40", "carbon_cost_8h_2x16"]
SEED = 4100
JOBLOG_CAP = 1 << 18


def oracle_job_rows(oracle, sp, seed, bin_s, rng_kind=0):
    """(rows [W + 1, 2, n_dc, 2], hist [n_dc, 2, LAT_BINS]) of one replica, binned from its oracle job log."""
    sim = oracle.OracleSim(sp.to_bytes(), seed, rng_kind=rng_kind, joblog_cap=JOBLOG_CAP)
    sim.advance(0)
    log = sim.job_log()
    jobs = int(sim.summary()[S.S_JOBS_FINISHED])
    sim.close()
    assert len(log) == jobs < JOBLOG_CAP
    return EN.rows_from_job_log(log, sp.n_dc, bin_s, sp.end_time)


def _check_recorded(oracle, sp, got, seed0, n, bin_s, rng_kind=0):
    assert np.all(got["summary"][:, S.S_STATUS] == 0)
    for r in range(n):
        rows, hist = oracle_job_rows(oracle, sp, seed0 + r, bin_s, rng_kind)
        assert np.array_equal(got["jens"][..., r], rows), (r, np.argwhere(got["jens"][..., r] != rows)[:5])
        assert np.array_equal(got["jens_hist"][r], hist), r
        assert got["jens"][-1, 0, :, :, r].sum() == got["summary"][r, S.S_JOBS_FINISHED]


@pytest.mark.parametrize("mode", ["one_shot", "chunks61", "uniform", "records_global"])
@pytest.mark.parametrize("name", FIXTURES)
def test_recorder_equals_oracle_job_logs(oracle, monkeypatch, name, mode):
    """Every replica's recorded counts, latency sums (added in finish order) and per-DC histogram equal its own oracle
    job log binned in numpy, bit for bit."""
    sp = SC.to_spec(SC.BY_NAME[name])
    kw = {}
    if mode == "chunks61":
        kw["chunk_events"] = 61
    if mode == "uniform":
        kw["uniform"] = True
    if mode == "records_global":
        monkeypatch.setenv("DCSIM_RECORDS", "global")
        kw["chunk_events"] = 977
    got = H.run_batch(sp.to_bytes(), 3, SEED, jens_bin=sp.log_interval, **kw)
    _check_recorded(oracle, sp, got, SEED, 3, sp.log_interval)


def test_recorder_mersenne_twister(oracle):
    sp = SC.to_spec(SC.BY_NAME["ragged_3dc_12_5_40"])
    got = H.run_batch(sp.to_bytes(), 2, 77, jens_bin=sp.log_interval, rng_kind=1, chunk_events=61)
    _check_recorded(oracle, sp, got, 77, 2, sp.log_interval, rng_kind=1)


def test_recorder_changes_no_summary_and_splits_the_batch_histogram(hostemu):
    sp = SC.to_spec(dict(SC.CFG3, duration=40.0))
    blob = sp.to_bytes()
    off = H.run_batch(blob, 3, 9)
    on = H.run_batch(blob, 3, 9, jens_bin=sp.log_interval)
    assert np.array_equal(off["summary"], hostemu.run_batch(blob, 3, 9)["summary"])    # == the plain host build
    assert np.array_equal(off["summary"], on["summary"])
    assert np.array_equal(off["lat_hist"], on["lat_hist"])
    assert np.array_equal(on["jens_hist"].sum(axis=1), on["lat_hist"])   # per-DC histogram summed over DCs
    assert on["lat_hist"].sum() == on["summary"][:, S.S_JOBS_FINISHED].sum() > 0


@pytest.mark.parametrize("bin_s,windows", [(5.0, 12), (7.0, 9), (500.0, 1), (None, 12)])
def test_window_rule(oracle, bin_s, windows):
    """60 s: a bin that divides end_time, one that does not, one wider than the run (W = 1), the default
    (log_interval = 5 s).  Host build, numpy and the recorder agree; every job is in one window and in the whole run."""
    sp = SC.to_spec(dict(SC.CFG3, duration=60.0))
    b = bin_s or sp.log_interval
    assert H.job_windows(sp.to_bytes(), b) == EN.job_windows(sp.end_time, b) == windows
    got = H.run_batch(sp.to_bytes(), 2, 31, jens_bin=b)
    assert got["jens"].shape[0] == windows + 1
    assert np.array_equal(got["jens"][:-1, 0].sum(axis=0), got["jens"][-1, 0])
    _check_recorded(oracle, sp, got, 31, 2, b)
    t = np.array([0.0, b * 0.5, b, 60.0, 60.0 + 1e-9, np.nextafter(b * windows, 0)])
    k = EN.job_window_index(t, b, windows)
    assert k[0] == 0 and k[3] == k[4] == windows - 1 and np.all(k < windows)
    assert k[2] == min(1, windows - 1)


def _oracle_batch(oracle, sp, n, first, bin_s):
    per = [oracle_job_rows(oracle, sp, first + r, bin_s) for r in range(n)]
    return np.stack([p[0] for p in per], axis=-1), np.stack([p[1] for p in per], axis=-1)


def numpy_job_check(res, rows, status, quantiles=EN.DEFAULT_QUANTILES):
    """A JobEnsembleResult against plain numpy on the rows: jobs exact (unit bins, inverted_cdf), mean_latency_s only
    over the replicas with a job in the cell."""
    good = np.asarray(status) == 0
    jobs, lat = rows[:, 0][..., good], rows[:, 1][..., good]
    J = EN.JOB_FIELDS.index("jobs")
    M = EN.JOB_FIELDS.index("mean_latency_s")
    assert np.all(res.n[:, J] == good.sum())
    assert np.array_equal(res.min[:, J], jobs.min(axis=-1)) and np.array_equal(res.max[:, J], jobs.max(axis=-1))
    np.testing.assert_allclose(res.mean[:, J], jobs.mean(axis=-1), rtol=1e-12)
    np.testing.assert_allclose(res.std[:, J], jobs.std(axis=-1, ddof=1), rtol=1e-12, atol=1e-12)
    span = jobs.max(axis=-1) - jobs.min(axis=-1)
    unit = span + 1 <= EN.BINS                          # unit bins, exact quantiles; else integer width ceil((span + 1) / BINS)
    for j, q in enumerate(quantiles):
        want = np.quantile(jobs, q, axis=-1, method="inverted_cdf")
        assert np.array_equal(res.quantiles[j][:, J][unit], want[unit]), q
        assert np.all(np.abs(res.quantiles[j][:, J][~unit] - want[~unit]) <= np.ceil((span[~unit] + 1) / EN.BINS)), q
    has = jobs > 0
    assert np.array_equal(res.n[:, M], has.sum(axis=-1))
    with np.errstate(invalid="ignore", divide="ignore"):
        per = lat / jobs
    for idx in np.ndindex(res.n[:, M].shape):
        vals = per[idx][has[idx]]
        if vals.size == 0:
            assert np.isnan(res.mean[:, M][idx]) and np.isnan(res.min[:, M][idx])
            continue
        np.testing.assert_allclose(res.mean[:, M][idx], vals.mean(), rtol=1e-12)
        assert res.min[:, M][idx] == vals.min() and res.max[:, M][idx] == vals.max()
        span = vals.max() - vals.min()
        for j, q in enumerate(quantiles):
            assert abs(res.quantiles[j][:, M][idx] - np.quantile(vals, q, method="inverted_cdf")) <= span / EN.BINS * (1 + 1e-12)
    with np.errstate(invalid="ignore", divide="ignore"):
        pooled = lat.sum(axis=-1) / jobs.sum(axis=-1)
    np.testing.assert_allclose(res.pooled_mean_latency_s, pooled, rtol=1e-12)


def test_host_mirror_equals_numpy(oracle):
    sp = SC.to_spec(dict(SC.BY_NAME["ragged_3dc_12_5_40"], duration=60.0))
    rows, hist = _oracle_batch(oracle, sp, 20, 600, 7.0)
    status = np.zeros(rows.shape[-1], dtype=np.int64)
    status[[3, 11]] = S.ST_RUN_OVERFLOW                 # two replicas that stopped: left out everywhere
    res = EN.job_ensemble_from_rows(rows, hist, status, 7.0, sp.end_time)
    assert res.n.shape == (EN.job_windows(sp.end_time, 7.0) + 1, len(EN.JOB_FIELDS), sp.n_dc, 2)
    assert res.t0_s[-1] == 0.0 and res.t1_s[-1] == sp.end_time and res.t0_s[1] == 7.0 and res.t1_s[0] == 7.0
    numpy_job_check(res, rows, status)
    assert np.array_equal(res.latency_histogram, hist[..., status == 0].sum(axis=-1))
    assert np.any(res.n[:-1, 2] < res.n[:-1, 0])       # empty cells are skipped by mean_latency_s


def test_to_csv_long_format(tmp_path, oracle):
    sp = SC.to_spec(dict(SC.CFG3, duration=20.0))
    rows, hist = _oracle_batch(oracle, sp, 5, 40, sp.log_interval)
    res = EN.job_ensemble_from_rows(rows, hist, np.zeros(5), sp.log_interval, sp.end_time)
    p = tmp_path / "jobs.csv"
    names = [f"dc{d}" for d in range(sp.n_dc)]
    res.to_csv(str(p), names)
    lines = p.read_text().splitlines()
    assert lines[0] == "t0_s,t1_s,dc,type,field,n,mean,std,min,p05,p25,p50,p75,p95,max"
    W = EN.job_windows(sp.end_time, sp.log_interval)
    assert len(lines) == 1 + (W + 1) * sp.n_dc * 2 * 2 + sp.n_dc * 2
    first = lines[1].split(",")
    assert first[:6] == ["0.0", "5.0", "dc0", "inference", "jobs", "5"]
    whole = [ln.split(",") for ln in lines[1:] if ln.startswith("0.0,20.0,")]
    lat_rows = [r for r in whole if r[4] == "latency_s"]
    assert len(lat_rows) == sp.n_dc * 2
    r = lat_rows[0]
    assert int(r[5]) == int(hist[0, 0].sum()) and r[7] == r[8] == r[-1] == ""
    assert float(r[6]) == res.pooled_mean_latency_s[-1, 0, 0]


def _gloo_worker(rank, world, port, name, n_total, out_path):
    for p in (ROOT, os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests")):
        if p not in sys.path:
            sys.path.insert(0, p)
    import oracle_lib
    from distributed_cluster_gpus_b200 import sharding
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        sp = SC.to_spec(dict(SC.BY_NAME[name], duration=40.0))
        first, count = sharding.shard(n_total, rank, world)
        rows, hist = _oracle_batch(oracle_lib, sp, count, 700 + first, 6.0)
        res = EN.job_ensemble_from_rows(rows, hist, np.zeros(count), 6.0, sp.end_time)
        if rank == 0:
            np.savez(out_path, n=res.n, mean=res.mean, std=res.std, min=res.min, max=res.max, quantiles=res.quantiles,
                     lat=res.latency_histogram, pooled=res.pooled_mean_latency_s)
    finally:
        dist.destroy_process_group()


def test_two_rank_gloo_matches_one_rank(tmp_path, oracle):
    name, n_total = "cfg3_4x64_sinusoid_120s", 13
    out = str(tmp_path / "jobs.npz")
    mp.spawn(_gloo_worker, args=(2, 29500 + (os.getpid() + 1311) % 2000, name, n_total, out), nprocs=2, join=True)
    got = np.load(out)
    sp = SC.to_spec(dict(SC.BY_NAME[name], duration=40.0))
    rows, hist = _oracle_batch(oracle, sp, n_total, 700, 6.0)
    one = EN.job_ensemble_from_rows(rows, hist, np.zeros(n_total), 6.0, sp.end_time)
    for k in ("n", "min", "max", "quantiles"):
        assert np.array_equal(got[k], getattr(one, k), equal_nan=True), k
    assert np.array_equal(got["lat"], one.latency_histogram)
    np.testing.assert_allclose(got["mean"], one.mean, rtol=1e-12)
    np.testing.assert_allclose(got["pooled"], one.pooled_mean_latency_s, rtol=1e-12)
    np.testing.assert_allclose(got["std"], one.std, rtol=1e-12, atol=1e-12 * np.nanmax(np.abs(one.std)))
