"""Cluster-log ensemble on the CPU: the recorder of the device source (host build, tests/hostemu) against every
replica's oracle cluster log, the library's default tick capacity, the numpy mirror of the two reductions against numpy,
and the two-rank all-reduce (gloo) against one rank."""
import os
import sys

import numpy as np
import pytest
import torch.distributed as dist
import torch.multiprocessing as mp

import hostemu_lib as H
from conftest import ROOT, golden_names
from distributed_cluster_gpus_b200 import ensemble as EN, scenarios as SC, spec as S

FIXTURES = ["cfg3_4x64_sinusoid_120s", "sweep_joint_nf", "cap_greedy_4x64", "ragged_3dc_12_5_40", "carbon_cost_8h_2x16"]
SEED = 4100


def _total_gpus(sp):
    return [sp.dc[d].total_gpus for d in range(sp.n_dc)]


def oracle_fields(oracle, sp, seed, rng_kind=0):
    """[ticks, FIELDS, n_dc] of one replica, derived from its oracle cluster log as write_csv_logs derives the CSV."""
    blob = sp.to_bytes()
    ticks = H.ens_ticks(blob)
    sim = oracle.OracleSim(blob, seed, rng_kind=rng_kind, clog_cap=(ticks + 2) * sp.n_dc)
    sim.advance(0)
    log = sim.cluster_log()
    assert len(log) == ticks * sp.n_dc
    return EN.fields_from_cluster_log(log, _total_gpus(sp)), log["time_s"][::sp.n_dc]


def oracle_rows(oracle, sp, n, first):
    """[ticks, FIELDS, n_dc, n] for replica keys first .. first + n - 1 (the CPU stand-in producer)."""
    return np.stack([oracle_fields(oracle, sp, first + r)[0] for r in range(n)], axis=-1)


def _check_recorded(oracle, sp, got, seed0, n, rng_kind=0):
    ticks = H.ens_ticks(sp.to_bytes())
    ens = got["ens"]
    assert np.all(got["summary"][:, S.S_STATUS] == 0)
    assert np.all(got["summary"][:, S.S_EV_LOG] == ticks)
    assert np.all(np.isnan(ens[ticks:])), "a tick past the replica's count was written"
    for r in range(n):
        want, times = oracle_fields(oracle, sp, seed0 + r, rng_kind)
        assert np.array_equal(ens[:ticks, :, :, r], want), (r, np.argwhere(ens[:ticks, :, :, r] != want)[:5])
        assert np.array_equal(EN.tick_times(sp.log_interval, ticks), times)


@pytest.mark.parametrize("mode", ["one_shot", "chunks61", "uniform", "records_global"])
@pytest.mark.parametrize("name", FIXTURES)
def test_recorder_equals_oracle_cluster_logs(oracle, monkeypatch, name, mode):
    """Every replica's recorded values equal the fields derived from its own oracle cluster log, bit for bit."""
    sp = SC.to_spec(SC.BY_NAME[name])
    blob = sp.to_bytes()
    ticks = H.ens_ticks(blob)
    kw = dict(ens_cap=ticks + 2)
    if mode == "chunks61":
        kw["chunk_events"] = 61
    if mode == "uniform":
        kw["uniform"] = True
    if mode == "records_global":
        monkeypatch.setenv("DCSIM_RECORDS", "global")
        kw["chunk_events"] = 977
    got = H.run_batch(blob, 3, SEED, **kw)
    _check_recorded(oracle, sp, got, SEED, 3)


def test_recorder_mersenne_twister(oracle):
    sp = SC.to_spec(SC.BY_NAME["ragged_3dc_12_5_40"])
    blob = sp.to_bytes()
    got = H.run_batch(blob, 2, 77, ens_cap=H.ens_ticks(blob), rng_kind=1, chunk_events=61)
    _check_recorded(oracle, sp, got, 77, 2, rng_kind=1)


def test_recorder_off_changes_nothing_and_capacity_is_respected(oracle, hostemu):
    sp = SC.to_spec(dict(SC.CFG3, duration=40.0))
    blob = sp.to_bytes()
    plain = H.run_batch(blob, 2, 9, ens_cap=0)
    full = H.run_batch(blob, 2, 9, ens_cap=H.ens_ticks(blob))
    short = H.run_batch(blob, 2, 9, ens_cap=3)
    assert np.array_equal(plain["summary"], hostemu.run_batch(blob, 2, 9)["summary"])    # == the plain host build
    assert np.array_equal(plain["summary"], full["summary"]) and np.array_equal(plain["summary"], short["summary"])
    assert np.array_equal(short["ens"], full["ens"][:3])
    assert short["summary"][0, S.S_EV_LOG] == H.ens_ticks(blob) > 3   # counts on past the capacity


@pytest.mark.parametrize("name", golden_names())
def test_default_tick_capacity_is_every_replicas_log_count(oracle, name):
    sc = SC.BY_NAME[name]
    if sc["duration"] > 300 and sc["n_dc"] >= 4:
        sc = dict(sc, duration=150.0)
    sp = SC.to_spec(sc)
    rows, _ = oracle.run_batch(sp.to_bytes(), 3, 31, 0)
    assert np.all(rows[:, S.S_EV_LOG] == H.ens_ticks(sp.to_bytes()))
    for interval, end in ((0.1, 1.0), (0.3, 0.9), (5.0, 4.0), (600.0, 30000.0)):
        sp2 = SC.to_spec(dict(sc, log_interval=interval, duration=end))
        t, n = interval, 0
        while not t > end:
            n, t = n + 1, t + interval
        assert H.ens_ticks(sp2.to_bytes()) == n


def numpy_reference_check(res, rows, quantiles=EN.DEFAULT_QUANTILES):
    """An EnsembleResult against numpy on the rows themselves (every replica recorded every tick)."""
    T = res.n.shape[0]
    x = rows[:T]
    assert np.all(res.n == rows.shape[-1])
    assert np.array_equal(res.min, x.min(axis=-1)) and np.array_equal(res.max, x.max(axis=-1))
    np.testing.assert_allclose(res.mean, x.mean(axis=-1), rtol=1e-12, atol=1e-300)
    np.testing.assert_allclose(res.std, x.std(axis=-1, ddof=1), rtol=1e-12, atol=1e-9 * np.abs(x).max())
    span = x.max(axis=-1) - x.min(axis=-1)
    unit = span + 1 <= EN.BINS                         # integer fields: unit bins, exact quantiles
    for j, q in enumerate(quantiles):
        want = np.quantile(x, q, axis=-1, method="inverted_cdf")
        got = res.quantiles[j]
        for f in range(len(EN.FIELDS)):
            if f in EN.INTEGER_FIELDS:
                u = unit[:, f]
                assert np.array_equal(got[:, f][u], want[:, f][u]), (q, EN.FIELDS[f])
                wide = np.ceil((span[:, f][~u] + 1) / EN.BINS)
                assert np.all(np.abs(got[:, f][~u] - want[:, f][~u]) <= wide), (q, EN.FIELDS[f])
            else:
                assert np.all(np.abs(got[:, f] - want[:, f]) <= span[:, f] / EN.BINS * (1 + 1e-12)), (q, EN.FIELDS[f])


@pytest.mark.parametrize("name", ["cfg3_4x64_sinusoid_120s", "cap_greedy_4x64"])
def test_host_mirror_equals_numpy(oracle, name):
    sp = SC.to_spec(dict(SC.BY_NAME[name], duration=60.0))
    rows = oracle_rows(oracle, sp, 24, 600)
    nlog = np.full(rows.shape[-1], rows.shape[0])
    res = EN.cluster_ensemble_from_rows(rows, nlog, sp.log_interval)
    assert res.n.shape == rows.shape[:3] and res.fields == EN.FIELDS
    assert np.array_equal(res.time_s, EN.tick_times(sp.log_interval, rows.shape[0]))
    numpy_reference_check(res, rows)


def test_host_mirror_counts_only_recorded_ticks_and_wide_integer_bins():
    rng = np.random.default_rng(5)
    rows = rng.normal(size=(4, len(EN.FIELDS), 2, 9)) * 100
    rows[:, 1] = rng.integers(0, 5000, size=(4, 2, 9))      # an integer field spread over more than BINS values
    nlog = np.array([4, 4, 2, 4, 3, 4, 4, 1, 4])
    res = EN.cluster_ensemble_from_rows(rows, nlog, 5.0)
    for k in range(4):
        keep = nlog > k
        assert np.all(res.n[k] == keep.sum())
        np.testing.assert_allclose(res.mean[k], rows[k][..., keep].mean(axis=-1), rtol=1e-12)
        assert np.array_equal(res.min[k], rows[k][..., keep].min(axis=-1))
    width = np.ceil((res.max[:, 1] - res.min[:, 1] + 1) / EN.BINS)
    want = np.stack([np.quantile(rows[k, 1][..., nlog > k], 0.5, axis=-1, method="inverted_cdf") for k in range(4)])
    assert np.all(np.abs(res.quantiles[2][:, 1] - want) <= width)


def test_to_csv_long_format(tmp_path):
    rng = np.random.default_rng(1)
    rows = rng.integers(0, 9, size=(3, len(EN.FIELDS), 2, 5)).astype(np.float64)
    res = EN.cluster_ensemble_from_rows(rows, np.full(5, 3), 5.0)
    p = tmp_path / "ens.csv"
    res.to_csv(str(p), ["east", "west"])
    lines = p.read_text().splitlines()
    assert lines[0] == "time_s,dc,field,n,mean,std,min,p05,p25,p50,p75,p95,max"
    assert len(lines) == 1 + 3 * 2 * len(EN.FIELDS)
    first = lines[1].split(",")
    assert first[:4] == ["5.0", "east", "freq", "5"] and float(first[-1]) == rows[0, 0, 0].max()


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
        rows = oracle_rows(oracle_lib, sp, count, 700 + first)
        res = EN.cluster_ensemble_from_rows(rows, np.full(count, rows.shape[0]), sp.log_interval)
        if rank == 0:
            np.savez(out_path, n=res.n, mean=res.mean, std=res.std, min=res.min, max=res.max, quantiles=res.quantiles)
    finally:
        dist.destroy_process_group()


def test_two_rank_gloo_matches_one_rank(tmp_path, oracle):
    name, n_total = "cfg3_4x64_sinusoid_120s", 13
    out = str(tmp_path / "ens.npz")
    mp.spawn(_gloo_worker, args=(2, 29500 + (os.getpid() + 977) % 2000, name, n_total, out), nprocs=2, join=True)
    got = np.load(out)
    sp = SC.to_spec(dict(SC.BY_NAME[name], duration=40.0))
    rows = oracle_rows(oracle, sp, n_total, 700)
    one = EN.cluster_ensemble_from_rows(rows, np.full(n_total, rows.shape[0]), sp.log_interval)
    assert np.array_equal(got["n"], one.n) and np.array_equal(got["min"], one.min) and np.array_equal(got["max"], one.max)
    for f in EN.INTEGER_FIELDS:
        assert np.array_equal(got["quantiles"][:, :, f], one.quantiles[:, :, f])
    np.testing.assert_allclose(got["quantiles"], one.quantiles, rtol=0, atol=0)   # same histograms -> same readout
    np.testing.assert_allclose(got["mean"], one.mean, rtol=1e-12)
    np.testing.assert_allclose(got["std"], one.std, rtol=1e-12, atol=1e-12 * np.nanmax(np.abs(one.std)))
