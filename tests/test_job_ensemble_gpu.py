"""Job-log ensemble on the H100: the recorder in every kernel instantiation against the oracle's job logs, the
reductions against the numpy mirror, the opt-in's error codes and engine cache, and the CLI at one and two ranks."""
import csv

import numpy as np
import pytest

from conftest import has_cuda
from distributed_cluster_gpus_b200 import ensemble as EN, scenarios as SC, spec as S

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not has_cuda(), reason="needs a CUDA device")]

RTOL = 1e-9


def _engine(sp, n, seed, **kw):
    from distributed_cluster_gpus_b200.engine import BatchedEngine
    return BatchedEngine(sp, n, base_seed=seed, **kw)


def _oracle_rows(sp, seed, bin_s):
    import oracle_lib
    sim = oracle_lib.OracleSim(sp.to_bytes(), seed, joblog_cap=1 << 18)
    sim.advance(0)
    log = sim.job_log()
    assert len(log) == int(sim.summary()[S.S_JOBS_FINISHED])
    sim.close()
    return EN.rows_from_job_log(log, sp.n_dc, bin_s, sp.end_time)


def assert_close_to_oracle(rows, hist, sp, seed0, replica_ids, bin_s):
    """rows[..., i] / hist[..., i] are replica replica_ids[i] (Philox key seed0 + id)."""
    for i, r in enumerate(replica_ids):
        want, want_h = _oracle_rows(sp, seed0 + int(r), bin_s)
        got = rows[..., i]
        assert got.shape == want.shape, (r, got.shape, want.shape)
        assert np.array_equal(got[:, 0], want[:, 0]), (r, np.argwhere(got[:, 0] != want[:, 0])[:5])
        assert np.array_equal(hist[..., i], want_h), r
        g, w = got[:, 1], want[:, 1]
        rel = np.where(g == w, 0.0, np.abs(g - w) / np.maximum(np.abs(w), 1e-300))
        assert rel.max() <= RTOL, (r, float(rel.max()))


@pytest.mark.parametrize("name,n", [("cfg3_4x64_sinusoid_120s", 41), ("cfg5_8x256_sinusoid_60s", 16), ("cap_greedy_4x64", 16)])
def test_recorded_rows_match_oracle_one_shot_and_chunked(name, n):
    """cfg3: 8 lanes per replica, 41 replicas leave a ragged last warp; cfg5: 32 lanes; cap_greedy: the <CAP> build.
    One shot equals chunked advance(997) bit for bit."""
    sp = SC.to_spec(SC.BY_NAME[name])
    with _engine(sp, n, 300) as eng:
        eng.enable_job_ensemble()
        eng.advance(0)
        one, one_h = eng.job_ensemble_rows()
        lanes = eng.launch_info()["lanes_per_replica"]
        eng.reset(300)
        while not eng.all_done():
            eng.advance(997)
        chunked, chunked_h = eng.job_ensemble_rows()
        summ = eng.summary()
    assert lanes == (8 if name == "cfg3_4x64_sinusoid_120s" else 32)
    assert np.array_equal(one, chunked) and np.array_equal(one_h, chunked_h)
    assert np.array_equal(one[-1, 0].sum(axis=(0, 1)), summ[:, S.S_JOBS_FINISHED])
    assert_close_to_oracle(one, one_h, sp, 300, range(n), sp.log_interval)


def test_logged_replica_rows_equal_its_job_log():
    sp = SC.to_spec(SC.BY_NAME["ragged_3dc_12_5_40"])
    with _engine(sp, 9, 55) as eng:
        eng.enable_job_ensemble(7.0)
        eng.set_logging(6, 1 << 16, 0)
        eng.advance(0)
        rows, hist = eng.job_ensemble_rows()
        log = eng.job_log()
    want, want_h = EN.rows_from_job_log(log, sp.n_dc, 7.0, sp.end_time)
    assert np.array_equal(rows[..., 6], want) and np.array_equal(hist[..., 6], want_h)


@pytest.mark.parametrize("name", ["cfg3_4x64_sinusoid_120s", "cfg5_8x256_sinusoid_60s", "cap_greedy_4x64"])
def test_recorder_leaves_summaries_bit_identical(name):
    sp = SC.to_spec(SC.BY_NAME[name])
    with _engine(sp, 64, 91) as eng:
        eng.enable_latency_histogram()
        eng.advance(0)
        off = eng.summary()
        lat_off = eng.latency_histogram()
    with _engine(sp, 64, 91) as eng:
        eng.enable_latency_histogram()
        eng.enable_job_ensemble()
        eng.advance(0)
        on = eng.summary()
        per_dc = eng.dc_latency_histogram()
    assert np.array_equal(off, on)
    assert np.array_equal(per_dc.sum(axis=0), lat_off)


def test_reductions_match_numpy_mirror_and_are_bit_stable():
    from test_job_ensemble import numpy_job_check
    sp = SC.to_spec(SC.BY_NAME["cfg3_4x64_sinusoid_120s"])
    with _engine(sp, 3001, 17) as eng:
        eng.enable_job_ensemble(7.0)
        eng.advance(0)
        rows, hist = eng.job_ensemble_rows()
        status = eng.summary()[:, S.S_STATUS]
        first = EN.job_ensemble(eng)
        eng.reset(17)
        eng.advance(0)
        second = EN.job_ensemble(eng)
    keys = ("n", "mean", "std", "min", "max", "quantiles", "pooled_mean_latency_s", "latency_histogram", "t0_s", "t1_s")
    for k in keys:
        assert np.array_equal(getattr(first, k), getattr(second, k), equal_nan=True), k
    host = EN.job_ensemble_from_rows(rows, hist, status, 7.0, sp.end_time)
    for k in ("n", "min", "max", "quantiles", "latency_histogram"):
        assert np.array_equal(getattr(first, k), getattr(host, k), equal_nan=True), k
    np.testing.assert_allclose(first.mean, host.mean, rtol=1e-12)
    numpy_job_check(first, rows, status)


def test_enable_errors_and_windows():
    from distributed_cluster_gpus_b200 import _native as N
    sp = SC.to_spec(dict(SC.CFG3, duration=30.0))
    with _engine(sp, 8, 5) as eng:
        for bad in (-1.0, float("nan"), float("inf")):
            with pytest.raises(N.DcsimError) as e:
                eng.enable_job_ensemble(bad)
            assert e.value.code == N.E_INVALID
        eng.enable_job_ensemble()
        assert eng.job_ensemble_windows == 6 and eng.job_ensemble_bin == sp.log_interval
        eng.advance(0)
        with pytest.raises(N.DcsimError) as e:
            eng.enable_job_ensemble(4.0)
        assert e.value.code == N.E_STATE
        eng.enable_job_ensemble(sp.log_interval)          # the same opt-in again: fine
    with _engine(sp, 8, 5) as eng:
        with pytest.raises(N.DcsimError) as e:
            eng.enable_job_ensemble(1e-300)               # more windows than memory
        assert e.value.code == N.E_NOMEM and "bytes" in str(e.value)


def test_failed_retarget_leaves_the_ensemble_off():
    """A re-target that does not fit frees the old ensemble (and the waits recorder in its windows) before it fails: the
    engine then reports the ensemble off, and the engine cache keys it so, instead of the old windows."""
    from distributed_cluster_gpus_b200 import _native as N
    from distributed_cluster_gpus_b200.engine import _engine_recorders
    sp = SC.to_spec(dict(SC.CFG3, duration=60.0))
    with _engine(sp, 8, 5) as eng:
        eng.enable_job_ensemble()
        eng.enable_job_waits()
        assert eng.job_ensemble_windows == 12 and eng.job_waits_enabled
        with pytest.raises(N.DcsimError) as e:
            eng.enable_job_ensemble(1e-12)                # 2^32 - 1 windows: refused before any allocation
        assert e.value.code == N.E_NOMEM
        assert eng.job_ensemble_windows == 0 and eng.job_ensemble_bin is None and not eng.job_waits_enabled
        kw = _engine_recorders(eng)
        assert not kw["job_ensemble"] and kw["job_ensemble_bin"] is None and not kw["job_waits"]
        with pytest.raises(RuntimeError, match="job ensemble not enabled"):
            eng.job_ensemble_rows()
        eng.enable_job_ensemble()                         # the handle stays usable
        assert eng.job_ensemble_windows == 12 and eng.job_ensemble_bin == sp.log_interval


def test_bench_size_sample_matches_oracle():
    sp = SC.to_spec(SC.BY_NAME["cfg3_4x64_sinusoid_120s"])
    n = 65536
    sample = np.sort(np.random.default_rng(2024).choice(n, 256, replace=False))
    with _engine(sp, n, 123) as eng:
        eng.enable_job_ensemble()
        eng.advance(0)
        assert np.all(eng.summary()[:, S.S_STATUS] == 0)
        rows, hist = eng.job_ensemble_rows()
    assert_close_to_oracle(rows[..., sample], hist[..., sample], sp, 123, sample, sp.log_interval)


def _read_csv(path):
    with open(path) as f:
        rd = csv.reader(f)
        return next(rd), [r for r in rd]


def test_cli_job_ensemble_csv_one_and_two_ranks(tmp_path):
    import torch
    from test_gpu_parity import _run_cli
    common = ["--duration", "20", "--inf-mode", "sinusoid", "--inf-rate", "10", "--inf-period", "3600", "--trn-rate", "1",
              "--n-dc", "4", "--gpus-per-dc", "64", "--replicas", "301", "--seed", "77", "--progress", "",
              "--job-ensemble-bin", "3"]
    one = _run_cli(common + ["--log-path", str(tmp_path / "one" / "x"), "--job-ensemble-csv", str(tmp_path / "one.csv")])
    assert one.returncode == 0, one.stderr[-2000:]
    extra = {} if torch.cuda.device_count() >= 2 else {"DCSIM_DIST_BACKEND": "gloo"}
    two = _run_cli(common + ["--gpus", "2", "--log-path", str(tmp_path / "two" / "x"), "--job-ensemble-csv",
                             str(tmp_path / "two.csv")], extra)
    assert two.returncode == 0, two.stderr[-3000:]
    ha, a = _read_csv(tmp_path / "one.csv")
    hb, b = _read_csv(tmp_path / "two.csv")
    assert ha == hb == ["t0_s", "t1_s", "dc", "type", "field", "n", "mean", "std", "min", "p05", "p25", "p50", "p75", "p95",
                        "max"]
    assert len(a) == len(b) == (7 + 1) * 4 * 2 * 2 + 4 * 2   # 7 windows of 3 s in 20 s + the whole run, 4 DCs
    for ra, rb in zip(a, b):
        assert ra[:6] == rb[:6]
        if ra[4] == "jobs":
            assert ra[5] == "301" and ra[8:] == rb[8:]                              # min, quantiles, max: exact
        if ra[4] == "mean_latency_s":
            assert ra[8] == rb[8] and ra[14] == rb[14]                              # min, max
        if ra[4] == "latency_s":
            assert ra[9:] == rb[9:]                                                 # same histogram -> same readout
        for i in (6, 7):
            if ra[i] == "":
                assert rb[i] == ""
                continue
            x, y = float(ra[i]), float(rb[i])
            assert x == y or abs(x - y) <= 1e-12 * max(abs(x), abs(y)) or (np.isnan(x) and np.isnan(y)), (ra, rb)


def test_drop_in_result_and_engine_cache_key_on_the_bin(tmp_path):
    """MultiIngressPaperSimulator(job_ensemble=True) fills sim.job_ensemble; a parked engine is only reused by a run that
    asks for the same bin; a capacity retry keeps the recorder on."""
    import logging
    from distributed_cluster_gpus_b200 import engine as E
    from distributed_cluster_gpus_b200.configs import paper_config as pc
    from distributed_cluster_gpus_b200.simcore.simulator_paper_multi import MultiIngressPaperSimulator
    sc = dict(SC.CFG3, duration=30.0)

    def run(**kw):
        sim = MultiIngressPaperSimulator(router_policy=pc.build_router_policy(), logger=logging.getLogger("t"),
                                         sim_duration=sc["duration"], log_interval=sc["log_interval"],
                                         log_path=str(tmp_path), rng_seed=8, algo=sc["algo"], show_progress=False,
                                         replicas=37, **kw, **SC.build_inputs(sc))
        sim.run()
        return sim, E._CACHED["engine"]

    E.free_cached_engine()
    try:
        a, eng_a = run(job_ensemble=True)
        assert eng_a.job_ensemble_windows == 6 and a.job_ensemble.n.shape == (7, len(EN.JOB_FIELDS), 4, 2)
        assert np.all(a.job_ensemble.n[:, 0] == 37)
        b, eng_b = run(job_ensemble=True, job_ensemble_bin=7.0)
        assert eng_b is not eng_a and eng_b.job_ensemble_windows == 5 and b.job_ensemble.n.shape[0] == 6
        c, eng_c = run(job_ensemble=False)
        assert c.job_ensemble is None and eng_c is not eng_b and eng_c.job_ensemble_windows == 0
        d, eng_d = run(job_ensemble=True, job_ensemble_bin=5.0)   # = the default bin of run a
        for k in ("n", "min", "max", "quantiles", "mean", "std", "latency_histogram"):
            assert np.array_equal(getattr(a.job_ensemble, k), getattr(d.job_ensemble, k), equal_nan=True), k
        E.free_cached_engine()
        attempts = []

        def factory(caps):   # the first attempt overflows the running set and is re-run with it raised
            attempts.append(dict(caps))
            return SC.to_spec(sc, caps=caps if caps else {"cap_run": 4})
        eng, _summ = E.run_to_completion(factory, 37, 8, job_ensemble=True)
        try:
            assert len(attempts) == 2 and eng.job_ensemble_windows == 6
            res = EN.job_ensemble(eng)
        finally:
            eng.close()
        for k in ("n", "min", "max", "quantiles", "latency_histogram"):
            assert np.array_equal(getattr(res, k), getattr(a.job_ensemble, k), equal_nan=True), k
    finally:
        E.free_cached_engine()
