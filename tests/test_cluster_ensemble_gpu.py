"""Cluster-log ensemble on the H100: the recorder in every kernel instantiation against the oracle's cluster logs, the
two reduction kernels against numpy, the overflow rule, and the CLI at one and two ranks."""
import csv

import numpy as np
import pytest

from conftest import has_cuda
from distributed_cluster_gpus_b200 import ensemble as EN, scenarios as SC, spec as S

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not has_cuda(), reason="needs a CUDA device")]

RTOL = 1e-9
INT = list(EN.INTEGER_FIELDS)
FLT = [f for f in range(len(EN.FIELDS)) if f not in EN.INTEGER_FIELDS]


def _engine(sp, n, seed, **kw):
    from distributed_cluster_gpus_b200.engine import BatchedEngine
    return BatchedEngine(sp, n, base_seed=seed, **kw)


def _oracle_fields(sp, seed):
    import oracle_lib
    sim = oracle_lib.OracleSim(sp.to_bytes(), seed, clog_cap=(int(sp.end_time / sp.log_interval) + 4) * sp.n_dc)
    sim.advance(0)
    log = sim.cluster_log()
    sim.close()
    return EN.fields_from_cluster_log(log, [sp.dc[d].total_gpus for d in range(sp.n_dc)])


def assert_close_to_oracle(rows, sp, seed0, replica_ids):
    """rows[..., i] is replica replica_ids[i] (Philox key seed0 + id)."""
    for i, r in enumerate(replica_ids):
        want = _oracle_fields(sp, seed0 + int(r))
        got = rows[:, :, :, i]
        assert got.shape == want.shape, (r, got.shape, want.shape)
        assert np.array_equal(got[:, INT], want[:, INT]), (r, np.argwhere(got[:, INT] != want[:, INT])[:5])
        g, w = got[:, FLT], want[:, FLT]
        rel = np.where(g == w, 0.0, np.abs(g - w) / np.maximum(np.abs(w), 1e-300))
        assert rel.max() <= RTOL, (r, float(rel.max()))


@pytest.mark.parametrize("name,n", [("cfg3_4x64_sinusoid_120s", 41), ("cfg5_8x256_sinusoid_60s", 16), ("cap_greedy_4x64", 16)])
def test_recorded_rows_match_oracle_one_shot_and_chunked(name, n):
    """cfg3: 8 lanes per replica, 41 replicas leave the last warp with one replica and three ghost lane groups; cfg5:
    32 lanes; cap_greedy: the <CAP> build (32 lanes: its pools make the head too large for four per warp).  One shot
    equals chunked advance(997) bit for bit."""
    sp = SC.to_spec(SC.BY_NAME[name])
    with _engine(sp, n, 300) as eng:
        eng.enable_cluster_ensemble()
        eng.advance(0)
        one = eng.cluster_ensemble_rows()
        lanes = eng.launch_info()["lanes_per_replica"]
        eng.reset(300)
        while not eng.all_done():
            eng.advance(997)
        chunked = eng.cluster_ensemble_rows()
    assert lanes == (8 if name == "cfg3_4x64_sinusoid_120s" else 32)
    assert np.array_equal(one, chunked, equal_nan=True)
    assert not np.any(np.isnan(one))
    assert_close_to_oracle(one, sp, 300, range(n))


def test_logged_replica_rows_equal_its_cluster_log():
    sp = SC.to_spec(SC.BY_NAME["ragged_3dc_12_5_40"])
    with _engine(sp, 9, 55) as eng:
        eng.enable_cluster_ensemble()
        eng.set_logging(6, 0, 4000)
        eng.advance(0)
        rows = eng.cluster_ensemble_rows()
        log = eng.cluster_log()
    want = EN.fields_from_cluster_log(log, [sp.dc[d].total_gpus for d in range(sp.n_dc)])
    assert np.array_equal(rows[:, :, :, 6], want)


@pytest.mark.parametrize("name", ["cfg3_4x64_sinusoid_120s", "cfg5_8x256_sinusoid_60s", "cap_greedy_4x64"])
def test_recorder_leaves_summaries_bit_identical(name):
    sp = SC.to_spec(SC.BY_NAME[name])
    with _engine(sp, 64, 91) as eng:
        eng.advance(0)
        off = eng.summary()
    with _engine(sp, 64, 91) as eng:
        eng.enable_cluster_ensemble()
        eng.advance(0)
        on = eng.summary()
    assert np.array_equal(off, on)


def test_reductions_match_numpy_and_are_bit_stable():
    from test_cluster_ensemble import numpy_reference_check
    sp = SC.to_spec(SC.BY_NAME["cfg3_4x64_sinusoid_120s"])
    with _engine(sp, 3001, 17) as eng:
        eng.enable_cluster_ensemble()
        eng.advance(0)
        rows = eng.cluster_ensemble_rows()
        first = EN.cluster_ensemble(eng)
        eng.reset(17)
        eng.advance(0)
        second = EN.cluster_ensemble(eng)
    numpy_reference_check(first, rows)
    for k in ("n", "mean", "std", "min", "max", "quantiles", "time_s"):
        assert np.array_equal(getattr(first, k), getattr(second, k), equal_nan=True), k
    host = EN.cluster_ensemble_from_rows(rows, np.full(rows.shape[-1], rows.shape[0]), sp.log_interval)
    for k in ("n", "min", "max", "quantiles"):
        assert np.array_equal(getattr(first, k), getattr(host, k)), k


def test_capacity_below_the_need_raises():
    from distributed_cluster_gpus_b200.engine import RecorderOverflow
    sp = SC.to_spec(dict(SC.CFG3, duration=30.0))
    with _engine(sp, 8, 5) as eng:
        eng.enable_cluster_ensemble(max_ticks=3)
        eng.advance(0)
        with pytest.raises(RecorderOverflow) as e:
            eng.cluster_ensemble_rows()
        assert e.value.needed == 6 and e.value.capacity == 3
        with pytest.raises(RecorderOverflow):
            EN.cluster_ensemble(eng)


def test_bench_size_sample_matches_oracle():
    sp = SC.to_spec(SC.BY_NAME["cfg3_4x64_sinusoid_120s"])
    n = 65536
    sample = np.sort(np.random.default_rng(2024).choice(n, 256, replace=False))
    with _engine(sp, n, 123) as eng:
        eng.enable_cluster_ensemble()
        eng.advance(0)
        assert np.all(eng.summary()[:, S.S_STATUS] == 0)
        rows = eng.cluster_ensemble_rows()[..., sample]
    assert_close_to_oracle(rows, sp, 123, sample)


def _read_ensemble_csv(path):
    with open(path) as f:
        rd = csv.reader(f)
        head = next(rd)
        return head, [r for r in rd]


def test_cli_ensemble_csv_one_and_two_ranks(tmp_path):
    import torch
    from test_gpu_parity import _run_cli
    common = ["--duration", "20", "--inf-mode", "sinusoid", "--inf-rate", "10", "--inf-period", "3600", "--trn-rate", "1",
              "--n-dc", "4", "--gpus-per-dc", "64", "--replicas", "301", "--seed", "77", "--progress", ""]
    one = _run_cli(common + ["--log-path", str(tmp_path / "one" / "x"), "--ensemble-csv", str(tmp_path / "one.csv")])
    assert one.returncode == 0, one.stderr[-2000:]
    extra = {} if torch.cuda.device_count() >= 2 else {"DCSIM_DIST_BACKEND": "gloo"}
    two = _run_cli(common + ["--gpus", "2", "--log-path", str(tmp_path / "two" / "x"), "--ensemble-csv", str(tmp_path / "two.csv")],
                   extra)
    assert two.returncode == 0, two.stderr[-3000:]
    ha, a = _read_ensemble_csv(tmp_path / "one.csv")
    hb, b = _read_ensemble_csv(tmp_path / "two.csv")
    assert ha == hb == ["time_s", "dc", "field", "n", "mean", "std", "min", "p05", "p25", "p50", "p75", "p95", "max"]
    assert len(a) == len(b) == 4 * 4 * len(EN.FIELDS)   # 4 ticks in 20 s at 5 s, 4 DCs
    for ra, rb in zip(a, b):
        assert ra[:4] == rb[:4] and ra[3] == "301"
        assert ra[6] == rb[6] and ra[12] == rb[12]                                   # min, max
        if EN.FIELDS.index(ra[2]) in EN.INTEGER_FIELDS:
            assert ra[7:12] == rb[7:12]                                              # quantiles
        for i in (4, 5):
            x, y = float(ra[i]), float(rb[i])
            assert x == y or abs(x - y) <= 1e-12 * max(abs(x), abs(y)), (ra, rb)


def test_drop_in_result_and_engine_cache_keep_the_opt_in_apart(tmp_path):
    """MultiIngressPaperSimulator(cluster_ensemble=True) fills sim.cluster_ensemble; the parked engine of a run with the
    recorder is not handed to a run without it, nor the reverse; a capacity retry keeps the recorder on."""
    import logging
    from distributed_cluster_gpus_b200 import engine as E
    from distributed_cluster_gpus_b200.configs import paper_config as pc
    from distributed_cluster_gpus_b200.simcore.simulator_paper_multi import MultiIngressPaperSimulator
    sc = dict(SC.CFG3, duration=30.0)

    def run(ens):
        sim = MultiIngressPaperSimulator(router_policy=pc.build_router_policy(), logger=logging.getLogger("t"),
                                         sim_duration=sc["duration"], log_interval=sc["log_interval"],
                                         log_path=str(tmp_path), rng_seed=8, algo=sc["algo"], show_progress=False,
                                         replicas=37, cluster_ensemble=ens, **SC.build_inputs(sc))
        sim.run()
        return sim, E._CACHED["engine"]

    E.free_cached_engine()
    try:
        a, eng_a = run(True)
        assert eng_a.cluster_ensemble_capacity == 6 and a.cluster_ensemble.n.shape == (6, len(EN.FIELDS), 4)
        assert np.all(a.cluster_ensemble.n == 37)
        b, eng_b = run(False)
        assert b.cluster_ensemble is None and eng_b is not eng_a and eng_b.cluster_ensemble_capacity == 0
        c, eng_c = run(True)
        assert eng_c is not eng_b and eng_c.cluster_ensemble_capacity == 6
        for k in ("n", "min", "max", "quantiles", "mean", "std"):
            assert np.array_equal(getattr(a.cluster_ensemble, k), getattr(c.cluster_ensemble, k), equal_nan=True), k
        E.free_cached_engine()
        attempts = []

        def factory(caps):   # the first attempt overflows the running set and is re-run with it raised
            attempts.append(dict(caps))
            return SC.to_spec(sc, caps=caps if caps else {"cap_run": 4})
        eng, _summ = E.run_to_completion(factory, 37, 8, cluster_ensemble=True)
        try:
            assert len(attempts) == 2 and eng.cluster_ensemble_capacity == 6
            res = EN.cluster_ensemble(eng)
        finally:
            eng.close()
        for k in ("n", "min", "max", "quantiles"):
            assert np.array_equal(getattr(res, k), getattr(a.cluster_ensemble, k), equal_nan=True), k
    finally:
        E.free_cached_engine()
