"""Waiting and response times on the H100: the recorder in every staging mode on 8 and 32 lanes against the oracle's
per-job instants, the device reductions against the numpy mirror, the C-ABI's refusals, and the full bench batch with the
recorder on against the recorder off."""
import numpy as np
import pytest

import hostemu_jwait_lib as HW
from conftest import has_cuda
from distributed_cluster_gpus_b200 import _native as N, ensemble as EN, scenarios as SC, spec as S
from test_job_waits import expected_rows
from test_launch_modes_gpu import MODES, force_mode, spec_for

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not has_cuda(), reason="needs a CUDA device")]

SCENARIOS = {"ragged": dict(SC.BY_NAME["ragged_3dc_12_5_40"], duration=60.0),
             "cap_greedy": dict(SC.BY_NAME["cap_greedy_4x64"], duration=30.0)}
SEED = 77
_FIRST = {}
_ORACLE = {}


def _engine(sp, n, seed=SEED):
    from distributed_cluster_gpus_b200.engine import BatchedEngine
    return BatchedEngine(sp, n, base_seed=seed)


def _oracle(name, n):
    if (name, n) not in _ORACLE:
        sp = SC.to_spec(SCENARIOS[name])
        _ORACLE[(name, n)] = [expected_rows(HW.oracle_jobs(sp.to_bytes(), SEED + r), sp.n_dc, sp.log_interval,
                                            sp.end_time) for r in range(n)]
    return _ORACLE[(name, n)]


def assert_close(got, want, rel=1e-9):
    err = np.where(got == want, 0.0, np.abs(got - want) / np.maximum(np.abs(want), 1e-300))
    assert float(err.max(initial=0.0)) <= rel, float(err.max())


@pytest.mark.parametrize("name", sorted(SCENARIOS))
@pytest.mark.parametrize("mode", ["staged", "head", "inplace"])
@pytest.mark.parametrize("lanes", [8, 32])
def test_recorder_matches_oracle(monkeypatch, lanes, mode, name):
    """Counts exact and sums within 1e-9 of the oracle's per-job instants, every kernel's rows bit-identical."""
    force_mode(monkeypatch, lanes, mode)
    sp = spec_for(SCENARIOS[name], mode)
    for n in (5, 7):
        want = _oracle(name, n)
        for chunk in (0, 61):
            with _engine(sp, n) as eng:
                eng.enable_job_ensemble()
                eng.enable_job_waits()
                while True:
                    eng.advance(chunk)
                    if eng.all_done():
                        break
                info = eng.launch_info()
                assert info["lanes_per_replica"] == lanes and info["staging_mode"] == MODES[mode]
                rows, hist = eng.job_waits_rows()
                summ = eng.summary()
            assert np.all(summ[:, S.S_STATUS] == 0)
            for r in range(n):
                w_rows, w_hist = want[r]
                assert np.array_equal(rows[:, 0, ..., r], w_rows[:, 0]), r
                assert_close(rows[:, 1:, ..., r], w_rows[:, 1:])
                assert np.array_equal(hist[..., r], w_hist), r
            key = (name, n)
            if key not in _FIRST:
                _FIRST[key] = (rows, hist)
            assert np.array_equal(rows, _FIRST[key][0]) and np.array_equal(hist, _FIRST[key][1])


def test_device_reductions_equal_mirror():
    """job_waits (device passes) against job_waits_from_rows (numpy) on the fetched rows: n, min, max and quantiles
    exact, mean and std to their last bits."""
    sp = SC.to_spec(SCENARIOS["ragged"])
    with _engine(sp, 203) as eng:
        eng.enable_job_ensemble(7.0)
        eng.enable_job_waits()
        eng.advance(0)
        dev = EN.job_waits(eng)
        rows, hist = eng.job_waits_rows()
        jobs = eng.job_ensemble_rows()[0][:, 0]
        status = eng.summary()[:, S.S_STATUS]
    host = EN.job_waits_from_rows(rows, hist, jobs, status, 7.0, sp.end_time)
    ok = dev.n > 0
    assert np.array_equal(dev.n, host.n) and np.any(ok)
    for f in ("min", "max"):
        assert np.array_equal(getattr(dev, f)[ok], getattr(host, f)[ok]), f
    assert np.array_equal(dev.quantiles[:, ok], host.quantiles[:, ok])
    for f in ("mean", "std"):
        a, b = getattr(dev, f)[ok], getattr(host, f)[ok]
        assert np.allclose(a, b, rtol=4e-16 * 64, atol=0.0, equal_nan=True), f
    assert np.array_equal(dev.wait_histogram, host.wait_histogram)
    assert np.array_equal(dev.jobs, host.jobs) and np.array_equal(dev.waited, host.waited)


def test_refusals():
    sp = SC.to_spec(SCENARIOS["ragged"])
    with _engine(sp, 4) as eng:
        with pytest.raises(N.DcsimError) as e:
            eng.enable_job_waits()                              # no job ensemble
        assert e.value.code == N.E_STATE
        eng.enable_job_ensemble()
        eng.advance(0)
        with pytest.raises(N.DcsimError) as e:
            eng.enable_job_waits()                              # after an advance
        assert e.value.code == N.E_STATE
        from distributed_cluster_gpus_b200.engine import BatchedEngine
        with BatchedEngine.shared(sp, eng) as member:
            member.enable_job_ensemble()
            with pytest.raises(N.DcsimError) as e:
                member.enable_job_waits()                       # on a member of a shared group
            assert e.value.code == N.E_STATE


def test_nomem_reports_the_bytes():
    """The job ensemble fits, the waits' 1.5x larger rows beside it do not: DCSIM_E_NOMEM with the byte count, and the
    handle stays usable.  A genuine failure of the second allocation needs the first to hold a large share of the card
    (45 % of what is free, for the moment between the two calls); if other work on the card moves the free memory in
    between so that either premise does not hold, the case is skipped rather than failed."""
    import torch
    sp = SC.to_spec(SCENARIOS["ragged"])
    n = 4096
    row = 2 * sp.n_dc * 2 * n * 8                               # one window of the job ensemble
    with _engine(sp, n) as eng:
        windows = int(0.45 * torch.cuda.mem_get_info()[0] / row)
        try:
            eng.enable_job_ensemble(sp.end_time / windows)
        except N.DcsimError as e:
            if e.code != N.E_NOMEM:
                raise
            pytest.skip("the card's free memory shrank before the job ensemble was allocated")
        try:
            eng.enable_job_waits()
            ok = True
        except N.DcsimError as e:
            assert e.code == N.E_NOMEM and "bytes" in str(e), e
            ok = False
        eng.enable_job_ensemble()                               # back to a small ensemble (frees the large one)
        if ok:
            pytest.skip("the card's free memory grew between the two allocations")
        eng.enable_job_waits()                                  # usable again
        eng.advance(0)
        assert np.all(eng.summary()[:, S.S_STATUS] == 0)


def _read_csv(path):
    import csv
    with open(path) as f:
        rd = csv.reader(f)
        return next(rd), [r for r in rd]


def test_cli_job_waits_one_and_two_ranks(tmp_path):
    """The CLI end to end (run_sim_paper --job-waits-csv / --summary-json, through the drop-in's job_waits=True), on one
    rank and on two (gloo when the box has one GPU): n, min, max and the quantiles equal."""
    import json
    import torch
    from test_gpu_parity import _run_cli
    common = ["--duration", "20", "--inf-mode", "sinusoid", "--inf-rate", "10", "--inf-period", "3600", "--trn-rate", "1",
              "--n-dc", "4", "--gpus-per-dc", "16", "--replicas", "301", "--seed", "77", "--progress", "",
              "--job-ensemble-bin", "3"]
    one = _run_cli(common + ["--log-path", str(tmp_path / "one" / "x"), "--job-waits-csv", str(tmp_path / "one.csv"),
                             "--summary-json", str(tmp_path / "one.json")])
    assert one.returncode == 0, one.stderr[-2000:]
    extra = {} if torch.cuda.device_count() >= 2 else {"DCSIM_DIST_BACKEND": "gloo"}
    two = _run_cli(common + ["--gpus", "2", "--log-path", str(tmp_path / "two" / "x"), "--job-waits-csv",
                             str(tmp_path / "two.csv"), "--summary-json", str(tmp_path / "two.json")], extra)
    assert two.returncode == 0, two.stderr[-3000:]
    ha, a = _read_csv(tmp_path / "one.csv")
    hb, b = _read_csv(tmp_path / "two.csv")
    assert ha == hb == ["t0_s", "t1_s", "dc", "type", "field", "n", "mean", "std", "min", "p05", "p25", "p50", "p75", "p95",
                        "max"]
    assert len(a) == len(b) == (7 + 1) * 4 * 2 * 3 + 4 * 2 * 3   # 7 windows + the whole run, 4 DCs; 3 whole-run rows
    waited = 0
    for ra, rb in zip(a, b):
        assert ra[:6] == rb[:6]
        if ra[4] in ("waited", "mean_wait_s", "mean_response_s"):
            assert ra[8:] == rb[8:] if ra[4] == "waited" else (ra[8] == rb[8] and ra[14] == rb[14])
        if ra[4] in ("wait_s", "response_s"):
            assert ra[9:] == rb[9:]                                 # same histograms -> same readout
        if ra[4] == "waited_share":
            waited += ra[6] not in ("0.0", "nan")
        for i in (6, 7):
            if ra[i] == "":
                assert rb[i] == ""
                continue
            x, y = float(ra[i]), float(rb[i])
            assert x == y or abs(x - y) <= 1e-12 * max(abs(x), abs(y)) or (np.isnan(x) and np.isnan(y)), (ra, rb)
    assert waited > 0, "the scenario is supposed to queue jobs"
    ja, jb = (json.load(open(tmp_path / f)) for f in ("one.json", "two.json"))
    assert ja["job_waits"]["inference"]["jobs"] > 0     # (training jobs outlast these 20 s: none finishes)
    for jt in ("inference", "training"):
        wa, wb = ja["job_waits"][jt], jb["job_waits"][jt]
        assert wa["jobs"] == wb["jobs"]
        for k in wa:
            same = wa[k] == wb[k] or (np.isnan(wa[k]) and np.isnan(wb[k]))
            if k.startswith("mean") and not same:
                same = abs(wa[k] - wb[k]) <= 1e-12 * abs(wa[k])
            assert same, (jt, k, wa[k], wb[k])


def test_capacity_retry_keeps_the_recorder():
    """run_to_completion from too small a FIFO: the retry re-enables the recorder, and the final rows equal a run that
    needed no retry."""
    from distributed_cluster_gpus_b200 import engine as E
    sc = SCENARIOS["ragged"]
    E.free_cached_engine()
    tiny = {"cap_q_inf": 16, "cap_q_trn": 16}
    eng, _ = E.run_to_completion(lambda caps: SC.to_spec(sc, caps=dict(caps) or tiny), 9, SEED, max_retries=10,
                                 job_waits=True)
    try:
        assert eng.job_waits_enabled and eng.spec.cap_q_inf > 1
        got = eng.job_waits_rows()
    finally:
        eng.close()
    with _engine(SC.to_spec(sc), 9) as ref:
        ref.enable_job_ensemble()
        ref.enable_job_waits()
        ref.advance(0)
        want = ref.job_waits_rows()
    assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1])


def test_bench_batch_summaries_unchanged():
    """The full bench batch (65 536 replicas): every summary row with the recorder on is bit-identical to a run with
    it off (the records then carry the job id: another layout, another launch geometry)."""
    sp = SC.to_spec(SC.BY_NAME["cfg3_4x64_sinusoid_120s"])
    n = 65536
    with _engine(sp, n, 123) as eng:
        eng.advance(0)
        off = eng.summary().copy()
    with _engine(sp, n, 123) as eng:
        eng.enable_job_ensemble()
        eng.enable_job_waits()
        eng.advance(0)
        on = eng.summary()
        res = EN.job_waits(eng)
    assert np.all(off[:, S.S_STATUS] == 0)
    assert np.array_equal(on, off)
    p = res.pooled()
    assert p["inference"]["jobs"] == int(off[:, S.S_FIN_INF].sum())
    print({k: {f: round(v, 4) if isinstance(v, float) else v for f, v in e.items()} for k, e in p.items()})
