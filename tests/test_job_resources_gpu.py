"""GPUs, frequency and predicted energy of every finished job on the H100: in every staging mode, on 8 and 32 lanes,
one shot and in chunks, the device cells bit for bit against the definition applied to the device's own job records
(its job_log.csv rows of one replica), bit-identical across every kernel, and against the host build (the pre-pass's
transcendental functions round differently on the device, so job sizes and instants may differ in their last bits
there: counts exact, energies to 1e-9); the same against the reference goldens; the device reductions against the numpy
mirror; one rank against two; the capacity retry; the error codes; and sampled replicas of the 65 536-replica bench
batch against the oracle, with the summaries unchanged by the recorder."""
import csv
import json
import math
import os

import numpy as np
import pytest

import hostemu_lib as H
from conftest import has_cuda
from distributed_cluster_gpus_b200 import _native as N, ensemble as EN, scenarios as SC, spec as S
from test_job_resources import GOLDEN_FILES, JRES_GOLDEN, expected, golden_arrays, oracle_job_log
from test_launch_modes_gpu import MODES, force_mode, spec_for

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not has_cuda(), reason="needs a CUDA device")]

SCENARIOS = {"cap_greedy": dict(SC.BY_NAME["cap_greedy_4x64"], duration=30.0),
             "joint_nf": dict(SC.BY_NAME["sweep_joint_nf"], duration=30.0)}
SEED = 77
RTOL = 1e-9
LOGGED = 3
_FIRST = {}
BENCH_N, BENCH_PICK = 65536, list(range(0, 65536, 4096))


def _engine(sp, n, seed=SEED):
    from distributed_cluster_gpus_b200.engine import BatchedEngine
    return BatchedEngine(sp, n, base_seed=seed)


def _stored(eng):
    """(rows, stored mix [n_dc, 2, G * 16 + 1, n], hist) as the recorder holds them."""
    rows, mix, off, hist = eng.job_resources_rows()
    n_dc, n = mix.shape[0], mix.shape[-1]
    return rows, np.concatenate([mix.reshape(n_dc, 2, -1, n), off[:, :, None]], axis=2), hist


def same_bits(a, b):
    return a.shape == b.shape and np.array_equal(np.ascontiguousarray(a).view(np.uint64), np.ascontiguousarray(b).view(np.uint64))


def close_to(rows, mix, hist, w_rows, w_mix, w_hist, what):
    """Counts, GPU and frequency sums exact; energy sums within RTOL (job sizes from another rounding of the pre-pass)."""
    assert np.array_equal(rows[:, :2], w_rows[:, :2]), (what, np.argwhere(rows[:, :2] != w_rows[:, :2])[:5])
    e, w = rows[:, 2], w_rows[:, 2]
    err = np.where(e == w, 0.0, np.abs(e - w) / np.maximum(np.abs(w), 1e-300))
    assert float(err.max(initial=0.0)) <= RTOL, (what, float(err.max()))
    assert np.array_equal(mix, w_mix) and np.array_equal(hist, w_hist), what


@pytest.mark.parametrize("name", sorted(SCENARIOS))
@pytest.mark.parametrize("mode", ["staged", "head", "inplace"])
@pytest.mark.parametrize("lanes", [8, 32])
def test_device_equals_host_build(monkeypatch, lanes, mode, name):
    """The logged replica's cells bit for bit against the definition over its own device job records; every replica's
    cells against the host build of the same source; and every kernel, one shot and in chunks of 61, bit-identical."""
    force_mode(monkeypatch, lanes, mode)
    sp = spec_for(SCENARIOS[name], mode)
    n = 7
    host = H.run_batch(sp.to_bytes(), n, SEED, jens_bin=sp.log_interval, jres=True)
    for chunk in (0, 61):
        with _engine(sp, n) as eng:
            eng.enable_job_ensemble()
            eng.enable_job_resources()
            eng.set_logging(LOGGED, 100000, 0)
            while True:
                eng.advance(chunk)
                if eng.all_done():
                    break
            info = eng.launch_info()
            assert info["lanes_per_replica"] == lanes and info["staging_mode"] == MODES[mode]
            rows, mix, hist = _stored(eng)
            summ = eng.summary()
            log = eng.job_log()
        assert np.all(summ[:, S.S_STATUS] == 0) and len(log) == summ[LOGGED, S.S_JOBS_FINISHED] > 0
        w_rows, w_mix, w_hist, _ = expected(sp, log, sp.log_interval)
        assert same_bits(rows[..., LOGGED], w_rows), (chunk, np.argwhere(rows[..., LOGGED] != w_rows)[:5])
        assert np.array_equal(mix[..., LOGGED], w_mix) and np.array_equal(hist[..., LOGGED], w_hist), chunk
        for r in range(n):
            close_to(rows[..., r], mix[..., r], hist[..., r], host["jres"][..., r], host["jres_mix"][..., r],
                     host["jres_hist"][..., r], (chunk, r))
        assert int(mix[:, :, -1].sum()) == 0
        if name not in _FIRST:
            _FIRST[name] = (rows, mix, hist)
        assert same_bits(rows, _FIRST[name][0]) and np.array_equal(mix, _FIRST[name][1]), (lanes, mode, chunk)
        assert np.array_equal(hist, _FIRST[name][2])


@pytest.mark.parametrize("fname", GOLDEN_FILES)
def test_reference_golden(fname):
    """The cells the unmodified reference gives (tests/golden/make_golden_jres.py), Philox and MT19937: counts exact,
    energies within RTOL."""
    with open(os.path.join(JRES_GOLDEN, fname)) as f:
        doc = json.load(f)
    sp = SC.to_spec(doc["scenario"])
    for case in doc["cases"]:
        with _engine(sp, 1, case["seed"]) as eng:
            if case["rng"] == "mt":
                eng.set_rng("mt19937")
            eng.enable_job_ensemble()
            eng.enable_job_resources()
            eng.advance(0)
            rows, mix, hist = _stored(eng)
        w_rows, w_mix, w_hist = golden_arrays(case)
        close_to(rows[..., 0], mix[..., 0], hist[..., 0], w_rows, w_mix, w_hist, (fname, case["seed"], case["rng"]))


def check_reductions(dev, host):
    ok = dev.n > 0
    assert np.array_equal(dev.n, host.n) and np.any(ok)
    for f in ("min", "max"):
        assert np.array_equal(getattr(dev, f)[ok], getattr(host, f)[ok]), f
    assert np.array_equal(dev.quantiles[:, ok], host.quantiles[:, ok])
    assert np.allclose(dev.mean[ok], host.mean[ok], rtol=4e-16 * 64, atol=0.0, equal_nan=True)
    # the spread sums (x - mean)^2 around a mean that differs in its last bits with the summation order: a column whose
    # values are all equal has a std of rounding noise on one side and 0 on the other
    scale = np.maximum(np.abs(host.mean[ok]), 1.0)
    assert np.all(np.abs(dev.std[ok] - host.std[ok]) <= 1e-9 * np.abs(host.std[ok]) + 1e-12 * scale)
    for f in ("jobs", "mix", "off_level", "energy_histogram"):
        assert np.array_equal(getattr(dev, f), getattr(host, f)), f
    for f in ("gpu_sum", "freq_sum", "energy_sum"):
        assert np.allclose(getattr(dev, f), getattr(host, f), rtol=1e-13, atol=0.0), f


def test_device_reductions_equal_mirror():
    """job_resources (device passes) against job_resources_from_rows (numpy) on the fetched rows, 7 s windows."""
    sp = SC.to_spec(SCENARIOS["joint_nf"])
    with _engine(sp, 203) as eng:
        eng.enable_job_ensemble(7.0)
        eng.enable_job_resources()
        eng.advance(0)
        dev = EN.job_resources(eng)
        rows, mix, off, hist = eng.job_resources_rows()
        jobs = eng.job_ensemble_rows()[0][:, 0]
        status = eng.summary()[:, S.S_STATUS]
    host = EN.job_resources_from_rows(rows, mix, off, hist, jobs, status, EN._res_levels(sp), 7.0, sp.end_time)
    check_reductions(dev, host)


def test_bench_batch():
    """All 65 536 replicas of the bench batch: summaries bit-identical with the recorder on and off, every 4096th
    replica's cells against the oracle's job records, and the reductions against the mirror."""
    sp = SC.to_spec(SC.CFG3)
    with _engine(sp, BENCH_N, 123) as eng:
        eng.enable_job_ensemble()
        eng.advance(0)
        off = eng.summary().copy()
    with _engine(sp, BENCH_N, 123) as eng:
        eng.enable_job_ensemble()
        eng.enable_job_resources()
        eng.advance(0)
        on = eng.summary()
        rows, mix, hist = _stored(eng)
        res = EN.job_resources(eng)
        jobs = eng.job_ensemble_rows()[0]
    assert same_bits(on, off), "summaries differ with the recorder on"
    assert np.all(on[:, S.S_STATUS] == 0)
    for r in BENCH_PICK:
        w_rows, w_mix, w_hist, _ = expected(sp, oracle_job_log(sp, 123 + r), sp.log_interval)
        close_to(rows[..., r], mix[..., r], hist[..., r], w_rows, w_mix, w_hist, r)
    n_dc = sp.n_dc
    G = H.jres_g(sp.to_bytes())
    host = EN.job_resources_from_rows(rows, mix[:, :, :-1].reshape(n_dc, 2, G, 16, BENCH_N), mix[:, :, -1], hist,
                                      jobs[:, 0], on[:, S.S_STATUS], EN._res_levels(sp), sp.log_interval, sp.end_time)
    check_reductions(res, host)
    assert int(res.off_level.sum()) == 0 and res.energy_histogram[..., 0].sum() == 0
    assert res.energy_histogram[..., -1].sum() == 0


def test_capacity_retry_re_enables_the_recorder():
    """run_to_completion(job_resources=True) from too small an arrival buffer: the retry re-enables the recorder, and
    the cells equal a run that needed no retry."""
    from distributed_cluster_gpus_b200 import engine as EG
    sc = dict(SC.CFG3, duration=20.0)
    EG.free_cached_engine()
    tiny = {"cap_arrivals": 64}
    eng, _ = EG.run_to_completion(lambda caps: SC.to_spec(sc, caps=dict(caps) or tiny), 9, SEED, max_retries=10,
                                  job_resources=True)
    try:
        assert eng.job_resources_enabled and eng.spec.cap_arrivals > 64
        got = _stored(eng)
    finally:
        eng.close()
    with _engine(SC.to_spec(sc), 9) as ref:
        ref.enable_job_ensemble()
        ref.enable_job_resources()
        ref.advance(0)
        want = _stored(ref)
    assert same_bits(got[0], want[0]) and np.array_equal(got[1], want[1]) and np.array_equal(got[2], want[2])


def test_error_codes_and_reset():
    """-4 without the job ensemble, after the first advance and on a shared-group member; -3 with the byte count when the
    buffers do not fit; a read before enabling is refused; after reset the same keys give a fresh engine's cells."""
    import torch
    from distributed_cluster_gpus_b200.engine import BatchedEngine
    sp = SC.to_spec(dict(SC.CFG3, duration=20.0))
    with _engine(sp, 16, 7) as eng:
        with pytest.raises(N.DcsimError) as ei:
            eng.enable_job_resources()
        assert ei.value.code == N.E_STATE
        with pytest.raises(RuntimeError):
            eng.job_resources_rows()
        eng.enable_job_ensemble()
        eng.enable_job_resources()
        eng.advance(0)
        first = _stored(eng)
        with pytest.raises(N.DcsimError) as ei:
            eng.enable_job_resources()
        assert ei.value.code == N.E_STATE
        with BatchedEngine.shared(sp, eng) as member:
            member.enable_job_ensemble()
            with pytest.raises(N.DcsimError) as ei:
                member.enable_job_resources()
            assert ei.value.code == N.E_STATE
        eng.reset(7)
        eng.advance(0)
        again = _stored(eng)
    assert same_bits(first[0], again[0]) and np.array_equal(first[1], again[1]) and np.array_equal(first[2], again[2])
    # -3: the windowed rows of a batch with 1 ms windows do not fit next to what is held on the device
    n = 4096
    with _engine(sp, n) as eng:
        eng.enable_job_ensemble(1.0)
        W = eng.job_ensemble_windows
        G = H.jres_g(sp.to_bytes())
        need = (W + 1) * 3 * sp.n_dc * 2 * n * 8 + sp.n_dc * 2 * (G * 16 + 1 + 128) * n * 4
        torch.cuda.synchronize()
        free, _ = torch.cuda.mem_get_info()
        hold = torch.empty(max(free - need // 2, 0), dtype=torch.uint8, device="cuda")
        try:
            with pytest.raises(N.DcsimError) as ei:
                eng.enable_job_resources()
            assert ei.value.code == N.E_NOMEM and str(need) in str(ei.value)
        finally:
            del hold
            torch.cuda.empty_cache()
        eng.enable_job_resources()                     # the handle stays usable
        assert eng.job_resources_enabled


def _read_csv(path):
    with open(path) as f:
        rd = csv.reader(f)
        return next(rd), [r for r in rd]


def test_cli_one_and_two_ranks(tmp_path):
    """run_sim_paper --job-resources-csv / --summary-json on one rank and on two (gloo when the box has one GPU): the
    same rows, counts and quantiles equal, the means to the last bits; no job_resources object without the flag."""
    import torch
    from test_gpu_parity import _run_cli
    common = ["--duration", "20", "--inf-mode", "sinusoid", "--inf-rate", "10", "--inf-period", "3600", "--trn-rate", "1",
              "--n-dc", "4", "--gpus-per-dc", "16", "--replicas", "301", "--seed", "77", "--progress", "",
              "--job-ensemble-bin", "4"]
    one = _run_cli(common + ["--log-path", str(tmp_path / "one" / "x"), "--job-resources-csv", str(tmp_path / "one.csv"),
                             "--summary-json", str(tmp_path / "one.json")])
    assert one.returncode == 0, one.stderr[-2000:]
    extra = {} if torch.cuda.device_count() >= 2 else {"DCSIM_DIST_BACKEND": "gloo"}
    two = _run_cli(common + ["--gpus", "2", "--log-path", str(tmp_path / "two" / "x"), "--job-resources-csv",
                             str(tmp_path / "two.csv"), "--summary-json", str(tmp_path / "two.json")], extra)
    assert two.returncode == 0, two.stderr[-3000:]
    ha, a = _read_csv(tmp_path / "one.csv")
    hb, b = _read_csv(tmp_path / "two.csv")
    assert ha == hb and len(a) == len(b) and len(a) > 0
    for ra, rb in zip(a, b):
        assert ra[:6] == rb[:6], (ra, rb)
        for x, y in zip(ra[6:], rb[6:]):
            if x == y:
                continue
            x, y = float(x), float(y)
            assert abs(x - y) <= 1e-12 * max(abs(x), abs(y)) or (math.isnan(x) and math.isnan(y)), (ra, rb)
    assert sum(1 for r in a if r[4] == "mean_energy_j") == 6 * 4 * 2
    ja, jb = (json.load(open(tmp_path / f)) for f in ("one.json", "two.json"))
    ra_, rb_ = ja["job_resources"], jb["job_resources"]
    assert set(ra_) == set(rb_) and len(ra_) == 4
    for dc in ra_:
        for t in ("inference", "training"):
            assert ra_[dc][t]["jobs"] == rb_[dc][t]["jobs"] and ra_[dc][t]["mix"] == rb_[dc][t]["mix"]
    plain = _run_cli(common + ["--log-path", str(tmp_path / "p" / "x"), "--summary-json", str(tmp_path / "p.json")])
    assert plain.returncode == 0 and "job_resources" not in json.load(open(tmp_path / "p.json"))


def test_simulator_fills_job_resources(tmp_path):
    """MultiIngressPaperSimulator(job_resources=True) fills sim.job_resources with the batch's statistics."""
    from distributed_cluster_gpus_b200 import run_sim_paper as R
    args = R.parse_args(["--duration", "10", "--replicas", "33", "--progress", "", "--log-path", str(tmp_path / "x"),
                         "--job-resources-csv", str(tmp_path / "r.csv")])
    sim = R.build_simulator(args, write_logs=False)
    sim.run()
    res = sim.job_resources
    assert res is not None and int(res.jobs.sum()) == int(sim.summary[:, S.S_JOBS_FINISHED].sum())
