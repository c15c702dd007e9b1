"""Occupancy on the H100: the reference-derived fixtures in 8- and 32-lane builds, the recorder in every profile
instantiation of the event loop against the host build (which tests/test_occupancy.py pins to the reference and the
oracle), the bench batch with the recorder on, the reductions against the numpy
mirror, all profile and wait recorders together, the capacity retry, the opt-in's error codes and the CLI."""
import os

import numpy as np
import pytest

import hostemu_lib as H
from conftest import has_cuda
from distributed_cluster_gpus_b200 import ensemble as E, scenarios as SC, spec as S
from test_launch_modes_gpu import MODES, SCENARIOS as LM_SCENARIOS, force_mode, spec_for
from test_occupancy import REF_DIR, REF_FIXTURES, reference_column

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not has_cuda(), reason="needs a CUDA device")]

RTOL = 1e-9
SEED = 123


def _engine(sp, n, seed=SEED, **kw):
    from distributed_cluster_gpus_b200.engine import BatchedEngine
    return BatchedEngine(sp, n, base_seed=seed, **kw)


def integer_rows(n_dc):
    return [1 + f * n_dc + d for f in (S.OCC_Q_INF_MAX, S.OCC_Q_TRN_MAX) for d in range(n_dc)]


def assert_close(got, want, n_dc, what):
    """The maxima exact, the rest within RTOL relative (exact where one of them is 0)."""
    for i in integer_rows(n_dc):
        assert np.array_equal(got[i], want[i]), (what, i, got[i], want[i])
    rel = np.where(got == want, 0.0, np.abs(got - want) / np.maximum(np.abs(want), 1e-300))
    assert rel.max() <= RTOL, (what, int(np.argmax(rel.max(axis=-1) if rel.ndim > 1 else rel)), float(rel.max()))


def _run(eng, chunk=0):
    total = eng.advance(chunk)
    guard = 0
    while chunk and not eng.all_done():
        total += eng.advance(chunk)
        guard += 1
        assert guard < 100000
    return total


@pytest.mark.parametrize("records", ["shared", "global"])
@pytest.mark.parametrize("group", ["8", "32"])
def test_reference_fixtures_in_every_build(group, records, monkeypatch):
    """The fixtures from the unmodified reference (tests/golden/make_golden_occupancy.py) on the device: maxima exact,
    the rest within RTOL."""
    import json
    monkeypatch.setenv("DCSIM_GROUP", group)
    monkeypatch.setenv("DCSIM_RECORDS", records)
    for name in REF_FIXTURES:
        with open(os.path.join(REF_DIR, name + ".json")) as f:
            doc = json.load(f)
        sp = SC.to_spec(doc["scenario"])
        for case in doc["cases"]:
            with _engine(sp, 1, case["seed"]) as eng:
                if case["rng"] == "mt":
                    eng.set_rng("mt19937")
                eng.enable_occupancy()
                _run(eng, 997 if case["seed"] == 124 else 0)
                got = eng.occupancy_rows()[:, 0]
                lanes = eng.launch_info()["lanes_per_replica"]
                assert int(eng.summary()[0, S.S_EVENTS]) == case["events"]
            assert lanes == int(group)
            assert_close(got, reference_column(doc, case), sp.n_dc, f"{name} {case['rng']} {case['seed']} g{group} {records}")


_FIRST = {}


@pytest.mark.parametrize("cap", [False, True], ids=["nocap", "cap"])
@pytest.mark.parametrize("mode", ["staged", "head", "inplace"])
@pytest.mark.parametrize("lanes", [8, 16, 32])
def test_every_profile_instantiation(monkeypatch, lanes, mode, cap):
    """The 18 profile kernels (lanes x staging x cap controller) with only the occupancy recorder on: the intended
    kernel runs (launch_info), 5 and 7 replicas (ghost lane groups), one shot and in chunks of 61, and all of them
    return bit-identical rows, equal to the host build."""
    force_mode(monkeypatch, lanes, mode)
    sc = LM_SCENARIOS[cap]
    sp = spec_for(sc, mode)
    for n in (5, 7):
        want = H.run_batch(SC.to_spec(sc).to_bytes(), n, 31, occ=True)["occ"]
        for chunk in (0, 61):
            with _engine(sp, n, 31) as eng:
                eng.enable_occupancy()
                _run(eng, chunk)
                rows = eng.occupancy_rows()
                info = eng.launch_info()
                assert np.all(eng.summary()[:, S.S_STATUS] == 0)
            what = (lanes, mode, cap, n, chunk)
            assert info["lanes_per_replica"] == lanes and info["staging_mode"] == MODES[mode], (what, info)
            first = _FIRST.setdefault((cap, n), (what, rows))
            assert np.array_equal(rows.view(np.uint64), first[1].view(np.uint64)), (what, "differs from", first[0])
            assert_close(rows, want, sp.n_dc, str(what))


def check_reductions(res, mirror):
    assert np.array_equal(res.n, mirror.n) and np.array_equal(res.min, mirror.min) and np.array_equal(res.max, mirror.max)
    assert np.array_equal(res.quantiles, mirror.quantiles, equal_nan=True)
    assert np.allclose(res.mean, mirror.mean, rtol=1e-12, atol=0, equal_nan=True)
    assert np.allclose(res.std, mirror.std, rtol=1e-9, atol=1e-12, equal_nan=True)
    for a, b in ((res.queue_bins, mirror.queue_bins), (res.busy_bins, mirror.busy_bins)):
        assert np.allclose(a, b, rtol=1e-12, atol=0)


def test_bench_batch_with_the_recorder_on():
    sp = SC.to_spec(SC.CFG3)
    n = 65536
    with _engine(sp, n) as eng:
        eng.advance(0)
        off = eng.summary().copy()
        info_off = eng.launch_info()
    with _engine(sp, n) as eng:
        eng.enable_occupancy()
        eng.advance(0)
        on = eng.summary()
        rows = eng.occupancy_rows()
        info_on = eng.launch_info()
        widths = eng.occupancy_bin_widths()
        res = E.occupancy(eng)
    assert info_on == info_off
    assert np.array_equal(on.view(np.uint64), off.view(np.uint64)), "summaries differ with the recorder on"
    assert np.all(on[:, S.S_STATUS] == 0)
    assert res.replicas == n and list(widths) == [1] * sp.n_dc
    check_reductions(res, E.occupancy_from_rows(rows, on, widths))
    for r in np.linspace(0, n - 1, 16).astype(np.int64):
        want = H.run_batch(sp.to_bytes(), 1, SEED + int(r), occ=True)["occ"][:, 0]
        assert_close(rows[:, r], want, sp.n_dc, f"replica {r}")


def test_all_recorders_together():
    """Occupancy, power profile and job waits in one batch: each recorder's rows equal that recorder alone."""
    sp = SC.to_spec(dict(SC.BY_NAME["cap_greedy_4x64"], duration=30.0))
    n = 64

    def run(occ, pp, waits):
        with _engine(sp, n) as eng:
            if waits:
                eng.enable_job_ensemble()
                eng.enable_job_waits()
            if pp:
                eng.enable_power_profile(20000.0)
            if occ:
                eng.enable_occupancy()
            eng.advance(0)
            return (eng.occupancy_rows() if occ else None, eng.power_profile_rows() if pp else None,
                    eng.job_waits_rows() if waits else None)

    both = run(True, True, True)
    assert np.array_equal(both[0], run(True, False, False)[0])
    assert np.array_equal(both[1], run(False, True, False)[1])
    alone = run(False, False, True)[2]
    assert np.array_equal(both[2][0], alone[0]) and np.array_equal(both[2][1], alone[1])


def test_capacity_retry_keeps_the_recorder():
    """run_to_completion(occupancy=True) from too small a running set: the retry re-enables the recorder, and the final
    rows equal a run that needed no retry."""
    from distributed_cluster_gpus_b200 import engine as EG
    sc = dict(SC.BY_NAME["ragged_3dc_12_5_40"], duration=30.0)
    EG.free_cached_engine()
    tiny = {"cap_run": 4}
    eng, _ = EG.run_to_completion(lambda caps: SC.to_spec(sc, caps=dict(caps) or tiny), 9, SEED, max_retries=10,
                                  occupancy=True)
    try:
        assert eng.occupancy_enabled and eng.spec.cap_run > 4
        got = eng.occupancy_rows()
    finally:
        eng.close()
    with _engine(SC.to_spec(sc), 9) as ref:
        ref.enable_occupancy()
        ref.advance(0)
        want = ref.occupancy_rows()
    assert np.array_equal(got, want)


def test_enable_error_codes():
    from distributed_cluster_gpus_b200 import _native as N
    from distributed_cluster_gpus_b200.engine import BatchedEngine
    sp = SC.to_spec(dict(SC.CFG3, duration=5.0))
    with _engine(sp, 8, 1) as eng:
        with pytest.raises(N.DcsimError) as ei:
            eng.occupancy_rows()
        assert ei.value.code == N.E_STATE
        eng.enable_occupancy()
        eng.advance(0)
        with pytest.raises(N.DcsimError) as ei:
            eng.enable_occupancy()
        assert ei.value.code == N.E_STATE
        with BatchedEngine.shared(sp, eng) as member:
            with pytest.raises(N.DcsimError) as ei:
                member.enable_occupancy()
            assert ei.value.code == N.E_STATE
        eng.reset(1)
        eng.enable_occupancy()                       # a reset batch is fresh again


def _read_csv(path):
    import csv
    with open(path) as f:
        rd = csv.reader(f)
        return next(rd), [r for r in rd]


def test_cli_occupancy_one_and_two_ranks(tmp_path):
    """run_sim_paper --occupancy-csv / --summary-json on one rank and on two (gloo when the box has one GPU): the same
    CSV within 1e-12."""
    import json
    import torch
    from test_gpu_parity import _run_cli
    common = ["--duration", "20", "--inf-mode", "sinusoid", "--inf-rate", "10", "--inf-period", "3600", "--trn-rate", "1",
              "--n-dc", "4", "--gpus-per-dc", "16", "--replicas", "301", "--seed", "77", "--progress", ""]
    one = _run_cli(common + ["--log-path", str(tmp_path / "one" / "x"), "--occupancy-csv", str(tmp_path / "one.csv"),
                             "--summary-json", str(tmp_path / "one.json")])
    assert one.returncode == 0, one.stderr[-2000:]
    extra = {} if torch.cuda.device_count() >= 2 else {"DCSIM_DIST_BACKEND": "gloo"}
    two = _run_cli(common + ["--gpus", "2", "--log-path", str(tmp_path / "two" / "x"), "--occupancy-csv",
                             str(tmp_path / "two.csv"), "--summary-json", str(tmp_path / "two.json")], extra)
    assert two.returncode == 0, two.stderr[-3000:]
    ha, a = _read_csv(tmp_path / "one.csv")
    hb, b = _read_csv(tmp_path / "two.csv")
    assert ha == hb == E.PP_CSV_HEADER
    assert len(a) == len(b) == 4 * len(E.OCC_STATS) + 4 * 2
    for ra, rb in zip(a, b):
        assert ra[:3] == rb[:3] and ra[3:] and ra[2] == "301"
        for x, y in zip(ra[3:], rb[3:]):
            if x == "":
                assert y == ""
                continue
            x, y = float(x), float(y)
            assert x == y or abs(x - y) <= 1e-12 * max(abs(x), abs(y)) or (np.isnan(x) and np.isnan(y)), (ra, rb)
    ja, jb = (json.load(open(tmp_path / f)) for f in ("one.json", "two.json"))
    assert set(ja["occupancy"]) == set(jb["occupancy"]) and len(ja["occupancy"]) == 4
    for dc in ja["occupancy"]:
        for k, x in ja["occupancy"][dc].items():
            y = jb["occupancy"][dc][k]
            assert x == y or abs(x - y) <= 1e-12 * max(abs(x), abs(y)), (dc, k, x, y)
