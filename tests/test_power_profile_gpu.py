"""Power profile on the H100: the recorder in every kernel instantiation against the reference-derived fixtures, the
bench batch with the recorder on, the reductions against the numpy mirror, the opt-in's error codes and the CLI."""
import os
import subprocess
import sys

import numpy as np
import pytest

import hostemu_lib as H
from conftest import ROOT, has_cuda
from distributed_cluster_gpus_b200 import ensemble as E, scenarios as SC, spec as S
from test_power_profile import FIXTURES, NF, expected_column, load, threshold_of

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not has_cuda(), reason="needs a CUDA device")]

RTOL = 1e-9
INTEGER_ROWS = (S.PP_EXCURSIONS, S.PP_OUT_OF_RANGE)


def _engine(sp, n, seed, **kw):
    from distributed_cluster_gpus_b200.engine import BatchedEngine
    return BatchedEngine(sp, n, base_seed=seed, **kw)


def assert_close(got, want, what):
    """Integer rows exact, the rest within RTOL relative (absolute for values that are 0 in one of them)."""
    for i in INTEGER_ROWS:
        assert np.array_equal(got[i], want[i]), (what, i, got[i], want[i])
    rel = np.where(got == want, 0.0, np.abs(got - want) / np.maximum(np.abs(want), 1e-300))
    assert rel.max() <= RTOL, (what, int(np.argmax(rel.max(axis=-1) if rel.ndim > 1 else rel)), float(rel.max()))


@pytest.mark.parametrize("records", ["shared", "global"])
@pytest.mark.parametrize("group", ["8", "32"])
def test_fixtures_in_every_build(group, records, monkeypatch):
    monkeypatch.setenv("DCSIM_GROUP", group)
    monkeypatch.setenv("DCSIM_RECORDS", records)
    for name in FIXTURES:
        doc = load(name)
        sp = SC.to_spec(doc["scenario"])
        for case in doc["cases"]:
            with _engine(sp, 1, case["seed"]) as eng:
                if case["rng"] == "mt":
                    eng.set_rng("mt19937")
                eng.enable_power_profile(None if threshold_of(doc) == np.inf else threshold_of(doc))
                assert eng.power_profile_range().hex() == doc["hi"]
                eng.advance(997 if case["seed"] == 124 else 0)
                while not eng.all_done():
                    eng.advance(997)
                lanes = eng.launch_info()["lanes_per_replica"]
                got = eng.power_profile_rows()[:, 0]
                assert int(eng.summary()[0, S.S_EVENTS]) == case["events"]
            assert lanes == int(group)
            assert_close(got, expected_column(doc, case), f"{name} {case['rng']} {case['seed']} g{group} {records}")


def test_bench_batch_with_the_recorder_on():
    sp = SC.to_spec(SC.CFG3)
    n = 65536
    with _engine(sp, n, 123) as eng:
        eng.advance(0)
        off = eng.summary().copy()
        info_off = eng.launch_info()
    with _engine(sp, n, 123) as eng:
        eng.enable_power_profile(30000.0)
        eng.advance(0)
        on = eng.summary()
        rows = eng.power_profile_rows()
        info_on = eng.launch_info()
        hi = eng.power_profile_range()
        res = E.power_profile(eng, summary=on)
    for k in ("regs_per_thread", "resident_warps_per_sm", "state_block_bytes", "staged_bytes_per_replica", "lanes_per_replica"):
        assert info_on[k] == info_off[k], k
    assert np.array_equal(on.view(np.uint64), off.view(np.uint64)), "summaries differ with the recorder on"
    assert np.all(on[:, S.S_STATUS] == 0) and np.all(rows[S.PP_OUT_OF_RANGE] == 0)
    n_dc = sp.n_dc
    prof, bins = rows[S.PP_PROFILE_S], rows[NF + n_dc:]
    assert np.allclose(bins.sum(axis=0), prof, rtol=1e-12, atol=0)
    energy = on[:, S.S_TOTAL_ENERGY_J]
    assert np.all(rows[S.PP_PEAK_W] * prof >= energy * (1 - 1e-12))
    width = hi / S.PP_BINS
    lo_e = (bins * (np.arange(S.PP_BINS) * width)[:, None]).sum(axis=0)
    hi_e = (bins * ((np.arange(S.PP_BINS) + 1) * width)[:, None]).sum(axis=0)
    assert np.all(lo_e <= energy * (1 + 1e-12)) and np.all(energy <= hi_e * (1 + 1e-12))
    ids = np.linspace(0, n - 1, 64).astype(np.int64)
    for r in ids:
        want = H.run_batch(sp.to_bytes(), 1, 123 + int(r), pp=True, pp_threshold=30000.0)["pp"][:, 0]
        assert_close(rows[:, r], want, f"replica {r}")
    assert res.replicas == n and res.n[S.PP_PEAK_W] == n
    mirror = E.power_profile_from_rows(rows, on, hi, 30000.0)
    check_reductions(res, mirror)


def check_reductions(res, mirror):
    assert np.array_equal(res.n, mirror.n) and np.array_equal(res.min, mirror.min) and np.array_equal(res.max, mirror.max)
    assert np.array_equal(res.quantiles, mirror.quantiles)
    assert np.allclose(res.mean, mirror.mean, rtol=1e-12, atol=0)
    assert np.allclose(res.std, mirror.std, rtol=1e-9, atol=1e-12)
    assert np.allclose(res.duration_curve[1], mirror.duration_curve[1], rtol=1e-12, atol=0)
    assert res.pooled_energy_j == pytest.approx(mirror.pooled_energy_j, rel=1e-12)


def test_reductions_are_bit_stable_and_skip_failed_replicas():
    sc = dict(SC.BY_NAME["cap_greedy_4x64"], duration=30.0)
    sp = SC.to_spec(sc)
    with _engine(sp, 300, 9) as eng:
        eng.enable_power_profile(20000.0)
        eng.advance(0)
        a = E.power_profile(eng)
        rows, summ = eng.power_profile_rows(), eng.summary()
        eng.reset(9)
        eng.advance(0)
        b = E.power_profile(eng)
        assert np.array_equal(eng.power_profile_rows(), rows)
    for x, y in ((a.mean, b.mean), (a.std, b.std), (a.duration_curve[1], b.duration_curve[1])):
        assert np.array_equal(x, y, equal_nan=True)
    check_reductions(a, E.power_profile_from_rows(rows, summ, a.hi, 20000.0))


def test_enable_error_codes():
    from distributed_cluster_gpus_b200 import _native as N
    from distributed_cluster_gpus_b200.engine import BatchedEngine
    sp = SC.to_spec(dict(SC.CFG3, duration=5.0))
    with _engine(sp, 8, 1) as eng:
        for bad in (float("nan"), -1.0):
            with pytest.raises(N.DcsimError) as ei:
                eng.enable_power_profile(bad)
            assert ei.value.code == N.E_INVALID
        with pytest.raises(N.DcsimError) as ei:
            eng.power_profile_rows()
        assert ei.value.code == N.E_STATE
        eng.enable_power_profile(None)
        eng.advance(0)
        with pytest.raises(N.DcsimError) as ei:
            eng.enable_power_profile(100.0)
        assert ei.value.code == N.E_STATE
        with BatchedEngine.shared(sp, eng) as member:
            with pytest.raises(N.DcsimError) as ei:
                member.enable_power_profile(100.0)
            assert ei.value.code == N.E_STATE
        eng.reset(1)
        eng.enable_power_profile(100.0)              # a reset batch is fresh again


def test_cli_power_profile_csv(tmp_path):
    out = tmp_path / "pp.csv"
    cmd = [sys.executable, "-m", "distributed_cluster_gpus_b200.run_sim_paper", "--algo", "cap_greedy", "--power-cap",
           "20000", "--replicas", "512", "--duration", "30", "--power-profile-csv", str(out),
           "--summary-json", str(tmp_path / "s.json")]
    subprocess.run(cmd, cwd=ROOT, check=True, capture_output=True, text=True)
    lines = out.read_text().splitlines()
    assert lines[0] == ",".join(E.PP_CSV_HEADER)
    rows = [ln.split(",") for ln in lines[1:]]
    over = [r for r in rows if r[1] == "over_s"][0]
    assert over[2] == "512" and float(over[3]) > 0
    assert rows[-1][1] == "power_w_time" and rows[-1][2] == "512"
    import json
    summ = json.loads((tmp_path / "s.json").read_text())
    assert summ["power_profile"]["threshold_w"] == 20000.0 and summ["power_profile"]["replicas"] == 512
