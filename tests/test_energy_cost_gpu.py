"""Energy cost and carbon on the H100: the recorder in every profile kernel (lane width x staging mode x CAP) against the
host build, the reference-derived fixtures on every lane width, the bench batch with the recorder on, the device
reductions against the numpy mirror (failed replicas included), the opt-in's error codes and the CLI on one and two
ranks.  Floats within 1e-9 relative of the host build: the tail's power goes through pow() when alpha != 3, and
libdevice's pow may differ from glibc's in the last bit."""
import csv
import json

import numpy as np
import pytest

import hostemu_cost_lib as H
import test_recorder_corpus as RC
from conftest import has_cuda
from distributed_cluster_gpus_b200 import ensemble as E, scenarios as SC, spec as S
from test_energy_cost import FIXTURES, expected_column, load
from test_launch_modes_gpu import MODES, SCENARIOS, force_mode, spec_for

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not has_cuda(), reason="needs a CUDA device")]

RTOL = 1e-9
LANES = (8, 16, 32)


def _engine(sp, n, seed, **kw):
    from distributed_cluster_gpus_b200.engine import BatchedEngine
    return BatchedEngine(sp, n, base_seed=seed, **kw)


def assert_close(got, want, what, rtol=RTOL):
    got, want = np.asarray(got, dtype=np.float64), np.asarray(want, dtype=np.float64)
    rel = np.where(got == want, 0.0, np.abs(got - want) / np.maximum(np.abs(want), 1e-300))
    assert rel.max(initial=0.0) <= rtol, (what, np.unravel_index(int(np.argmax(rel)), rel.shape), float(rel.max()))


def run_device(sp, n, seed, chunk=0, rng=None):
    with _engine(sp, n, seed) as eng:
        if rng == "mt":
            eng.set_rng("mt19937")
        eng.enable_energy_cost()
        eng.advance(chunk)
        while not eng.all_done():
            eng.advance(chunk)
        return eng.energy_cost_rows(), eng.summary(), eng.launch_info()


@pytest.mark.parametrize("cap", [False, True], ids=["plain", "cap"])
@pytest.mark.parametrize("mode", sorted(MODES))
@pytest.mark.parametrize("lanes", LANES)
def test_every_profile_kernel_equals_the_host_build(lanes, mode, cap, monkeypatch):
    force_mode(monkeypatch, lanes, mode)
    sc = SCENARIOS[cap]
    sp = spec_for(sc, mode)
    n, seed, chunk = 5, 31, 61 if lanes == 16 else 0
    rows, summ, info = run_device(sp, n, seed, chunk)
    assert (info["lanes_per_replica"], info["staging_mode"]) == (lanes, MODES[mode]), info
    monkeypatch.delenv("DCSIM_RECORDS", raising=False)
    host = H.run_batch(sp.to_bytes(), n, seed, cost=True)
    assert np.array_equal(summ[:, S.S_EVENTS], host["summary"][:, S.S_EVENTS])
    assert_close(rows, host["cost"], (lanes, mode, cap))


@pytest.mark.parametrize("lanes", LANES)
def test_reference_fixtures_on_every_lane_width(lanes, monkeypatch):
    force_mode(monkeypatch, lanes, "staged")
    for name in FIXTURES:
        doc = load(name)
        sp = SC.to_spec(doc["scenario"])
        for case in doc["cases"]:
            rows, summ, info = run_device(sp, 1, case["seed"], 997 if case["seed"] == 124 else 0, case["rng"])
            assert info["lanes_per_replica"] == lanes
            assert int(summ[0, S.S_EVENTS]) == case["events"], (name, case["seed"], case["rng"])
            assert_close(rows[:, 0], expected_column(doc, case), (name, case["seed"], case["rng"], lanes))


def check_reductions(res, mirror):
    assert np.array_equal(res.n, mirror.n) and np.array_equal(res.min, mirror.min) and np.array_equal(res.max, mirror.max)
    assert np.array_equal(res.quantiles, mirror.quantiles, equal_nan=True)
    assert np.allclose(res.mean, mirror.mean, rtol=1e-12, atol=0, equal_nan=True)
    assert np.allclose(res.std, mirror.std, rtol=1e-9, atol=1e-12, equal_nan=True)
    assert np.allclose(res.sum, mirror.sum, rtol=1e-12, atol=0)


def test_bench_batch_with_the_recorder_on():
    """65 536 replicas of the bench workload: summaries bit-identical to the recorder off, the launch unchanged, 64
    replicas' columns equal to the host build, ENERGY_J within 1e-10 of the summary's energy, and the device
    reductions equal to the numpy mirror over the fetched rows."""
    sp = SC.to_spec(SC.CFG3)
    n, n_dc = 65536, sp.n_dc
    with _engine(sp, n, 123) as eng:
        eng.advance(0)
        off = eng.summary().copy()
        info_off = eng.launch_info()
    with _engine(sp, n, 123) as eng:
        eng.enable_energy_cost()
        eng.advance(0)
        on = eng.summary()
        rows = eng.energy_cost_rows()
        info_on = eng.launch_info()
        res = E.energy_cost(eng)
    for k in ("regs_per_thread", "resident_warps_per_sm", "state_block_bytes", "staged_bytes_per_replica", "lanes_per_replica"):
        assert info_on[k] == info_off[k], k
    assert np.array_equal(on.view(np.uint64), off.view(np.uint64)), "summaries differ with the recorder on"
    assert np.all(on[:, S.S_STATUS] == 0)
    for d in range(n_dc):
        want = on[:, S.S_DC0 + d * S.S_DC_STRIDE + S.SD_ENERGY_J]
        assert_close(rows[S.cost_energy_j(n_dc, d)], want, ("energy", d), rtol=1e-10)
    for r in np.linspace(0, n - 1, 64).astype(np.int64):
        want = H.run_batch(sp.to_bytes(), 1, 123 + int(r), cost=True)["cost"][:, 0]
        assert_close(rows[:, r], want, f"replica {r}")
    assert res.replicas == n
    check_reductions(res, E.energy_cost_from_rows(rows, on[:, S.S_STATUS], *E._cost_tables(sp)))


def test_reductions_skip_failed_replicas(monkeypatch):
    """Replicas that overflow cap_run count in no column; the rest equal the host build and the mirror."""
    caps, need = RC.status_caps()
    sp = SC.to_spec(RC.STATUS_SC, caps=caps)
    n = RC.STATUS_REP
    bad = need > caps["cap_run"]
    with _engine(sp, n, 0) as eng:
        eng.enable_energy_cost()
        eng.advance(0)
        summ, rows = eng.summary(), eng.energy_cost_rows()
        res = E.energy_cost(eng)
    st = summ[:, S.S_STATUS].astype(np.int64)
    assert np.array_equal(st != 0, bad) and bad.any() and (~bad).any()
    host = H.run_batch(sp.to_bytes(), n, 0, cost=True)
    assert_close(rows[:, ~bad], host["cost"][:, ~bad], "valid replicas")
    assert np.all(res.n == int((~bad).sum()))
    check_reductions(res, E.energy_cost_from_rows(rows, summ[:, S.S_STATUS], *E._cost_tables(sp)))


def test_enable_error_codes():
    import torch
    from distributed_cluster_gpus_b200 import _native as N
    from distributed_cluster_gpus_b200.engine import BatchedEngine
    sp = SC.to_spec(dict(SC.CFG3, duration=5.0))
    with _engine(sp, 8, 1) as eng:
        with pytest.raises(N.DcsimError) as ei:
            eng.energy_cost_rows()                       # not enabled
        assert ei.value.code == N.E_STATE
        eng.enable_energy_cost()
        with pytest.raises(N.DcsimError) as ei:
            eng.energy_cost_rows()                       # before the first advance
        assert ei.value.code == N.E_STATE
        eng.advance(0)
        first = eng.energy_cost_rows()
        with pytest.raises(N.DcsimError) as ei:
            eng.enable_energy_cost()
        assert ei.value.code == N.E_STATE
        with BatchedEngine.shared(sp, eng) as member:
            with pytest.raises(N.DcsimError) as ei:
                member.enable_energy_cost()
            assert ei.value.code == N.E_STATE
        eng.reset(1)                                     # stays on across reset, zeroed by it
        eng.advance(0)
        assert np.array_equal(eng.energy_cost_rows(), first)
        eng.reset(1)
        eng.enable_energy_cost()                         # a reset batch is fresh again
    n = 65536
    need = S.cost_bytes_per_replica(sp.n_dc) * n
    with _engine(sp, n, 1) as eng:
        torch.cuda.synchronize()
        free, _ = torch.cuda.mem_get_info()
        hold = torch.empty(max(free - need // 2, 0), dtype=torch.uint8, device="cuda")
        try:
            with pytest.raises(N.DcsimError) as ei:
                eng.enable_energy_cost()
            assert ei.value.code == N.E_NOMEM and str(need) in str(ei.value)
        finally:
            del hold
            torch.cuda.empty_cache()
        eng.enable_energy_cost()                         # the handle stays usable
        assert eng.energy_cost_enabled


def _read_csv(path):
    with open(path) as f:
        rd = csv.reader(f)
        return next(rd), list(rd)


def test_cli_energy_cost_one_and_two_ranks(tmp_path):
    """run_sim_paper --energy-cost-csv / --summary-json on one rank and on two (gloo when the box has one GPU): the same
    CSV within 1e-12, the summary's energy_cost object only with the flag."""
    import torch
    from test_gpu_parity import _run_cli
    common = ["--algo", "carbon_cost", "--duration", "20", "--n-dc", "4", "--gpus-per-dc", "16", "--replicas", "301",
              "--seed", "77", "--progress", ""]
    one = _run_cli(common + ["--log-path", str(tmp_path / "one" / "x"), "--energy-cost-csv", str(tmp_path / "one.csv"),
                             "--summary-json", str(tmp_path / "one.json")])
    assert one.returncode == 0, one.stderr[-2000:]
    extra = {} if torch.cuda.device_count() >= 2 else {"DCSIM_DIST_BACKEND": "gloo"}
    two = _run_cli(common + ["--gpus", "2", "--log-path", str(tmp_path / "two" / "x"), "--energy-cost-csv",
                             str(tmp_path / "two.csv"), "--summary-json", str(tmp_path / "two.json")], extra)
    assert two.returncode == 0, two.stderr[-3000:]
    none = _run_cli(common + ["--log-path", str(tmp_path / "none" / "x"), "--summary-json", str(tmp_path / "none.json")])
    assert none.returncode == 0, none.stderr[-2000:]
    ha, a = _read_csv(tmp_path / "one.csv")
    hb, b = _read_csv(tmp_path / "two.csv")
    assert ha == hb == E.COST_CSV_HEADER
    assert len(a) == len(b) == 4 * 27 + 3
    for ra, rb in zip(a, b):
        assert ra[:4] == rb[:4] and (ra[0] == "" or ra[3] == "301")
        for x, y in zip(ra[4:], rb[4:]):
            x, y = float(x), float(y)
            assert x == y or abs(x - y) <= 1e-12 * max(abs(x), abs(y)), (ra, rb)
    ja, jb, jn = (json.load(open(tmp_path / f)) for f in ("one.json", "two.json", "none.json"))
    assert "energy_cost" not in jn
    for j in (ja, jb):
        c = j["energy_cost"]
        assert c["replicas"] == 301 and len(c["dc"]) == 4
        assert c["cluster"]["cost_usd"] > 0 and c["cluster"]["usd_per_kwh"] == pytest.approx(0.12, rel=1e-9)
    assert ja["energy_cost"]["cluster"]["carbon_g"] == pytest.approx(jb["energy_cost"]["cluster"]["carbon_g"], rel=1e-12)
