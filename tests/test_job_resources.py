"""GPUs, frequency and predicted energy of every finished job, on the CPU: the recorder of the device source (host
build, tests/hostemu_ens/hostemu_jres.cpp) against every replica's job records from the C oracle and against the
reference goldens (tests/golden/make_golden_jres.py), the off switch, the numpy mirror, and the CLI flag."""
import json
import math
import os
import sys

import numpy as np
import pytest

import hostemu_jres_lib as HJ
from conftest import GOLDEN_DIR
from distributed_cluster_gpus_b200 import ensemble as EN, scenarios as SC, spec as S

sys.path.insert(0, os.path.join(os.path.dirname(GOLDEN_DIR), "..", "oracle"))
import oracle_lib as OL  # noqa: E402

SEED = 5200
N_REP = 3
FIXTURES = ["sweep_default_perf_first", "sweep_joint_nf", "sweep_carbon_cost", "sweep_debug_n2", "sweep_bandit",
            "cap_greedy_4x64", "cfg3_4x64_sinusoid_120s", "ragged_3dc_12_5_40", "all_off_2x8", "underloaded_1x64"]
JRES_GOLDEN = os.path.join(GOLDEN_DIR, "jres")
GOLDEN_FILES = sorted(f for f in os.listdir(JRES_GOLDEN) if f.endswith(".json"))
RNG = {"philox": 0, "mt": 1}


def e_job(sp, d, jt, g, f, size):
    """E_pred * size with E_pred = task_power_w(g, f) * step_time_s(g, f) (energy_paper.py:9-12, latency_paper.py:4-9),
    in the oracle's order."""
    k = sp.dc[d].coeffs[jt]
    fp = f if f > 0.0 else 0.0
    p = max(g, 0) * (k.alpha_p * fp ** 3 + k.beta_p * fp + k.gamma_p)
    n, ft = max(g, 1), (f if f > 1e-9 else 1e-9)
    t = k.alpha_t + k.beta_t / ft if n == 1 else (k.alpha_t + k.beta_t / ft + k.gamma_t * n) / n
    return p * t * size


def ebin_exact(e):
    """clamp(floor(4 * log2(e)), 0, 127) by exact rational comparison (independent of the recorder's significand test)."""
    from fractions import Fraction
    if not e >= 1.0:
        return 0
    x, b = Fraction(e) ** 4, 0
    while b < 127 and x >= 2 ** (b + 1):
        b += 1
    return b


def expected(sp, jobs, bin_s):
    """One replica's oracle job log (finish order) -> (rows [W + 1, 3, n_dc, 2], mix [n_dc, 2, G * 16 + 1],
    hist [n_dc, 2, 128], E_job values); each sum a plain sequential f64 sum in finish order."""
    W = EN.job_windows(sp.end_time, bin_s)
    G = HJ.mix_g(sp.max_gpus_per_job)
    rows = np.zeros((W + 1, 3, sp.n_dc, 2))
    mix = np.zeros((sp.n_dc, 2, G * 16 + 1), dtype=np.uint32)
    hist = np.zeros((sp.n_dc, 2, 128), dtype=np.uint32)
    es = []
    for j in jobs:
        d, jt, g, f = int(j["dc"]), int(j["jtype"]), int(j["n_gpus"]), float(j["f_used"])
        e = e_job(sp, d, jt, g, f, float(j["size"]))
        es.append(e)
        k = int(EN.job_window_index(float(j["finish_s"]), bin_s, W))
        for row in (k, W):
            rows[row, 0, d, jt] += float(g)
            rows[row, 1, d, jt] += f
            rows[row, 2, d, jt] += e
        lv = [q for q in range(sp.dc[d].n_freq) if sp.dc[d].freq_levels[q] == f]
        mix[d, jt, (min(g, G) - 1) * 16 + lv[0] if lv else G * 16] += 1
        hist[d, jt, ebin_exact(e)] += 1
    return rows, mix, hist, es


def oracle_job_log(sp, seed, rng_kind=0):
    o = OL.OracleSim(sp.to_bytes(), seed, rng_kind=rng_kind, joblog_cap=400000)
    o.advance(0)
    s, log = o.summary(), o.job_log()
    o.close()
    assert len(log) == s[S.S_JOBS_FINISHED]
    return log


def check(sp, got, seed0, n, bin_s, rng_kind=0):
    """Every stored cell of every replica bit for bit; returns every E_job and the whole-run off-level count."""
    assert np.all(got["summary"][:, S.S_STATUS] == 0)
    es = []
    for r in range(n):
        rows, mix, hist, e = expected(sp, oracle_job_log(sp, seed0 + r, rng_kind), bin_s)
        assert np.array_equal(got["rows"][..., r].view(np.uint64), rows.view(np.uint64)), \
            (r, np.argwhere(got["rows"][..., r] != rows)[:5])
        assert np.array_equal(got["mix"][..., r], mix), r
        assert np.array_equal(got["hist"][..., r], hist), r
        # the counts agree with the job ensemble's: every finished job once in the mix and once in the histogram
        assert np.array_equal(got["mix"][..., r].sum(axis=-1), got["jens"][-1, 0, ..., r])
        assert np.array_equal(got["hist"][..., r].sum(axis=-1), got["jens"][-1, 0, ..., r])
        es += e
    return es


@pytest.mark.parametrize("mode", ["one_shot", "chunks61", "uniform", "uniform_chunks61"])
@pytest.mark.parametrize("name", FIXTURES)
def test_recorder_equals_oracle_jobs(name, mode):
    """Every GPU_SUM / FREQ_SUM / ENERGY_SUM cell, mix count and energy-bin count equals what the oracle's job records
    give in finish order, bit for bit; plain and warp-uniform loop, one shot and in chunks.  No job's frequency misses
    its DC's levels (OFF_LEVEL stays 0) and no E_job is clamped into an end bin."""
    sp = SC.to_spec(SC.BY_NAME[name])
    kw = {"chunk_events": 61 if "chunks" in mode else 0, "uniform": mode.startswith("uniform")}
    got = HJ.run_batch(sp.to_bytes(), N_REP, SEED, sp.log_interval, sp.max_gpus_per_job, **kw)
    es = check(sp, got, SEED, N_REP, sp.log_interval)
    assert int(got["mix"][:, :, -1].sum()) == 0, "OFF_LEVEL"
    if name == "all_off_2x8":
        assert not es and not got["rows"].any()
        return
    assert 1.0 <= min(es) and ebin_exact(max(es)) < 127, (min(es), max(es))


def test_recorder_mt19937():
    """MT19937 replicas (the stock reference's own random stream) on the cap_greedy cluster."""
    sp = SC.to_spec(SC.BY_NAME["cap_greedy_4x64"])
    got = HJ.run_batch(sp.to_bytes(), 2, SEED, sp.log_interval, sp.max_gpus_per_job, chunk_events=61, rng_kind=1)
    check(sp, got, SEED, 2, sp.log_interval, rng_kind=1)


def test_recorder_head_staged_records(monkeypatch):
    """The head-staged host mode (the running records used where they live), with a window width that is not
    log_interval."""
    monkeypatch.setenv("DCSIM_RECORDS", "global")
    sp = SC.to_spec(SC.BY_NAME["cap_greedy_4x64"])
    got = HJ.run_batch(sp.to_bytes(), 2, SEED, 7.0, sp.max_gpus_per_job, chunk_events=977)
    check(sp, got, SEED, 2, 7.0)


def test_mix_tells_the_policies_apart():
    """The (n, f) mix shows how each policy chose: bandit explores more than one level, joint_nf's static winner and
    default_policy's thresholds give different mixes on the same arrivals."""
    seen = {}
    for name in ("sweep_joint_nf", "sweep_bandit", "sweep_default_perf_first"):
        sp = SC.to_spec(SC.BY_NAME[name])
        got = HJ.run_batch(sp.to_bytes(), N_REP, SEED, sp.log_interval, sp.max_gpus_per_job)
        m = got["mix"][:, :, :-1].sum(axis=(0, 1, 3)).reshape(HJ.mix_g(sp.max_gpus_per_job), 16)
        seen[name] = (np.count_nonzero(m.sum(axis=1)), np.count_nonzero(m.sum(axis=0)))
    assert seen["sweep_bandit"][1] > 1 and seen["sweep_joint_nf"] != seen["sweep_default_perf_first"], seen


@pytest.mark.parametrize("name", ["cap_greedy_4x64", "sweep_bandit", "ragged_3dc_12_5_40"])
def test_summaries_unchanged_by_the_recorder(name):
    """With the recorder on (the records then carry size / f / jid) every summary row, and the job ensemble, are
    bit-identical to the recorder off."""
    sp = SC.to_spec(SC.BY_NAME[name])
    on = HJ.run_batch(sp.to_bytes(), N_REP, SEED, sp.log_interval, sp.max_gpus_per_job, chunk_events=61)
    off = HJ.run_batch(sp.to_bytes(), N_REP, SEED, sp.log_interval, sp.max_gpus_per_job, chunk_events=61,
                       resources=False)
    assert np.array_equal(on["summary"], off["summary"]) and on["events"] == off["events"]
    assert np.array_equal(on["jens"], off["jens"]) and np.array_equal(on["jens_hist"], off["jens_hist"])


def golden_arrays(case):
    rows = np.array([[[[float.fromhex(v) for v in c] for c in f] for f in r] for r in case["rows"]])
    return rows, np.array(case["mix"], dtype=np.uint32), np.array(case["hist"], dtype=np.uint32)


@pytest.mark.parametrize("fname", GOLDEN_FILES)
def test_golden_from_reference(fname):
    """The host build's cells equal those tests/golden/make_golden_jres.py derived from the unmodified reference's own
    g, f_used, E_pred and size, bit for bit (Philox seeds and MT19937 runs)."""
    with open(os.path.join(JRES_GOLDEN, fname)) as f:
        doc = json.load(f)
    sp = SC.to_spec(doc["scenario"])
    for case in doc["cases"]:
        got = HJ.run_batch(sp.to_bytes(), 1, case["seed"], sp.log_interval, sp.max_gpus_per_job,
                           rng_kind=RNG[case["rng"]])
        rows, mix, hist = golden_arrays(case)
        assert got["summary"][0, S.S_JOBS_FINISHED] == case["jobs_finished"]
        assert np.array_equal(got["rows"][..., 0].view(np.uint64), rows.view(np.uint64)), (fname, case["seed"])
        assert np.array_equal(got["mix"][..., 0], mix) and np.array_equal(got["hist"][..., 0], hist), (fname, case["seed"])


def test_goldens_cover_the_edges():
    docs = [json.load(open(os.path.join(JRES_GOLDEN, f))) for f in GOLDEN_FILES]
    assert {c["rng"] for d in docs for c in d["cases"]} == {"philox", "mt"}
    assert any(c["jobs_finished"] == 0 for d in docs for c in d["cases"])
    for d in docs:
        for c in d["cases"]:
            assert all(m[-1] == 0 for dc in c["mix"] for m in dc), "OFF_LEVEL"
            assert all(h[0] == 0 and h[-1] == 0 for dc in c["hist"] for h in dc), "clamped energy bin"


def _mirror_inputs(name="ragged_3dc_12_5_40", n=4, bad=(1,)):
    sp = SC.to_spec(SC.BY_NAME[name])
    got = HJ.run_batch(sp.to_bytes(), n, SEED, sp.log_interval, sp.max_gpus_per_job)
    status = np.zeros(n)
    status[list(bad)] = 1
    G = HJ.mix_g(sp.max_gpus_per_job)
    mix = got["mix"][:, :, :-1].reshape(sp.n_dc, 2, G, 16, n)
    return sp, got, status, mix


def test_mirror_statistics():
    """job_resources_from_rows: bad-status replicas are left out; the pooled sums, mix and histogram are the sums over
    the valid replicas; MEAN_* columns are *_SUM / JOBS per replica; the energy quantiles lie in their bins."""
    sp, got, status, mix = _mirror_inputs()
    good = status == 0
    res = EN.job_resources_from_rows(got["rows"], mix, got["mix"][:, :, -1], got["hist"], got["jens"][:, 0], status,
                                     EN._res_levels(sp), sp.log_interval, sp.end_time)
    assert np.array_equal(res.jobs, got["jens"][-1, 0][..., good].sum(axis=-1))
    assert np.array_equal(res.mix, mix[..., good].sum(axis=-1))
    assert np.array_equal(res.energy_histogram, got["hist"][..., good].sum(axis=-1))
    assert np.allclose(res.energy_sum, got["rows"][-1, 2][..., good].sum(axis=-1), rtol=1e-12)
    W = got["rows"].shape[0] - 1
    i = res.fields.index("mean_gpus")
    for d in range(sp.n_dc):
        for jt in range(2):
            jobs = got["jens"][W, 0, d, jt][good]
            vals = got["rows"][W, 0, d, jt][good][jobs > 0] / jobs[jobs > 0]
            assert res.n[W, i, d, jt] == len(vals)
            if len(vals):
                assert res.min[W, i, d, jt] == vals.min() and res.max[W, i, d, jt] == vals.max()
                sh = res.mix_shares(d, jt)
                assert math.isclose(float(np.nansum(sh)), 1.0, rel_tol=1e-12)
                edges = EN.energy_bin_edges()
                for q, v in zip((0.5, 0.99), res.energy_quantiles(d, jt, (0.5, 0.99))):
                    cum = np.cumsum(res.energy_histogram[d, jt])
                    b = int(np.searchsorted(cum, q * cum[-1]))
                    assert edges[b] <= v <= edges[b + 1]
    pooled = res.pooled()
    assert set(pooled) == set(range(sp.n_dc)) and set(pooled[0]) == {"inference", "training"}
    e = pooled[2]["inference"]
    assert e["jobs"] == int(res.jobs[2, 0]) and math.isclose(sum(e["mix"].values()), 1.0, rel_tol=1e-12)
    assert e["off_level_share"] == 0.0


def test_mirror_energy_bin_rule():
    """ensemble.energy_bin is the recorder's rule: floor(4 log2 E) decided exactly, around every edge."""
    vals = [0.0, 0.5, 1.0, 2.0 ** 31.99, 2.0 ** 40]
    for k in range(1, 128):
        x = 2.0 ** (k / 4.0)
        vals += [x, math.nextafter(x, 0.0), math.nextafter(x, math.inf)]
    assert [int(b) for b in EN.energy_bin(np.array(vals))] == [ebin_exact(v) for v in vals]


def test_mirror_csv_and_accessors(tmp_path):
    """The CSV: window rows of the three means, then per DC and type energy_j, one mix row per (n, f) and the
    off-level row; the mix rows' counts add up to the jobs."""
    sp, got, status, mix = _mirror_inputs()
    res = EN.job_resources_from_rows(got["rows"], mix, got["mix"][:, :, -1], got["hist"], got["jens"][:, 0], status,
                                     EN._res_levels(sp), sp.log_interval, sp.end_time)
    names = [f"DC{d}" for d in range(sp.n_dc)]
    out = tmp_path / "r.csv"
    res.to_csv(str(out), names)
    import csv as _csv
    rows = list(_csv.reader(open(out)))
    assert rows[0] == EN.JOB_CSV_HEADER_HEAD + res.quantile_names() + ["max"]
    W = got["rows"].shape[0] - 1
    win = [r for r in rows[1:] if r[4] in EN.RES_CSV_FIELDS]
    assert len(win) == (W + 1) * sp.n_dc * 2 * 3
    for d in range(sp.n_dc):
        for jt, t in enumerate(EN.JOB_TYPES):
            mine = [r for r in rows[1:] if r[2] == names[d] and r[3] == t]
            e = [r for r in mine if r[4] == "energy_j"][0]
            assert int(e[5]) == int(res.jobs[d, jt])
            m = [r for r in mine if r[4].startswith("mix_")]
            assert len(m) == HJ.mix_g(sp.max_gpus_per_job) * sp.dc[d].n_freq + 1
            assert sum(int(r[5]) for r in m) == int(res.jobs[d, jt])
            assert m[-1][4] == "mix_off_level" and int(m[-1][5]) == 0


def test_cli_flag_summary_and_compare_refusal():
    """--job-resources-csv turns the drop-in's job_resources on (windows of --job-ensemble-bin); --summary-json gains
    the job_resources object only then; --compare-algos refuses the flag."""
    from distributed_cluster_gpus_b200 import run_sim_paper as R
    a = R.parse_args(["--job-resources-csv", "r.csv", "--job-ensemble-bin", "3"])
    assert a.job_resources_csv == "r.csv" and a.job_ensemble_bin == 3.0
    assert R.parse_args([]).job_resources_csv is None
    with pytest.raises(SystemExit) as ei:
        R.main(["--compare-algos", "default_policy,cap_greedy", "--job-resources-csv", "r.csv"])
    assert "--job-resources-csv" in str(ei.value)
    sp, got, status, mix = _mirror_inputs()
    res = EN.job_resources_from_rows(got["rows"], mix, got["mix"][:, :, -1], got["hist"], got["jens"][:, 0], status,
                                     EN._res_levels(sp), sp.log_interval, sp.end_time)

    class _Sim:
        dcs = {f"n{d}": type("D", (), {"name": f"DC{d}"})() for d in range(sp.n_dc)}
    stats = {}
    R._add_job_resources(stats, None, _Sim)
    assert "job_resources" not in stats
    R._add_job_resources(stats, res, _Sim)
    obj = json.loads(json.dumps(stats["job_resources"]))
    assert set(obj) == {f"DC{d}" for d in range(sp.n_dc)}
    assert {"jobs", "mean_gpus", "mean_freq_ghz", "mean_energy_j", "mix"} <= set(obj["DC0"]["inference"])
