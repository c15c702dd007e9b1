"""Waiting and response times on the CPU: the recorder of the device source (host build, tests/hostemu_ens) against
every replica's per-job instants from the oracle (tests/oracle_jobs), the wait invariants, the off switch, and the
numpy mirror's CSV against a pinned fixture."""
import importlib.util
import os

import numpy as np
import pytest

import hostemu_jwait_lib as HW
from conftest import GOLDEN_DIR
from distributed_cluster_gpus_b200 import ensemble as EN, scenarios as SC, spec as S

_spec = importlib.util.spec_from_file_location("make_golden_waits", os.path.join(GOLDEN_DIR, "make_golden_waits.py"))
G = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(G)

SEED = 5200
N_REP = 3
# saturated multi-ingress, cap_greedy (jobs re-timed after start), eco_route, an inf_priority dequeue on a ragged cluster
FIXTURES = ["cfg3_4x64_sinusoid_120s", "cap_greedy_4x64", "sweep_eco_route", "ragged_3dc_12_5_40"]


def expected_rows(jobs, n_dc, bin_s, end_time):
    """One replica's oracle jobs (finish order) -> what its recorder holds: (rows [W + 1, 3, n_dc, 2] {waited, wait_sum,
    resp_sum}, hist [n_dc, 2 kinds, 2, LAT_BINS]); each sum a plain sequential f64 sum in finish order."""
    W = EN.job_windows(end_time, bin_s)
    rows = np.zeros((W + 1, 3, n_dc, 2))
    hist = np.zeros((n_dc, 2, 2, EN.LAT_BINS), dtype=np.uint32)
    for j in jobs:
        d, jt = int(j["dc"]), int(j["jtype"])
        wait = float(j["start"]) - float(j["xfer_done"])
        resp = float(j["finish"]) - float(j["arrival"])
        k = int(EN.job_window_index(float(j["finish"]), bin_s, W))
        for row in (k, W):
            if wait > 0.0:
                rows[row, 0, d, jt] += 1.0
            rows[row, 1, d, jt] = rows[row, 1, d, jt] + wait
            rows[row, 2, d, jt] = rows[row, 2, d, jt] + resp
        hist[d, 0, jt, EN.latency_bin(wait)] += 1
        hist[d, 1, jt, EN.latency_bin(resp)] += 1
    return rows, hist


def _check(sp, got, seed0, n, bin_s):
    assert np.all(got["summary"][:, S.S_STATUS] == 0)
    all_jobs = []
    for r in range(n):
        jobs = HW.oracle_jobs(sp.to_bytes(), seed0 + r)
        assert len(jobs) == got["summary"][r, S.S_JOBS_FINISHED]
        rows, hist = expected_rows(jobs, sp.n_dc, bin_s, sp.end_time)
        assert np.array_equal(got["rows"][..., r], rows), (r, np.argwhere(got["rows"][..., r] != rows)[:5])
        assert np.array_equal(got["hist"][r], hist), r
        # WAITED <= jobs in every cell; the histograms count every finished job once per kind
        assert np.all(got["rows"][:, 0, ..., r] <= got["jens"][:, 0, ..., r])
        assert np.array_equal(got["hist"][r].sum(axis=-1)[:, 0], got["jens"][-1, 0, :, :, r])
        all_jobs.append(jobs)
    return np.concatenate(all_jobs)


def _invariants(jobs):
    wait = jobs["start"] - jobs["xfer_done"]
    at = jobs["at_xfer"] == 1
    assert np.all(wait[at] == 0.0), "a job started at its xfer_done waited"
    assert np.all(wait[~at] >= 0.0)
    return wait, at


@pytest.mark.parametrize("mode", ["one_shot", "chunks61", "uniform", "uniform_chunks61"])
@pytest.mark.parametrize("name", FIXTURES)
def test_recorder_equals_oracle_jobs(name, mode):
    """Every WAITED / WAIT_SUM / RESP_SUM cell and every histogram count equals what the oracle's per-job instants give
    in finish order, bit for bit; plain and warp-uniform loop, one shot and in chunks."""
    sp = SC.to_spec(SC.BY_NAME[name])
    kw = {"chunk_events": 61 if "chunks" in mode else 0, "uniform": mode.startswith("uniform")}
    got = HW.run_batch(sp.to_bytes(), N_REP, SEED, sp.log_interval, **kw)
    jobs = _check(sp, got, SEED, N_REP, sp.log_interval)
    wait, at = _invariants(jobs)
    if name != "sweep_eco_route":                    # (eco_route spreads this load without queueing)
        assert np.count_nonzero(wait > 0.0) > 0, "the scenario is supposed to queue jobs"


def test_recorder_head_staged_records(monkeypatch):
    """The head-staged host mode (the running records used where they live)."""
    monkeypatch.setenv("DCSIM_RECORDS", "global")
    sp = SC.to_spec(SC.BY_NAME["cap_greedy_4x64"])
    _check(sp, HW.run_batch(sp.to_bytes(), 2, SEED, 7.0, chunk_events=977), SEED, 2, 7.0)


@pytest.fixture
def quantum():
    yield HW.set_test_time_quantum
    HW.set_test_time_quantum(0.0)


@pytest.mark.parametrize("uniform", [False, True])
def test_tie_hook_run(quantum, uniform):
    """With the tie hook (arrival and xfer_done instants on a 0.25 s grid, so same-instant events are common) the
    recorder still equals the oracle bit for bit, and a job started in its own xfer_done handler waited exactly 0."""
    sc = dict(SC.BY_NAME["cfg3_4x64_sinusoid_120s"])
    sp = SC.to_spec(sc, caps={"cap_xfer": 4096})
    quantum(0.25)
    got = HW.run_batch(sp.to_bytes(), N_REP, SEED, sp.log_interval, chunk_events=61, uniform=uniform)
    jobs = _check(sp, got, SEED, N_REP, sp.log_interval)
    wait, at = _invariants(jobs)
    assert np.count_nonzero(wait > 0.0) > 0 and np.count_nonzero(at) > 0


@pytest.mark.parametrize("uniform", [False, True])
def test_same_instant_dequeue_does_not_count_as_waited(quantum, uniform):
    """WAITED means wait > 0, not "was queued".  The hook only puts arrivals and xfer_done events on the grid, so a
    job_finish lands on a queued job's xfer_done instant only when the service time is nothing: DC 0's inference jobs
    get a step time of 1e-30 s, so they finish at the instant they start (t + size * 1e-30 rounds to t).  Two xfer_dones
    at one instant on a full DC then queue the second job, and the first one's finish dequeues it at that same instant:
    started from the dequeue loop, wait exactly 0.  The other DCs keep their service times, so jobs also really wait."""
    sp = SC.to_spec(dict(SC.BY_NAME["cfg3_4x64_sinusoid_120s"]), caps={"cap_xfer": 4096})
    k = sp.dc[0].coeffs[0]
    k.alpha_t, k.beta_t, k.gamma_t = 1e-30, 0.0, 0.0
    quantum(0.25)
    got = HW.run_batch(sp.to_bytes(), N_REP, SEED, sp.log_interval, chunk_events=61, uniform=uniform)
    jobs = _check(sp, got, SEED, N_REP, sp.log_interval)
    wait, at = _invariants(jobs)
    dequeued_at_once = np.count_nonzero(~at & (wait == 0.0))
    assert dequeued_at_once > 0, "no job was dequeued at its own xfer_done instant"
    assert np.count_nonzero(wait > 0.0) > 0
    # the recorder's whole-run WAITED counts only the jobs that waited, not every job that went through a queue
    assert got["rows"][-1, 0].sum() == np.count_nonzero(wait > 0.0) < np.count_nonzero(~at)


@pytest.mark.parametrize("name", FIXTURES)
def test_summaries_unchanged_by_the_recorder(name):
    """With the recorder on (the records then carry the job id) every summary row, and the job ensemble, are
    bit-identical to the recorder off."""
    sp = SC.to_spec(SC.BY_NAME[name])
    on = HW.run_batch(sp.to_bytes(), N_REP, SEED, sp.log_interval, chunk_events=61)
    off = HW.run_batch(sp.to_bytes(), N_REP, SEED, sp.log_interval, chunk_events=61, waits=False)
    assert np.array_equal(on["summary"], off["summary"]) and on["events"] == off["events"]
    assert np.array_equal(on["jens"], off["jens"]) and np.array_equal(on["jens_hist"], off["jens_hist"])


def test_mirror_csv_pinned(tmp_path):
    """The numpy mirror's CSV byte for byte against the fixture tests/golden/make_golden_waits.py wrote: ragged job
    counts, bad-status replicas, all-zero waits, empty cells, and the exact-zero quantile rule."""
    assert sorted(os.listdir(G.OUT_DIR)) == sorted(f"job_waits_{n}.csv" for n in G.cases())
    for name, (args, kw) in G.cases().items():
        out = tmp_path / name
        EN.job_waits_from_rows(*args, **kw).to_csv(str(out), G.DC_NAMES[:args[0].shape[2]])
        with open(os.path.join(G.OUT_DIR, f"job_waits_{name}.csv"), "rb") as f:
            assert out.read_bytes() == f.read(), name


def test_zero_wait_quantiles_exact():
    """Quantiles of wait_s whose share lies at or below the pooled zero-wait share are exactly 0."""
    args, kw = G.cases()["mixed"]
    res = EN.job_waits_from_rows(*args, **kw)
    checked = 0
    for d in range(res.jobs.shape[0]):
        for jt in range(2):
            if not res.jobs[d, jt]:
                continue
            zero_share = res.zero_wait_share(d, jt)
            for share, v in zip(res.q, res.wait_quantiles(d, jt)):
                assert (v == 0.0) if share <= zero_share else (v > 0.0), (d, jt, share, zero_share, v)
                checked += share <= zero_share < 1.0
    assert checked > 0
    args, kw = G.cases()["all_zero_waits"]
    res = EN.job_waits_from_rows(*args, **kw)
    assert np.all(res.waited == 0) and all(v == 0.0 for v in res.wait_quantiles(0, 0))


def test_cli_flag_and_compare_refusal():
    """--job-waits-csv turns the drop-in's job_waits on (windows of --job-ensemble-bin); --compare-algos refuses it."""
    from distributed_cluster_gpus_b200 import run_sim_paper as R
    a = R.parse_args(["--job-waits-csv", "w.csv", "--job-ensemble-bin", "3"])
    assert a.job_waits_csv == "w.csv" and a.job_ensemble_bin == 3.0
    with pytest.raises(SystemExit) as ei:
        R.main(["--compare-algos", "default_policy,cap_greedy", "--job-waits-csv", "w.csv"])
    assert "--job-waits-csv" in str(ei.value)
