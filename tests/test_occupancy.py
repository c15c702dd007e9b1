"""Occupancy on the CPU: the recorder of the device source (host build, tests/hostemu) against the
unmodified reference's fixtures and the C oracle stepped one event at a time (tests/oracle_jobs/oracle_occ.c), Little's
law against the oracle's per-job instants, the recorder's invariants and off switch, and the numpy mirror's CSV against
pinned fixtures."""
import importlib.util
import os

import numpy as np
import pytest

import hostemu_lib as H
import oracle_probes_lib as OP
from conftest import GOLDEN_DIR
from distributed_cluster_gpus_b200 import ensemble as EN, scenarios as SC, spec as S

_spec = importlib.util.spec_from_file_location("make_golden_occ_csv", os.path.join(GOLDEN_DIR, "make_golden_occ_csv.py"))
G = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(G)

SEED = 123
N_REP = 2
# a DC saturated for long stretches; ragged DCs of which the 5-GPU one queues; cap_greedy (stale finishes); eco_route;
# both dequeue orders; zero transfer time; a cluster that never queues; every DC off
SCENARIOS = ["cfg1_1x4_poisson_5000s", "ragged_3dc_12_5_40", "cap_greedy_4x64", "eco_route_cap_2x16",
             "sweep_default_perf_first", "no_inf_priority_perf_first", "zero_xfer_4x64_sin10_60s", "underloaded_1x64",
             "all_off_2x8"]
MT_SCENARIOS = ["ragged_3dc_12_5_40", "cap_greedy_4x64"]


def _spec_of(name, **over):
    return SC.to_spec(dict(SC.BY_NAME[name], **over))


def _field(rows, sp, f, d):
    return rows[1 + f * sp.n_dc + d]


def _qbins(rows, sp, d):
    o = 1 + S.OCC_FIELDS * sp.n_dc + d * S.OCC_BINS
    return rows[o:o + S.OCC_BINS]


def _bbins(rows, sp, d):
    o = 1 + S.OCC_FIELDS * sp.n_dc + (sp.n_dc + d) * S.OCC_BINS
    return rows[o:o + S.OCC_BINS]


REF_DIR = os.path.join(GOLDEN_DIR, "occupancy")
REF_FIXTURES = sorted(f[:-5] for f in os.listdir(REF_DIR) if f.endswith(".json"))


def reference_column(doc, case):
    """One run of a fixture of tests/golden/make_golden_occupancy.py -> the library's column of one replica."""
    D = doc["scenario"]["n_dc"]
    col = np.zeros(H.occ_rows(D))
    col[0] = float.fromhex(case["profile_s"])
    col[1:1 + S.OCC_FIELDS * D] = [float.fromhex(x) for x in case["fields"]]
    for i, x in case["bins"].items():
        col[int(i)] = float.fromhex(x)
    return col


@pytest.mark.parametrize("chunk", [0, 61])
@pytest.mark.parametrize("name", REF_FIXTURES)
def test_recorder_equals_reference_fixtures(name, chunk):
    """Every field and bin equals what the unmodified reference's accrual saw, bit for bit, one shot and in chunks."""
    import json
    with open(os.path.join(REF_DIR, name + ".json")) as f:
        doc = json.load(f)
    sp = SC.to_spec(doc["scenario"])
    for case in doc["cases"]:
        got = H.run_batch(sp.to_bytes(), 1, case["seed"], occ=True, chunk_events=chunk, rng_kind=int(case["rng"] == "mt"),
                           uniform=bool(chunk))
        assert int(got["summary"][0, S.S_EVENTS]) == case["events"]
        want = reference_column(doc, case)
        bad = np.nonzero(got["occ"][:, 0] != want)[0]
        assert len(bad) == 0, (case["seed"], case["rng"], bad[:8], got["occ"][bad[:4], 0], want[bad[:4]])


def _check_oracle(sp, got, seed0, n, rng_kind=0):
    assert np.all(got["summary"][:, S.S_STATUS] == 0)
    for r in range(n):
        want = OP.oracle_occupancy(sp.to_bytes(), seed0 + r, rng_kind)
        bad = np.nonzero(got["occ"][:, r] != want)[0]
        assert len(bad) == 0, (r, bad[:8], got["occ"][bad[:4], r], want[bad[:4]])


@pytest.mark.parametrize("mode", ["one_shot", "chunks61", "uniform", "uniform_chunks61"])
@pytest.mark.parametrize("name", SCENARIOS)
def test_recorder_equals_oracle(name, mode):
    """Every field and bin equals the definition applied to the oracle's state before every event, bit for bit; plain
    and warp-uniform loop, one shot and in chunks of 61 events."""
    sp = _spec_of(name)
    got = H.run_batch(sp.to_bytes(), N_REP, SEED, occ=True, chunk_events=61 if "chunks" in mode else 0,
                       uniform=mode.startswith("uniform"))
    _check_oracle(sp, got, SEED, N_REP)


@pytest.mark.parametrize("name", MT_SCENARIOS)
def test_recorder_equals_oracle_mt19937(name):
    sp = _spec_of(name)
    _check_oracle(sp, H.run_batch(sp.to_bytes(), N_REP, 124, occ=True, chunk_events=61, rng_kind=1), 124, N_REP, rng_kind=1)


def test_recorder_head_staged_records(monkeypatch):
    """The head-staged host mode (the running records used where they live)."""
    monkeypatch.setenv("DCSIM_RECORDS", "global")
    sp = _spec_of("cap_greedy_4x64")
    _check_oracle(sp, H.run_batch(sp.to_bytes(), N_REP, 124, occ=True, chunk_events=977), 124, N_REP)


def _set_quantum(q):
    H.set_test_time_quantum(q)
    OP.set_test_time_quantum(q)


@pytest.fixture
def quantum():
    yield _set_quantum
    _set_quantum(0.0)


@pytest.mark.parametrize("uniform", [False, True])
def test_tie_hook_run(quantum, uniform):
    """Arrival and xfer_done instants on a 0.25 s grid: same-instant events are common, and a finish followed by a
    start at the same instant must leave one level of busy GPUs, not two."""
    sp = SC.to_spec(dict(SC.BY_NAME["cfg3_4x64_sinusoid_120s"]), caps={"cap_xfer": 4096})
    quantum(0.25)
    got = H.run_batch(sp.to_bytes(), N_REP, SEED, occ=True, chunk_events=61, uniform=uniform)
    _check_oracle(sp, got, SEED, N_REP)


def test_coverage():
    """The scenarios above reach what the definition distinguishes: time in the last queue bin, long saturation, a DC
    that never queues, and empty profiles."""
    last_bin = saturated = never_queued = 0
    for name in SCENARIOS:
        sp = _spec_of(name)
        rows = H.run_batch(sp.to_bytes(), N_REP, SEED, occ=True)["occ"]
        for d in range(sp.n_dc):
            last_bin += np.count_nonzero(_qbins(rows, sp, d)[-1] > 0)
            saturated += np.count_nonzero(_field(rows, sp, S.OCC_SATURATED_S, d) > 0.5 * rows[0])
            never_queued += np.count_nonzero(_field(rows, sp, S.OCC_QUEUED_S, d) == 0)
    assert last_bin > 0 and saturated > 0 and never_queued > 0


def test_empty_profile():
    """A run that ends before its first event has PROFILE_S = 0 and nothing else."""
    sp = _spec_of("cfg3_4x64_sinusoid_120s", duration=1e-4)
    got = H.run_batch(sp.to_bytes(), N_REP, SEED, occ=True)
    assert np.all(got["summary"][:, S.S_EVENTS] == 0) and np.all(got["occ"] == 0.0)
    _check_oracle(sp, got, SEED, N_REP)


def _rel_close(a, b, tol=1e-12):
    return abs(a - b) <= tol * max(abs(a), abs(b), 1e-300)


@pytest.mark.parametrize("name", ["ragged_3dc_12_5_40", "cap_greedy_4x64", "no_inf_priority_perf_first",
                                  "cfg1_1x4_poisson_5000s"])
def test_littles_law(name):
    """Q_*_AREA of a DC = sum over the jobs that reached it of min(start, end_time) - xfer_done, RUN_AREA = sum over the
    started jobs of min(finish, end_time) - start, per job type, from the oracle's per-job instants."""
    sp = _spec_of(name)
    got = H.run_batch(sp.to_bytes(), N_REP, SEED, occ=True)
    end = sp.end_time
    checked = 0
    for r in range(N_REP):
        jobs = OP.oracle_reached(sp.to_bytes(), SEED + r)
        rows = got["occ"][:, r]
        for d in range(sp.n_dc):
            at = jobs["dc"] == d
            run = 0.0
            for jt, f in ((0, S.OCC_Q_INF_AREA), (1, S.OCC_Q_TRN_AREA)):
                j = jobs[at & (jobs["jtype"] == jt)]
                q = float(np.sum(np.minimum(j["start"], end) - j["xfer_done"]))
                assert _rel_close(_field(rows, sp, f, d), q), (r, d, jt, _field(rows, sp, f, d), q)
                checked += q > 0
            j = jobs[at & np.isfinite(jobs["start"])]
            run = float(np.sum(np.minimum(j["finish"], end) - j["start"]))
            assert _rel_close(_field(rows, sp, S.OCC_RUN_AREA, d), run), (r, d, _field(rows, sp, S.OCC_RUN_AREA, d), run)
    assert checked > 0


@pytest.mark.parametrize("name", SCENARIOS)
def test_invariants(name):
    """Each DC's queue bins and busy bins sum to PROFILE_S; sum_k k * bin_k of B is the summary's util_gpu_time when the
    bin width is 1; the maxima are integers no larger than the engine's instantaneous S_MAX_Q."""
    sp = _spec_of(name)
    got = H.run_batch(sp.to_bytes(), N_REP, SEED, occ=True)
    for r in range(N_REP):
        rows, summ = got["occ"][:, r], got["summary"][r]
        prof = rows[0]
        assert prof == (sp.end_time - summ[S.S_UTIL_BEGIN] if summ[S.S_EVENTS] else 0.0)
        for d in range(sp.n_dc):
            for bins in (_qbins(rows, sp, d), _bbins(rows, sp, d)):
                assert _rel_close(bins.sum(), prof) or prof == bins.sum() == 0.0
            if sp.dc[d].total_gpus < S.OCC_BINS and prof > 0:
                util = summ[S.S_DC0 + d * S.S_DC_STRIDE + S.SD_UTIL_GPU_TIME]
                assert _rel_close(float(np.sum(np.arange(S.OCC_BINS) * _bbins(rows, sp, d))), util)
            for f in (S.OCC_Q_INF_MAX, S.OCC_Q_TRN_MAX):
                m = _field(rows, sp, f, d)
                assert m == np.floor(m) and m <= summ[S.S_MAX_Q]


@pytest.mark.parametrize("name", ["cap_greedy_4x64", "ragged_3dc_12_5_40", "eco_route_cap_2x16"])
def test_no_side_effects(name):
    """With the recorder on every summary row is bit-identical to it off, and the power profile's rows with the
    occupancy recorder beside it are bit-identical to the power profile alone."""
    sp = _spec_of(name)
    off = H.run_batch(sp.to_bytes(), N_REP, SEED, chunk_events=61)
    on = H.run_batch(sp.to_bytes(), N_REP, SEED, occ=True, chunk_events=61)
    pp = H.run_batch(sp.to_bytes(), N_REP, SEED, chunk_events=61, pp=True)
    both = H.run_batch(sp.to_bytes(), N_REP, SEED, occ=True, chunk_events=61, pp=True)
    assert np.array_equal(on["summary"], off["summary"]) and on["events"] == off["events"]
    assert np.array_equal(both["summary"], off["summary"])
    assert np.array_equal(both["pp"], pp["pp"]) and np.array_equal(both["occ"], on["occ"])


def test_mirror_csv_pinned(tmp_path):
    """The numpy mirror's CSV byte for byte against tests/golden/make_golden_occ_csv.py's fixtures: a bad-status
    replica and an empty profile, a single replica that counts, and none."""
    assert sorted(f for f in os.listdir(G.OUT_DIR) if f.endswith(".csv")) == sorted(f"occupancy_{n}.csv" for n in G.cases())
    for name, (rows, summ, widths) in G.cases().items():
        out = tmp_path / name
        EN.occupancy_from_rows(rows, summ, widths).to_csv(str(out), G.DC_NAMES[:len(widths)])
        with open(os.path.join(G.OUT_DIR, f"occupancy_{name}.csv"), "rb") as f:
            assert out.read_bytes() == f.read(), name


def test_mirror_on_recorded_rows():
    """The mirror's statistics on real rows: counts, batch means, and pooled curves that are the bins' sums."""
    sp = _spec_of("ragged_3dc_12_5_40")
    got = H.run_batch(sp.to_bytes(), 4, SEED, occ=True)
    w = [(g.total_gpus + S.OCC_BINS) // S.OCC_BINS for g in sp.dc[:sp.n_dc]]
    res = EN.occupancy_from_rows(got["occ"], got["summary"], w)
    assert res.replicas == 4
    for d in range(sp.n_dc):
        prof = got["occ"][0]
        c = res.column("mean_q_inf", d)
        assert res.mean[c] == np.sum(_field(got["occ"], sp, S.OCC_Q_INF_AREA, d) / prof) / 4
        assert np.array_equal(res.queue_curve(d)[1], _qbins(got["occ"], sp, d).sum(axis=1))
        assert np.array_equal(res.busy_curve(d)[1], _bbins(got["occ"], sp, d).sum(axis=1))
        top = res.time_quantiles("queue", d, [1e-9])[0]
        assert top == np.nonzero(res.queue_curve(d)[1] > 0)[0].max()


def test_cli_flag_and_compare_refusal():
    """--occupancy-csv turns the drop-in's occupancy on; --compare-algos refuses it."""
    from distributed_cluster_gpus_b200 import run_sim_paper as R
    a = R.parse_args(["--occupancy-csv", "o.csv"])
    assert a.occupancy_csv == "o.csv"
    with pytest.raises(SystemExit) as ei:
        R.main(["--compare-algos", "default_policy,cap_greedy", "--occupancy-csv", "o.csv"])
    assert "--occupancy-csv" in str(ei.value)
