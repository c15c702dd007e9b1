"""Every batch recorder at once, on random scenarios and at the edges no fixture reaches, on the CPU: the host build of
the device source (tests/hostemu) with the cluster ensemble, the job ensemble with waits and job resources, the power
profile, occupancy, tail latency and the batch latency histogram all on, every replica held bit for bit to the C oracle
through each recorder's own checker and the oracle's power-profile probe (tests/oracle_jobs/oracle_power.c); the
identities the recorders share (one finish handler, one layout switch); the summaries against a run with every recorder
off; the other loop and staging modes and MT19937.  tests/test_recorder_corpus_gpu.py runs the same corpus and edges on
the H100."""
import functools
import os
import random
import sys

import numpy as np
import pytest

import hostemu_lib as H
import oracle_probes_lib as OP
import test_cluster_ensemble as TCE
import test_job_ensemble as TJE
import test_job_resources as TJR
import test_job_waits as TJW
import test_occupancy as TOC
import test_power_profile as TPP
import test_tail_latency as TTL
from conftest import ROOT
from distributed_cluster_gpus_b200 import ensemble as EN, scenarios as SC, spec as S

sys.path.insert(0, os.path.join(ROOT, "tools"))
import fuzz_core  # noqa: E402

# the generator seed of test_gpu_parity.test_random_scenarios_match_oracle: its first 90 cases are known to be well
# conditioned at 1e-9 on the device; the CPU takes more of the same stream
CORPUS_SEED = 20260923
N_CPU = 200
N_REP = 2
SLA = TTL.SLA                 # the tail checker's SLA (0.5 s)
MODE_SLICE = range(0, N_CPU, 10)


def corpus(n):
    """[(scenario, seed)] of the first n cases: the stream of fuzz_core.random_scenario at CORPUS_SEED."""
    rnd = random.Random(CORPUS_SEED)
    out = []
    for case in range(n):
        sc = fuzz_core.random_scenario(rnd, case)
        out.append((sc, rnd.randrange(1, 2 ** 40)))
    return out


def pp_threshold(sc, blob):
    """The case's power cap, else a quarter of the histogram range: a threshold most runs cross."""
    return sc["power_cap"] if sc.get("power_cap", 0.0) > 0 else H.power_range(blob) / 4


def _scaled_power(sp, k):
    """Every DC's busy-power coefficients times k (the oracle reads the same Spec): E_job and the power profile move
    by k, nothing the event loop decides from does."""
    for d in range(sp.n_dc):
        for jt in range(2):
            c = sp.dc[d].coeffs[jt]
            c.alpha_p, c.beta_p, c.gamma_p = c.alpha_p * k, c.beta_p * k, c.gamma_p * k
    return sp


def _saturated(g):
    return SC.scenario(f"saturated_1x{g}", 1, g, SC.POI(200.0), SC.POI(10.0), 12.0)


# name -> (scenario, Spec transform or None): the edges of the recorders' rules that the random corpus does not reach, each asserted to be reached by test_corpus_reaches_its_edges
EDGES = {
    # debug pins every job at fixed_freq, here between two levels of the 8-level ladder: the mix's OFF_LEVEL column
    "off_ladder_debug": (SC.scenario("off_ladder_debug", 2, 16, SC.POI(8.0), SC.POI(0.5), 30.0, algo="debug",
                                     fixed_freq=0.85), None),
    # E_job below 1 J (energy bin 0) and above 2^(127/4) J (clamped into bin 127)
    "power_x1e-4": (dict(SC.CFG3, name="power_x1e-4", duration=30.0), lambda sp: _scaled_power(sp, 1e-4)),
    "power_x1e9": (dict(SC.CFG3, name="power_x1e9", duration=30.0), lambda sp: _scaled_power(sp, 1e9)),
    # busy-GPU bin widths 1, 2, 2, 3; 200 inference and 10 training jobs/s keep the queue past its last bin
    **{f"saturated_1x{g}": (_saturated(g), None) for g in (127, 128, 255, 256)},
    # log_interval > duration: the cluster ensemble has zero ticks
    "no_log_tick": (SC.scenario("no_log_tick", 2, 16, SC.POI(5.0), SC.POI(0.5), 20.0, log_interval=1000.0), None),
    # no arrival and no log tick: not one event, every recorder empty
    "empty_run": (SC.scenario("empty_run", 2, 8, SC.OFF, SC.OFF, 20.0, log_interval=1000.0), None),
}
STATUS_EDGE = "cap_run_overflow"
STATUS_SC = dict(SC.BY_NAME["sweep_joint_nf"], name=STATUS_EDGE, duration=30.0)  # replicas need 33 to 45 records
STATUS_REP = 7


def edge_spec(name):
    sc, fn = EDGES[name]
    sp = SC.to_spec(sc)
    return sc, (fn(sp) if fn else sp)


@functools.lru_cache(maxsize=None)
def status_caps():
    """cap_run between the smallest and the largest need (S_MAX_RUN) of the STATUS_REP replicas, so some overflow."""
    need = H.run_batch(SC.to_spec(STATUS_SC).to_bytes(), STATUS_REP, 0, lat_hist=False)["summary"][:, S.S_MAX_RUN]
    lo, hi = int(need.min()), int(need.max())
    assert hi > lo + 1, (lo, hi)
    return {"cap_run": (lo + hi) // 2}, need


def run_all(sc, sp, n, seed0, **kw):
    """The host build with every recorder on at once."""
    blob = sp.to_bytes()
    return H.run_batch(blob, n, seed0, ens_cap=H.ens_ticks(blob), jens_bin=sp.log_interval, jwait=True, jres=True,
                       pp=True, pp_threshold=pp_threshold(sc, blob), occ=True, tail=True, tail_sla=SLA, prepass=True,
                       **kw)


def bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.uint64) if a.dtype == np.float64 else a


def assert_same_outputs(got, want, what):
    """Every recorder's output and the summaries bit for bit (NaN bit patterns included)."""
    for k in OUTPUTS:
        if k in want:
            assert np.array_equal(bits(got[k]), bits(want[k])), (what, k, np.argwhere(bits(got[k]) != bits(want[k]))[:5])


OUTPUTS = ("summary", "lat_hist", "ens", "jens", "jens_hist", "jwait", "jwait_hist", "jres", "jres_mix", "jres_hist",
           "pp", "occ", "tail_cols")


def check_oracle(oracle, sc, sp, got, seed0, n, rng_kind=0):
    """Every replica of every recorder against the oracle, bit for bit, through each recorder's own checker."""
    blob = sp.to_bytes()
    bin_s = sp.log_interval
    if H.ens_ticks(blob):
        TCE._check_recorded(oracle, sp, got, seed0, n, rng_kind)
    TJE._check_recorded(oracle, sp, got, seed0, n, bin_s, rng_kind)
    TJW._check(sp, got, seed0, n, bin_s, rng_kind)
    TJR.check(sp, got, seed0, n, bin_s, rng_kind)
    TOC._check_oracle(sp, got, seed0, n, rng_kind)
    TTL._check(sp, got, seed0, n, rng_kind)
    thr, hi = pp_threshold(sc, blob), H.power_range(blob)
    for r in range(n):
        TPP.assert_bits(got["pp"][:, r], OP.oracle_power_profile(blob, seed0 + r, thr, rng_kind, hi), f"power replica {r}")


def check_identities(sp, got, what):
    """What the recorders share: every finished job is counted once by each of them, in the same (DC, type) cell."""
    n_dc, sm = sp.n_dc, got["summary"]
    jobs = got["jens"][-1, 0]                                                     # [n_dc, 2, R]
    tail = got["tail_cols"]
    tail_jobs = np.stack([np.stack([tail[S.tail_col(n_dc, jt, S.TAIL_JOBS, d)] for jt in range(2)]) for d in range(n_dc)])
    for name, x in (("tail JOBS", tail_jobs), ("jres mix", got["jres_mix"].sum(axis=2)),
                    ("jres energy bins", got["jres_hist"].sum(axis=2)),
                    ("wait counts", got["jwait_hist"].sum(axis=-1)[:, :, 0].transpose(1, 2, 0)),
                    ("response counts", got["jwait_hist"].sum(axis=-1)[:, :, 1].transpose(1, 2, 0))):
        assert np.array_equal(x, jobs), (what, name)
    assert np.array_equal(jobs.sum(axis=(0, 1)), sm[:, S.S_JOBS_FINISHED]), what
    assert np.array_equal(jobs.sum(axis=0)[0], sm[:, S.S_FIN_INF]) and np.array_equal(jobs.sum(axis=0)[1], sm[:, S.S_FIN_TRN])
    assert np.array_equal(got["jens_hist"].sum(axis=1), got["lat_hist"]), what
    assert np.array_equal(bits(got["occ"][0]), bits(got["pp"][S.PP_PROFILE_S])), what
    unf = sum(tail[S.tail_col(n_dc, jt, S.TAIL_UNFINISHED, d)] for jt in range(2) for d in range(n_dc))
    assert np.array_equal(unf, sm[:, S.S_JOBS_CREATED] - sm[:, S.S_JOBS_FINISHED]), what
    assert np.all(got["pp"][S.PP_OUT_OF_RANGE] == 0), what


def check_summaries_unchanged(sp, got, n, seed0, what, **kw):
    off = H.run_batch(sp.to_bytes(), n, seed0, lat_hist=False, **kw)
    assert np.array_equal(bits(got["summary"]), bits(off["summary"])), what


def test_power_probe_equals_reference_fixtures():
    """The oracle's power-profile probe against every case of the reference-derived fixtures (tests/golden/power),
    Philox and MT19937, bit for bit: only then is it a reference for scenarios without a fixture."""
    n = 0
    for name in TPP.FIXTURES:
        doc = TPP.load(name)
        blob = SC.to_spec(doc["scenario"]).to_bytes()
        for case in doc["cases"]:
            rng = 1 if case["rng"] == "mt" else 0
            got = OP.oracle_power_profile(blob, case["seed"], TPP.threshold_of(doc), rng, float.fromhex(doc["hi"]))
            TPP.assert_bits(got, TPP.expected_column(doc, case), f"{name} {case['rng']} {case['seed']}")
            n += 1
    assert n == 22


SLICES = 5


@pytest.mark.parametrize("part", range(SLICES))
def test_corpus_equals_oracle(oracle, part):
    """Every recorder of every replica against the oracle, bit for bit; the identities; the summaries of a run with
    every recorder off."""
    for case, (sc, seed) in enumerate(corpus(N_CPU)):
        if case % SLICES != part:
            continue
        sp = SC.to_spec(sc)
        got = run_all(sc, sp, N_REP, seed)
        if np.any(got["summary"][:, S.S_STATUS] != 0):
            pytest.fail(f"case {case}: status {got['summary'][:, S.S_STATUS]} {sc}")
        what = (case, sc["name"], seed)
        check_oracle(oracle, sc, sp, got, seed, N_REP)
        check_identities(sp, got, what)
        check_summaries_unchanged(sp, got, N_REP, seed, what)


def test_corpus_modes_give_identical_outputs(oracle, monkeypatch):
    """A slice of the corpus in chunks of 61 events, in the warp-uniform loop and with the running-job records used where
    they live (head-staged): every output bit for bit the one-shot run's.  On MT19937: the oracle, bit for bit."""
    cases = corpus(N_CPU)
    for case in MODE_SLICE:
        sc, seed = cases[case]
        sp = SC.to_spec(sc)
        one = run_all(sc, sp, N_REP, seed)
        for mode, kw, records in (("chunks61", dict(chunk_events=61), "shared"), ("uniform", dict(uniform=True), "shared"),
                                  ("head_staged", dict(chunk_events=977), "global")):
            monkeypatch.setenv("DCSIM_RECORDS", records)
            assert_same_outputs(run_all(sc, sp, N_REP, seed, **kw), one, (case, mode))
        monkeypatch.setenv("DCSIM_RECORDS", "shared")
        mt = run_all(sc, sp, N_REP, seed, rng_kind=1, chunk_events=61)
        check_oracle(oracle, sc, sp, mt, seed, N_REP, rng_kind=1)
        check_identities(sp, mt, (case, "mt"))


ALONE = (("lat", dict(lat_hist=True), ("lat_hist",)), ("ens", dict(ens_cap=None), ("ens",)),
         ("jens", dict(jens_bin=True), ("jens", "jens_hist")), ("jwait", dict(jens_bin=True, jwait=True), ("jwait", "jwait_hist")),
         ("jres", dict(jens_bin=True, jres=True), ("jres", "jres_mix", "jres_hist")), ("pp", dict(pp=True), ("pp",)),
         ("occ", dict(occ=True), ("occ",)), ("tail", dict(tail=True, prepass=True), ("tail_cols",)))


@pytest.mark.parametrize("case", [0, 1, 2, 6])
def test_each_recorder_alone_equals_all_on(case):
    """Each recorder alone (the job recorders with the job ensemble they hang off, nothing else, not even the batch
    latency histogram) gives bit for bit what it gives with every recorder on, with the summaries unchanged: each one
    must be reached by the finish handler's opt-in test on its own."""
    sc, seed = corpus(N_CPU)[case]
    sp = SC.to_spec(sc)
    blob = sp.to_bytes()
    together = run_all(sc, sp, N_REP, seed)
    for rec, kw, keys in ALONE:
        kw = dict(kw, lat_hist=kw.get("lat_hist", False))
        if "ens_cap" in kw:
            kw["ens_cap"] = H.ens_ticks(blob)
        if "jens_bin" in kw:
            kw["jens_bin"] = sp.log_interval
        if "pp" in kw:
            kw["pp_threshold"] = pp_threshold(sc, blob)
        if "tail" in kw:
            kw["tail_sla"] = SLA
        alone = H.run_batch(blob, N_REP, seed, **kw)
        assert np.array_equal(bits(alone["summary"]), bits(together["summary"])), (case, rec)
        for k in keys:
            if k in together:
                assert np.array_equal(bits(alone[k]), bits(together[k])), (case, rec, k)


@pytest.mark.parametrize("name", list(EDGES))
def test_edge_equals_oracle(oracle, name):
    """Each edge scenario with every recorder on: the oracle bit for bit, the identities, the summaries unchanged; one
    shot and in chunks of 61 events on the warp-uniform loop."""
    sc, sp = edge_spec(name)
    got = run_all(sc, sp, N_REP, 900)
    assert np.all(got["summary"][:, S.S_STATUS] == 0)
    check_oracle(oracle, sc, sp, got, 900, N_REP)
    check_identities(sp, got, name)
    check_summaries_unchanged(sp, got, N_REP, 900, name)
    assert_same_outputs(run_all(sc, sp, N_REP, 900, chunk_events=61, uniform=True), got, name)


def test_zero_tick_and_empty_runs():
    """log_interval > duration: no tick (the default tick capacity is 0), the cluster ensemble's statistics are empty.
    No event at all: every recorder holds zeros, every order statistic of the tail is NaN and its SLA bit too."""
    sc, sp = edge_spec("no_log_tick")
    blob = sp.to_bytes()
    got = run_all(sc, sp, N_REP, 900)
    assert H.ens_ticks(blob) == 0 and np.all(got["summary"][:, S.S_EV_LOG] == 0)
    assert np.all(got["summary"][:, S.S_JOBS_FINISHED] > 0)
    res = EN.cluster_ensemble_from_rows(np.zeros((0, len(EN.FIELDS), sp.n_dc, N_REP)), got["summary"][:, S.S_EV_LOG],
                                        sp.log_interval)
    assert res.n.shape == res.mean.shape == (0, len(EN.FIELDS), sp.n_dc) and len(res.time_s) == 0
    sc, sp = edge_spec("empty_run")
    got = run_all(sc, sp, N_REP, 900)
    sm = got["summary"]
    assert np.all(sm[:, S.S_EVENTS] == 0) and np.all(sm[:, S.S_STATUS] == 0) and np.all(sm[:, S.S_DONE] == 1)
    for k in ("lat_hist", "jens", "jens_hist", "jwait", "jwait_hist", "jres", "jres_mix", "jres_hist", "pp", "occ"):
        assert not np.any(got[k]), k
    n_dc = sp.n_dc
    counts = [S.tail_col(n_dc, jt, f, d) for jt in range(2) for f in (S.TAIL_JOBS, S.TAIL_UNFINISHED)
              for d in range(-1, n_dc)]
    assert np.all(got["tail_cols"][counts] == 0)
    rest = np.setdiff1d(np.arange(S.tail_cols(n_dc)), counts)
    assert np.all(np.isnan(got["tail_cols"][rest]))


def test_status_bit_replicas():
    """A batch in which some replicas overflow cap_run: exactly those carry the bit; every recorder's column of every
    other replica is bit for bit what it is with room to spare; the tail columns of the failed replicas are NaN."""
    caps, need = status_caps()
    sp_ok = SC.to_spec(STATUS_SC)
    sp = SC.to_spec(STATUS_SC, caps=caps)
    got, full = run_all(STATUS_SC, sp, STATUS_REP, 0), run_all(STATUS_SC, sp_ok, STATUS_REP, 0)
    st = got["summary"][:, S.S_STATUS].astype(np.int64)
    bad = need > caps["cap_run"]
    assert np.array_equal((st & S.ST_RUN_OVERFLOW) != 0, bad) and np.all(st[~bad] == 0) and bad.any() and (~bad).any()
    assert np.all(np.isnan(got["tail_cols"][:, bad]))
    for k in OUTPUTS:
        a, b = got[k], full[k]
        if k in ("summary", "lat_hist"):
            a, b = a[~bad], b[~bad]
        elif k in ("jens_hist", "jwait_hist"):
            a, b = a[~bad], b[~bad]
        else:
            a, b = a[..., ~bad], b[..., ~bad]
        if k == "summary":
            a, b = a.copy(), b.copy()
            a[:, S.S_MAX_XFER] = b[:, S.S_MAX_XFER] = 0
        assert np.array_equal(bits(a), bits(b)), k


@functools.lru_cache(maxsize=None)
def edge_reach():
    """What the edge scenarios reach, from the host build alone."""
    out = {}
    for name in EDGES:
        sc, sp = edge_spec(name)
        blob = sp.to_bytes()
        got = run_all(sc, sp, N_REP, 900)
        q_last = sum(TOC._qbins(got["occ"], sp, d)[-1].sum() for d in range(sp.n_dc))
        out[name] = dict(off_level=int(got["jres_mix"][:, :, -1].sum()), ebins=got["jres_hist"].sum(axis=(0, 1, 3)),
                         widths={(sp.dc[d].total_gpus + S.OCC_BINS) // S.OCC_BINS for d in range(sp.n_dc)},
                         q_last=q_last, ticks=H.ens_ticks(blob), events=int(got["summary"][:, S.S_EVENTS].sum()))
    return out


def test_corpus_reaches_its_edges():
    """The corpus and the edge scenarios reach what they are there for, so a later change to the generator or to a
    scenario cannot silently drop an edge: every algo and 1, 5 and 8 DCs; OFF_LEVEL > 0; energy bins 0 and 127;
    busy-GPU bin widths 1, 2 and 3 and the last queue-length bin; a zero-tick run, an empty run and replicas with a
    status bit."""
    cases = corpus(N_CPU)
    assert {sc["algo"] for sc, _ in cases} == set(fuzz_core.ALGOS)
    assert {1, 5, 8} <= {sc["n_dc"] for sc, _ in cases}
    assert any(sc["log_interval"] > sc["duration"] for sc, _ in cases)
    reach = edge_reach()
    assert reach["off_ladder_debug"]["off_level"] > 0
    assert reach["power_x1e-4"]["ebins"][0] > 0 and reach["power_x1e9"]["ebins"][127] > 0
    assert [reach[f"saturated_1x{g}"]["widths"] for g in (127, 128, 255, 256)] == [{1}, {2}, {2}, {3}]
    assert all(reach[f"saturated_1x{g}"]["q_last"] > 0 for g in (127, 128, 255, 256))
    assert reach["no_log_tick"]["ticks"] == 0 and reach["no_log_tick"]["events"] > 0
    assert reach["empty_run"]["events"] == 0
    caps, need = status_caps()
    assert np.any(need > caps["cap_run"]) and np.any(need <= caps["cap_run"])
