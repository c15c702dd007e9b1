"""Per-run tail latency on the CPU: the recorder and the selection pass of the device source (host build,
tests/hostemu_ens/hostemu_tail.cpp) against numpy's inverted_cdf order statistics over the oracle's per-job instants
(tests/oracle_jobs/oracle_tail.c) and against golden columns from the unmodified reference; the selection pass alone on
synthetic edge cases; the off switch; the numpy mirror's CSV against a pinned fixture; and the CLI."""
import importlib.util
import json
import math
import os

import numpy as np
import pytest

import hostemu_tail_lib as HT
from conftest import GOLDEN_DIR
from distributed_cluster_gpus_b200 import ensemble as EN, scenarios as SC, spec as S

_spec = importlib.util.spec_from_file_location("make_golden_tail_csv", os.path.join(GOLDEN_DIR, "make_golden_tail_csv.py"))
G = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(G)

SEED = 5200
N_REP = 3
SLA = 0.5
# saturated multi-ingress, cap_greedy (jobs re-timed after start), eco_route, a ragged cluster; groups of one or two jobs;
# mostly exact-zero waits; no jobs at all
FIXTURES = ["cfg3_4x64_sinusoid_120s", "cap_greedy_4x64", "sweep_eco_route", "ragged_3dc_12_5_40", "short_0p3s_4x64",
            "underloaded_1x64", "all_off_2x8"]
TAIL_GOLDEN = os.path.join(GOLDEN_DIR, "tail")


def same(a, b):
    """Bit-identical, NaN where the other is NaN."""
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    return a.shape == b.shape and bool(np.all((a.view(np.uint64) == b.view(np.uint64)) | (np.isnan(a) & np.isnan(b))))


def _check(sp, got, seed0, n, rng_kind=0):
    """Every replica: the slot buffer holds the oracle's created jobs (type, DC, finished or not, instants: exact), and
    every column equals numpy's inverted_cdf over the oracle's instants bit for bit."""
    assert np.all(got["summary"][:, S.S_STATUS] == 0)
    for r in range(n):
        created = int(got["summary"][r, S.S_JOBS_CREATED])
        dev = HT.jobs_from_slots(got["slots"][r], got["arr_t"][r], got["arr_tx"][r], got["arr_meta"][r], created)
        ora = HT.oracle_created(sp.to_bytes(), seed0 + r, rng_kind)
        assert len(ora) == created
        for f in ("jtype", "dc"):
            assert np.array_equal(dev[f], ora[f]), (r, f)
        fin = ~np.isnan(ora["finish"])
        assert np.array_equal(~np.isnan(dev["finish"]), fin), r
        assert np.count_nonzero(fin) == got["summary"][r, S.S_JOBS_FINISHED]
        for f in ("arrival", "start", "finish"):
            assert same(dev[f][fin], ora[f][fin]), (r, f)
        assert same(dev["xfer_done"][fin], ora["xfer_done"][fin])
        want = EN.tail_rows_from_jobs([ora], [0], sp.n_dc, SLA)[:, 0]
        assert same(got["cols"][:, r], want), (r, np.argwhere(~((got["cols"][:, r] == want) | np.isnan(want)))[:5].ravel())
        unf = sum(got["cols"][S.tail_col(sp.n_dc, jt, S.TAIL_UNFINISHED), r] for jt in range(2))
        assert unf == created - got["summary"][r, S.S_JOBS_FINISHED]
        per_dc = sum(got["cols"][S.tail_col(sp.n_dc, jt, S.TAIL_JOBS, d), r] for jt in range(2) for d in range(sp.n_dc))
        assert per_dc == got["summary"][r, S.S_JOBS_FINISHED]


@pytest.mark.parametrize("mode", ["one_shot", "chunks61", "uniform", "uniform_chunks61"])
@pytest.mark.parametrize("name", FIXTURES)
def test_columns_equal_numpy_over_oracle_jobs(name, mode):
    """Every column of every replica is numpy's inverted_cdf order statistic (and count, max, SLA bit) over the oracle's
    per-job instants, bit for bit; plain and warp-uniform loop, one shot and in chunks of 61 events."""
    sp = SC.to_spec(SC.BY_NAME[name])
    got = HT.run_batch(sp.to_bytes(), N_REP, SEED, chunk_events=61 if "chunks" in mode else 0,
                       uniform=mode.startswith("uniform"), sla_s=SLA)
    _check(sp, got, SEED, N_REP)


def test_head_staged_records(monkeypatch):
    """The head-staged host mode (the running records used where they live)."""
    monkeypatch.setenv("DCSIM_RECORDS", "global")
    sp = SC.to_spec(SC.BY_NAME["cap_greedy_4x64"])
    _check(sp, HT.run_batch(sp.to_bytes(), 2, SEED, chunk_events=977, sla_s=SLA), SEED, 2)


def test_fixtures_reach_their_edges():
    """The fixtures cover what they are there for: groups of one or two jobs, mostly exact-zero waits, no jobs at all,
    unfinished jobs and empty groups."""
    def cols(name):
        sp = SC.to_spec(SC.BY_NAME[name])
        return sp, HT.run_batch(sp.to_bytes(), N_REP, SEED, sla_s=SLA)["cols"]
    sp, c = cols("short_0p3s_4x64")
    jobs = c[[S.tail_col(sp.n_dc, jt, S.TAIL_JOBS, d) for jt in range(2) for d in range(-1, sp.n_dc)]]
    assert np.any(jobs == 1) and np.any(jobs == 2)
    sp, c = cols("underloaded_1x64")
    max_wait = c[S.tail_col(sp.n_dc, 0, S.TAIL_STATS_BASE + 1 * 5 + 4)]      # every wait exactly 0
    assert np.all(max_wait == 0.0) and np.all(c[S.tail_col(sp.n_dc, 0, S.TAIL_JOBS)] > 100)
    sp, c = cols("all_off_2x8")
    assert np.all(c[S.tail_col(sp.n_dc, 0, S.TAIL_JOBS)] == 0) and np.all(np.isnan(c[S.tail_col(sp.n_dc, 0, 2)]))
    sp, c = cols("cfg3_4x64_sinusoid_120s")
    assert np.all(c[S.tail_col(sp.n_dc, 0, S.TAIL_UNFINISHED)] > 0)


@pytest.fixture
def quantum():
    yield HT.set_test_time_quantum
    HT.set_test_time_quantum(0.0)


def test_tie_hook_run(quantum):
    """With the tie hook (instants on a 0.25 s grid: ties in every kind) the columns still equal numpy over the
    oracle's instants."""
    sp = SC.to_spec(dict(SC.BY_NAME["cfg3_4x64_sinusoid_120s"]), caps={"cap_xfer": 4096})
    quantum(0.25)
    _check(sp, HT.run_batch(sp.to_bytes(), N_REP, SEED, chunk_events=61, uniform=True, sla_s=SLA), SEED, N_REP)


def test_mt19937_replicas():
    """MT19937 replicas (the stock reference's generator)."""
    sp = SC.to_spec(SC.BY_NAME["ragged_3dc_12_5_40"])
    _check(sp, HT.run_batch(sp.to_bytes(), 2, 123, rng_kind=1, sla_s=SLA), 123, 2, rng_kind=1)


GOLDEN_FILES = sorted(f for f in os.listdir(TAIL_GOLDEN) if f.endswith(".json"))


@pytest.mark.parametrize("fname", GOLDEN_FILES)
def test_golden_from_reference(fname):
    """The host build's columns equal those tests/golden/make_golden_tail.py derived from the unmodified reference's
    own per-job instants, bit for bit (Philox seeds and MT19937 runs)."""
    with open(os.path.join(TAIL_GOLDEN, fname)) as f:
        doc = json.load(f)
    sp = SC.to_spec(doc["scenario"])
    for case in doc["cases"]:
        got = HT.run_batch(sp.to_bytes(), 1, case["seed"], rng_kind=1 if case["rng"] == "mt" else 0,
                           sla_s=doc["meta"]["sla_s"])
        assert got["summary"][0, S.S_JOBS_CREATED] == case["jobs_created"]
        assert got["summary"][0, S.S_JOBS_FINISHED] == case["jobs_finished"]
        want = np.array([np.nan if v is None else float.fromhex(v) for v in case["cols"]])
        assert same(got["cols"][:, 0], want), (fname, case["seed"], case["rng"])


def test_golden_covers_the_edges():
    docs = [json.load(open(os.path.join(TAIL_GOLDEN, f))) for f in GOLDEN_FILES]
    rngs = {c["rng"] for d in docs for c in d["cases"]}
    assert rngs == {"philox", "mt"}
    assert any(c["jobs_created"] > c["jobs_finished"] for d in docs for c in d["cases"])
    assert any(c["jobs_created"] == 0 for d in docs for c in d["cases"])
    assert any(v is None for d in docs for c in d["cases"] for v in c["cols"])


@pytest.mark.parametrize("name", ["cfg3_4x64_sinusoid_120s", "cap_greedy_4x64", "sweep_eco_route", "ragged_3dc_12_5_40"])
def test_summaries_unchanged_by_the_recorder(name):
    """With the recorder on (the records then carry the job id) every summary row is bit-identical to the recorder
    off."""
    sp = SC.to_spec(SC.BY_NAME[name])
    on = HT.run_batch(sp.to_bytes(), N_REP, SEED, chunk_events=61, sla_s=SLA)
    off = HT.run_batch(sp.to_bytes(), N_REP, SEED, chunk_events=61, tail=False)
    assert same(on["summary"], off["summary"]) and on["events"] == off["events"]


# ---- the selection pass alone ------------------------------------------------------------------------------------
SIZES = [1, 2, 3, 20, 99, 100, 101, 1000, 1001, 4097]


def _values(kind, n, rng):
    if kind == "spread":
        return 10.0 ** rng.uniform(-9.0, 6.0, n)
    if kind == "ties":
        return rng.choice(np.array([0.0, 1e-9, 0.25, 0.5, 3.0, 1e6]), n)
    if kind == "all_equal":
        return np.full(n, 0.125)
    if kind == "zeros":
        return np.where(rng.random(n) < 0.9, 0.0, rng.lognormal(0.0, 2.0, n))
    if kind == "reversed":
        return np.sort(10.0 ** rng.uniform(-9.0, 6.0, n))[::-1].copy()
    raise ValueError(kind)


@pytest.mark.parametrize("kind", ["spread", "ties", "all_equal", "zeros", "reversed"])
@pytest.mark.parametrize("n", SIZES)
def test_selection_matches_numpy(n, kind):
    """Synthetic jobs through the selection pass: p50 / p95 / p99 / p99.9 and max of each kind equal np.quantile(...,
    method="inverted_cdf") and max exactly — ties, all-equal values, exact zeros, values from 1e-9 to 1e6, reversed
    order.  Latency = finish - start, wait = start - tx, response = finish - 0 carry three different value sets."""
    rng = np.random.default_rng(n * 7 + len(kind))
    lat, wait = _values(kind, n, rng), _values(kind, n, rng)
    tx = rng.uniform(0.0, 1.0, n)
    start = tx + wait
    finish = start + lat
    cols = HT.select_synthetic(tx, start, finish)
    kinds = (finish - start, start - tx, finish)
    for k, v in enumerate(kinds):
        base = S.tail_col(1, 0, S.TAIL_STATS_BASE + k * 5)
        for i, q in enumerate(S.TAIL_QUANTILES):
            assert same(cols[base + i], np.quantile(v, q, method="inverted_cdf")), (k, q)
            assert same(cols[S.tail_col(1, 0, S.TAIL_STATS_BASE + k * 5 + i, 0)], cols[base + i])
        assert same(cols[base + 4], v.max())
    assert cols[S.tail_col(1, 0, S.TAIL_JOBS)] == n and cols[S.tail_col(1, 0, S.TAIL_UNFINISHED)] == 0
    assert cols[S.tail_col(1, 1, S.TAIL_JOBS)] == 0 and np.isnan(cols[S.tail_col(1, 1, S.TAIL_STATS_BASE)])


def test_rank_rule_below_3000():
    """k = max(ceil(fl(n * q)), 1) is numpy's inverted_cdf index for every n < 3000 at the four quantiles."""
    for n in range(1, 3000):
        v = np.arange(n, dtype=np.float64)
        for q in S.TAIL_QUANTILES:
            k = max(math.ceil(n * q), 1)
            assert np.quantile(v, q, method="inverted_cdf") == k - 1, (n, q)


def test_selection_unfinished_types_and_status():
    """Unfinished jobs (NaN finish) count per type and never enter a quantile; a replica with a status != 0 has every
    column NaN; SLA_MET is p99 <= sla_s, NaN without an SLA or a finished job of the type."""
    rng = np.random.default_rng(3)
    n = 500
    tx = rng.uniform(0.0, 10.0, n)
    start = tx + np.where(rng.random(n) < 0.5, 0.0, rng.uniform(0.0, 2.0, n))
    finish = start + rng.uniform(0.01, 1.0, n)
    jt = (rng.random(n) < 0.3).astype(np.int32)
    finish[rng.random(n) < 0.2] = np.nan
    fin = ~np.isnan(finish)
    p99 = np.quantile((finish - start)[fin & (jt == 0)], 0.99, method="inverted_cdf")
    for sla, want in ((p99, 1.0), (np.nextafter(p99, 0.0), 0.0), (None, np.nan)):
        cols = HT.select_synthetic(tx, start, finish, jt, sla_s=sla)
        assert same(cols[S.tail_sla_col(1, 0, 0)], want)
        for t in range(2):
            assert cols[S.tail_col(1, t, S.TAIL_JOBS)] == np.count_nonzero(fin & (jt == t))
            assert cols[S.tail_col(1, t, S.TAIL_UNFINISHED)] == np.count_nonzero(~fin & (jt == t))
            v = (finish - start)[fin & (jt == t)]
            assert same(cols[S.tail_col(1, t, S.TAIL_STATS_BASE + 2)], np.quantile(v, 0.99, method="inverted_cdf"))
    only_inf = HT.select_synthetic(tx, start, finish, np.zeros(n, dtype=np.int32), sla_s=1.0)
    assert np.isnan(only_inf[S.tail_sla_col(1, 0, 1)]) and not np.isnan(only_inf[S.tail_sla_col(1, 0, 0)])
    assert np.all(np.isnan(HT.select_synthetic(tx, start, finish, jt, sla_s=1.0, status=4.0)))
    empty = HT.select_synthetic(np.zeros(0), np.zeros(0), np.zeros(0), sla_s=1.0)
    assert np.all(empty[[S.tail_col(1, t, f, d) for t in range(2) for d in (-1, 0) for f in (0, 1)]] == 0)
    assert np.all(np.isnan(empty[[S.tail_sla_col(1, k, t) for k in range(3) for t in range(2)]]))


# ---- the numpy mirror ----------------------------------------------------------------------------------------------
def test_mirror_csv_pinned(tmp_path):
    """The numpy mirror's CSV byte for byte against the fixtures tests/golden/make_golden_tail_csv.py wrote: ragged job
    counts, unfinished jobs, bad-status replicas, empty groups, and a run without an SLA."""
    assert sorted(f for f in os.listdir(G.OUT_DIR) if f.endswith(".csv")) == sorted(f"tail_latency_{n}.csv" for n in G.cases())
    for name, (args, kw) in G.cases().items():
        out = tmp_path / name
        EN.tail_latency_from_jobs(*args, **kw).to_csv(str(out), G.DC_NAMES[:args[2]])
        with open(os.path.join(G.OUT_DIR, f"tail_latency_{name}.csv"), "rb") as f:
            assert out.read_bytes() == f.read(), name


def test_mirror_result_accessors():
    """column(), sla_attainment() with its Wilson interval, and pooled() read the right columns."""
    args, kw = G.cases()["mixed"]
    res = EN.tail_latency_from_jobs(*args, **kw)
    rows = EN.tail_rows_from_jobs(args[0], args[1], args[2], kw["sla_s"])
    good = args[1] == 0
    c = res.column("response", "inference", "p99")
    assert c == S.tail_col(3, 0, S.TAIL_STATS_BASE + 2 * 5 + 2)
    vals = rows[c][good & ~np.isnan(rows[c])]
    assert res.n[c] == len(vals) and res.max[c] == vals.max() and res.min[c] == vals.min()
    att = res.sla_attainment("latency", 1)
    met = rows[S.tail_sla_col(3, 0, 1)][good]
    met = met[~np.isnan(met)]
    assert att["runs"] == len(met) and att["met"] == int(met.sum()) and att["share"] == met.mean()
    assert att["ci95_lo"] <= att["share"] <= att["ci95_hi"]
    assert res.pooled()["training"]["latency"]["sla_attainment"] == att
    assert res.column(None, 0, "unfinished", 2) == S.tail_col(3, 0, S.TAIL_UNFINISHED, 2)


def test_wilson_interval():
    lo, hi = EN.wilson_interval(0, 10)
    assert lo == 0.0 and 0.27 < hi < 0.28
    lo, hi = EN.wilson_interval(10, 10)
    assert abs(hi - 1.0) < 1e-12 and 0.72 < lo < 0.73
    assert all(math.isnan(x) for x in EN.wilson_interval(0, 0))


# ---- CLI -------------------------------------------------------------------------------------------------------------
def test_cli_flag_and_compare_refusal():
    """--tail-latency-csv turns the drop-in's tail_latency on (SLA from --sla_p99_ms); --compare-algos refuses it."""
    from distributed_cluster_gpus_b200 import run_sim_paper as R
    a = R.parse_args(["--tail-latency-csv", "t.csv", "--sla_p99_ms", "250"])
    assert a.tail_latency_csv == "t.csv" and a.sla_p99_ms == 250.0
    assert R.parse_args([]).tail_latency_csv is None
    with pytest.raises(SystemExit) as ei:
        R.main(["--compare-algos", "default_policy,cap_greedy", "--tail-latency-csv", "t.csv"])
    assert "--tail-latency-csv" in str(ei.value)


def test_summary_json_tail_object():
    """The --summary-json object: per kind and type the SLA attainment and the spread of the per-run p99; absent
    without the flag."""
    from distributed_cluster_gpus_b200 import run_sim_paper as R
    args, kw = G.cases()["mixed"]
    stats = {}
    R._add_tail_latency(stats, None)
    assert "tail_latency" not in stats
    R._add_tail_latency(stats, EN.tail_latency_from_jobs(*args, **kw))
    obj = stats["tail_latency"]
    assert obj["inference"]["latency"]["sla_attainment"]["runs"] == 4
    assert set(obj) == set(EN.TAIL_TYPES) and set(obj["training"]) == set(EN.TAIL_KINDS)
    assert {"p99_mean_s", "p99_p05_s", "p99_p50_s", "p99_p95_s"} <= set(obj["training"]["wait"])
