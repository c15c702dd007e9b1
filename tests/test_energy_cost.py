"""Energy cost and carbon on the CPU: the recorder of the device source (its single-lane host build) against fixtures
derived from the unmodified reference and against the stepped C oracle, bit for bit; its agreement with the summary's
per-DC energy; its independence from every other recorder; the hour rule; the numpy mirror of the reductions, its CSV
and its all-reduce over two ranks; the CLI surface."""
import glob
import importlib.util
import json
import os
import random
import sys

import numpy as np
import pytest

import hostemu_cost_lib as H
import oracle_cost_lib as OP
from conftest import GOLDEN_DIR, ROOT
from distributed_cluster_gpus_b200 import ensemble as E
from distributed_cluster_gpus_b200 import scenarios as SC
from distributed_cluster_gpus_b200 import spec as S

sys.path.insert(0, os.path.join(ROOT, "tools"))
import fuzz_core  # noqa: E402

COST_DIR = os.path.join(GOLDEN_DIR, "cost")
FIXTURES = sorted(os.path.basename(p)[:-5] for p in glob.glob(os.path.join(COST_DIR, "*.json")))
_gen = importlib.util.spec_from_file_location("make_golden_cost_csv", os.path.join(GOLDEN_DIR, "make_golden_cost.py"))
# the CSV recipes only: the generator's module body needs no reference tree
GC = importlib.util.module_from_spec(_gen)
_gen.loader.exec_module(GC)

CORPUS_SEED = 20260923        # the generator seed of the recorder corpus (tests/test_recorder_corpus.py)
N_CORPUS = 200
ENERGY_RTOL = 1e-10


def load(name):
    with open(os.path.join(COST_DIR, name + ".json")) as f:
        return json.load(f)


def spec_of(doc):
    return SC.to_spec(doc["scenario"]).to_bytes()


def expected_column(doc, case):
    """The fixture's values as one replica's column [cost_cols(n_dc)]."""
    n_dc = doc["scenario"]["n_dc"]
    c = case["cols"]
    col = np.zeros(S.cost_cols(n_dc))
    for d in range(n_dc):
        for h in range(24):
            col[S.cost_hour_j(n_dc, d, h)] = float.fromhex(c["hour_j"][d][h])
        col[S.cost_energy_j(n_dc, d)] = float.fromhex(c["energy_j"][d])
        col[S.cost_usd(n_dc, d)] = float.fromhex(c["cost_usd"][d])
        col[S.cost_carbon_g(n_dc, d)] = float.fromhex(c["carbon_g"][d])
    col[list(S.cost_totals(n_dc))] = [float.fromhex(c[k]) for k in ("total_j", "total_usd", "total_g")]
    return col


def run_case(doc, case, **kw):
    return H.run_batch(spec_of(doc), 1, case["seed"], cost=True, rng_kind=1 if case["rng"] == "mt" else 0, **kw)


def assert_bits(got, want, what):
    got, want = np.ascontiguousarray(got, dtype=np.float64), np.ascontiguousarray(want, dtype=np.float64)
    bad = np.nonzero(got.view(np.uint64) != want.view(np.uint64))[0]
    assert not len(bad), f"{what}: {len(bad)} values differ, first at {bad[0]}: {got.ravel()[bad[0]]!r} != {want.ravel()[bad[0]]!r}"


def energy_gap(cost, summary, n_dc):
    """Largest relative gap between ENERGY_J[d] and the summary's DCSIM_SD_ENERGY_J over DCs and replicas."""
    gap = 0.0
    for d in range(n_dc):
        want = summary[:, S.S_DC0 + d * S.S_DC_STRIDE + S.SD_ENERGY_J]
        got = cost[S.cost_energy_j(n_dc, d)]
        gap = max(gap, float(np.max(np.abs(got - want) / np.maximum(np.abs(want), 1e-300), initial=0.0)))
    return gap


def test_fixture_set_covers_the_cases():
    """The tariff step at 07:00 with events on hour boundaries, hours folding over more than a day, a per-DC tariff, DCs
    absent from the carbon map, the cap controller's writes, power-gated DCs, a run shorter than one hour, the empty run
    and MT19937 runs are all pinned."""
    assert set(FIXTURES) == {"carbon_cost_8h_2x16", "light_2x8_27h", "tariff_per_dc_3dc_3h", "cap_greedy_4x64",
                             "cfg3_4x64_sinusoid_120s", "short_0p3s_4x64", "all_off_2x8_1s_empty"}
    reached = set()
    for name in FIXTURES:
        doc = load(name)
        sc, sp = doc["scenario"], SC.to_spec(doc["scenario"])
        price = [[float.fromhex(x) for x in row] for row in doc["price_kwh"]]
        for c in doc["cases"]:
            hours = set(c["hours_reached"])
            if {6, 7} <= hours and price[0][6] != price[0][7] and 3600.0 % sc["log_interval"] == 0:
                reached.add("tariff_step_on_boundaries")
            if sc["duration"] > 86400.0 and hours == set(range(24)):
                reached.add("folds_days")
            if c["events"] > 0 and sc["duration"] < 3600.0:
                reached.add("under_an_hour")
            if c["events"] == 0:
                reached.add("empty")
            if c["rng"] == "mt":
                reached.add("mt")
        if "energy_price" in sc and any(row != price[0] for row in price):
            reached.add("per_dc_tariff")
        if any(float.fromhex(x) == 0.0 for x in doc["carbon_intensity"]) and any(float.fromhex(x) > 0 for x in doc["carbon_intensity"]):
            reached.add("absent_from_carbon_map")
        if sc["algo"] == "cap_greedy" and sc["power_cap"] > 0:
            reached.add("cap_controller")
        if any(sp.dc[d].power_gating for d in range(sp.n_dc)):
            reached.add("power_gated")
    assert reached == {"tariff_step_on_boundaries", "folds_days", "under_an_hour", "empty", "mt", "per_dc_tariff",
                       "absent_from_carbon_map", "cap_controller", "power_gated"}, reached


@pytest.mark.parametrize("name", FIXTURES)
def test_spec_tables_are_the_references(name):
    """The spec's price_kwh and carbon_intensity per DC are what the reference's _price_kwh and carbon.get resolve."""
    doc = load(name)
    sp = SC.to_spec(doc["scenario"])
    for d in range(sp.n_dc):
        assert [sp.dc[d].price_kwh[h].hex() for h in range(24)] == doc["price_kwh"][d], (name, d)
        assert sp.dc[d].carbon_intensity.hex() == doc["carbon_intensity"][d], (name, d)


@pytest.mark.parametrize("uniform", [False, True], ids=["plain", "uniform_loop"])
@pytest.mark.parametrize("name", FIXTURES)
def test_host_build_equals_reference_fixture_bit_for_bit(name, uniform):
    doc = load(name)
    for case in doc["cases"]:
        got = run_case(doc, case, uniform=uniform)
        assert got["events"] == case["events"], (name, case["seed"], case["rng"])
        assert_bits(got["cost"][:, 0], expected_column(doc, case), f"{name} {case['rng']} {case['seed']}")


@pytest.mark.parametrize("name", FIXTURES)
def test_chunked_and_head_staged_equal_the_fixture(name, monkeypatch):
    doc = load(name)
    case = doc["cases"][0]
    want = expected_column(doc, case)
    assert_bits(run_case(doc, case, chunk_events=61)["cost"][:, 0], want, "chunks of 61")
    monkeypatch.setenv("DCSIM_RECORDS", "global")
    assert_bits(run_case(doc, case)["cost"][:, 0], want, "head-staged")
    assert_bits(run_case(doc, case, chunk_events=61, uniform=True)["cost"][:, 0], want, "head-staged, uniform, chunked")


@pytest.mark.parametrize("name", FIXTURES)
def test_oracle_probe_equals_reference_fixture_bit_for_bit(name):
    doc = load(name)
    for case in doc["cases"]:
        got = OP.oracle_energy_cost(spec_of(doc), case["seed"], 1 if case["rng"] == "mt" else 0)
        assert_bits(got, expected_column(doc, case), f"{name} {case['rng']} {case['seed']}")


@pytest.mark.parametrize("name", FIXTURES)
def test_fixture_energy_agrees_with_the_references_accrual(name):
    """ENERGY_J[d] sums level pieces, the reference's energy_joules one product per event: equal to 1e-10."""
    doc = load(name)
    for case in doc["cases"]:
        for d, e in enumerate(case["dc_energy_j"]):
            ref, got = float.fromhex(e), float.fromhex(case["cols"]["energy_j"][d])
            assert abs(got - ref) <= ENERGY_RTOL * abs(ref), (name, case["seed"], d, got, ref)


def corpus(n):
    rnd = random.Random(CORPUS_SEED)
    out = []
    for case in range(n):
        sc = fuzz_core.random_scenario(rnd, case)
        out.append((sc, rnd.randrange(1, 2 ** 40)))
    return out


def test_random_scenarios_equal_the_probe_and_the_summary_energy(capsys):
    """200 random scenarios, two replicas each: the host build equals the oracle probe bit for bit, and ENERGY_J[d]
    agrees with DCSIM_SD_ENERGY_J to a relative 1e-10 (the largest gap is printed)."""
    worst = (0.0, None)
    for sc, seed in corpus(N_CORPUS):
        blob = SC.to_spec(sc).to_bytes()
        got = H.run_batch(blob, 2, seed, cost=True)
        for r in range(2):
            if got["summary"][r, S.S_STATUS] != 0:
                continue
            assert_bits(got["cost"][:, r], OP.oracle_energy_cost(blob, seed + r), f"{sc['name']} replica {r}")
        ok = got["summary"][:, S.S_STATUS] == 0
        gap = energy_gap(got["cost"][:, ok], got["summary"][ok], sc["n_dc"])
        if gap > worst[0]:
            worst = (gap, sc["name"])
    with capsys.disabled():
        print(f"\nenergy cost: largest relative gap ENERGY_J vs DCSIM_SD_ENERGY_J over {N_CORPUS} scenarios: "
              f"{worst[0]:.3e} ({worst[1]})")
    assert worst[0] <= ENERGY_RTOL


def test_summaries_and_other_recorders_do_not_depend_on_it():
    """With the cost recorder on, the summaries and every other recorder's outputs are bit-identical to a run with it
    off; the cost columns are the same whether it runs alone or beside them."""
    everything = dict(ens_cap=64, jens_bin=5.0, jwait=True, jres=True, pp=True, pp_threshold=20000.0, occ=True, tail=True,
                      tail_sla=0.5)
    for name in ("cap_greedy_4x64", "ragged_3dc_12_5_40", "sweep_joint_nf"):
        blob = SC.to_spec(SC.BY_NAME[name]).to_bytes()
        off = H.run_batch(blob, 3, 123, **everything)
        on = H.run_batch(blob, 3, 123, cost=True, **everything)
        alone = H.run_batch(blob, 3, 123, cost=True, lat_hist=False)
        for key, v in off.items():
            if isinstance(v, np.ndarray) and v.dtype.names is None:
                assert np.array_equal(on[key].view(np.uint8), v.view(np.uint8)), (name, key)
        assert_bits(on["cost"], alone["cost"], name)
        assert_bits(alone["summary"], off["summary"], name)


def test_piece_hour_agrees_with_the_handlers_hour():
    """At every hour boundary of a multi-day grid, on it and one ulp either side: the hour of day the recorder files a
    piece starting there under (window mod 24) is the hour the handlers price by (dcsim_current_hour)."""
    for k in range(1, 24 * 3 + 1):
        b = 3600.0 * k
        for t in (np.nextafter(b, 0.0), b, np.nextafter(b, np.inf)):
            w = H.cost_window(t)
            assert 3600.0 * w <= t < 3600.0 * (w + 1.0), (k, t, w)
            assert int(w) % 24 == H.current_hour(t), (k, t, w)
            assert int(w) % 24 == int((t % 86400) // 3600)           # the reference's _current_hour


def test_layout_constants_agree():
    hdr = open(os.path.join(ROOT, "include", "dcsim_b200.h")).read()
    for n_dc in (1, 4, 8):
        assert S.cost_cols(n_dc) == (24 + 3) * n_dc + 3 == len(E._cost_columns(n_dc))
        cols = E._cost_columns(n_dc)
        assert cols[S.cost_hour_j(n_dc, n_dc - 1, 23)] == ("hour_j", n_dc - 1, 23)
        assert cols[S.cost_usd(n_dc, 0)] == ("cost_usd", 0, -1)
        assert [cols[c] for c in S.cost_totals(n_dc)] == [(f, -1, -1) for f in E.COST_FIELDS]
    assert "#define DCSIM_COST_COLS(n_dc) ((DCSIM_HOURS + 3) * (n_dc) + 3)" in hdr
    assert S.cost_bytes_per_replica(4) == 984


def brute_force(rows, good, qs):
    x = rows[:, good]
    return {"sum": x.sum(axis=1), "min": x.min(axis=1), "max": x.max(axis=1), "std": x.std(axis=1, ddof=1),
            "q": np.quantile(x, qs, axis=1, method="inverted_cdf")}


def test_numpy_mirror_matches_brute_force():
    sc = SC.BY_NAME["ragged_3dc_12_5_40"]
    sp = SC.to_spec(sc)
    got = H.run_batch(sp.to_bytes(), 30, 500, cost=True)
    status = got["summary"][:, S.S_STATUS].copy()
    status[[3, 17]] = 4.0
    good = status == 0
    price, carbon = E._cost_tables(sp)
    res = E.energy_cost_from_rows(got["cost"], status, price, carbon)
    ref = brute_force(got["cost"], good, res.q)
    assert np.all(res.n == good.sum()) and res.replicas == good.sum()
    assert np.array_equal(res.min, ref["min"]) and np.array_equal(res.max, ref["max"])
    assert np.allclose(res.mean, ref["sum"] / good.sum(), rtol=1e-12)
    assert np.allclose(res.std, ref["std"], rtol=1e-9, atol=1e-12)
    width = E.bin_widths_for(res.min, res.max, np.zeros(len(res.n), dtype=bool))
    assert np.all(np.abs(res.quantiles - ref["q"]) <= width[None, :] + 1e-9)
    p = res.pooled()
    kwh = ref["sum"][S.cost_totals(3)[0]] / 3.6e6
    assert p["cluster"]["energy_kwh"] == pytest.approx(kwh, rel=1e-12)
    assert p["cluster"]["usd_per_kwh"] == pytest.approx(ref["sum"][S.cost_totals(3)[1]] / kwh, rel=1e-12)
    assert p["cluster"]["usd_per_kwh"] == pytest.approx(0.12, rel=1e-12)   # 200 s after midnight: the 00-07 band
    assert p[1]["g_per_kwh"] == 0.0 and p[0]["g_per_kwh"] == pytest.approx(350.0, rel=1e-12)
    hourly = res.hourly(2)
    assert np.allclose(hourly["mean"], ref["sum"][[S.cost_hour_j(3, 2, h) for h in range(24)]] / good.sum(), rtol=1e-12)


@pytest.mark.parametrize("name", sorted(GC.CSV_CASES))
def test_mirror_csv_is_bit_identical_to_the_fixture(name, tmp_path):
    path = tmp_path / name
    GC.CSV_CASES[name](str(path))
    with open(os.path.join(COST_DIR, name), "rb") as f:
        assert path.read_bytes() == f.read()


def test_csv_layout(tmp_path):
    p = tmp_path / "cost.csv"
    GC.CSV_CASES["energy_cost_mixed.csv"](str(p))
    lines = p.read_text().splitlines()
    assert lines[0] == "dc,field,carbon_g_per_kwh,n,mean,std,min,p05,p25,p50,p75,p95,p99,max"
    body = [ln.split(",") for ln in lines[1:]]
    assert len(body) == 3 * 27 + 3
    assert [r[1] for r in body[:27]] == list(E.COST_FIELDS) + [f"hour_j_{h:02d}" for h in range(24)]
    assert {r[2] for r in body if r[0] == "us-east"} == {"0.0"}      # absent from the carbon map: shown as 0 g/kWh
    assert [r[:3] for r in body[-3:]] == [["", f, ""] for f in E.COST_FIELDS]


def _gloo_worker(rank, world, port, out_path):
    import torch.distributed as dist
    for p in (ROOT, os.path.join(ROOT, "tests")):
        if p not in sys.path:
            sys.path.insert(0, p)
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        rows, status, price, carbon = _sharded_inputs()
        half = rows.shape[1] // 2
        mine = slice(0, half) if rank == 0 else slice(half, None)
        res = E.energy_cost_from_rows(rows[:, mine], status[mine], price, carbon)
        if rank == 0:
            np.savez(out_path, n=res.n, mean=res.mean, std=res.std, min=res.min, max=res.max, q=res.quantiles, sum=res.sum)
    finally:
        dist.destroy_process_group()


def _sharded_inputs():
    sp = SC.to_spec(SC.BY_NAME["cap_greedy_4x64"])
    got = H.run_batch(sp.to_bytes(), 9, 77, cost=True)
    status = got["summary"][:, S.S_STATUS].copy()
    status[5] = 2.0
    return got["cost"], status, *E._cost_tables(sp)


def test_two_rank_gloo_equals_one_rank(tmp_path):
    """two_passes over the mirror's columns on two gloo ranks (replicas split between them) equals the one-rank result:
    counts, min, max and the quantiles exactly, means and stds to summation order."""
    import torch.multiprocessing as mp
    out = str(tmp_path / "two.npz")
    port = 29700 + (os.getpid() % 2000)
    mp.spawn(_gloo_worker, args=(2, port, out), nprocs=2, join=True)
    two = np.load(out)
    rows, status, price, carbon = _sharded_inputs()
    one = E.energy_cost_from_rows(rows, status, price, carbon)
    assert np.array_equal(two["n"], one.n) and np.array_equal(two["min"], one.min) and np.array_equal(two["max"], one.max)
    assert np.array_equal(two["q"], one.quantiles)
    assert np.allclose(two["mean"], one.mean, rtol=1e-12) and np.allclose(two["sum"], one.sum, rtol=1e-12)
    assert np.allclose(two["std"], one.std, rtol=1e-9, atol=1e-9)


def test_cli_flag_and_compare_refusal():
    from distributed_cluster_gpus_b200 import run_sim_paper as R
    assert R.parse_args(["--energy-cost-csv", "c.csv"]).energy_cost_csv == "c.csv"
    assert R.parse_args([]).energy_cost_csv is None
    with pytest.raises(SystemExit) as ei:
        R.main(["--compare-algos", "default_policy,carbon_cost", "--energy-cost-csv", "c.csv"])
    assert "--energy-cost-csv" in str(ei.value)
