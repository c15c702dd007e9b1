"""Power profile on the CPU: the recorder of the device source (its single-lane host build) against fixtures derived
from the unmodified reference, bit for bit; the identities the profile obeys; the numpy mirror of the reductions; the
CSV and CLI surface."""
import glob
import json
import math
import os

import numpy as np
import pytest

import hostemu_pp_lib as H
from distributed_cluster_gpus_b200 import ensemble as E
from distributed_cluster_gpus_b200 import scenarios as SC
from distributed_cluster_gpus_b200 import spec as S

POWER_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "power")
FIXTURES = sorted(os.path.basename(p)[:-5] for p in glob.glob(os.path.join(POWER_DIR, "*.json")))
NF = S.PP_FIELDS


def load(name):
    with open(os.path.join(POWER_DIR, name + ".json")) as f:
        return json.load(f)


def threshold_of(doc):
    return math.inf if doc["threshold"] == "inf" else float.fromhex(doc["threshold"])


def expected_column(doc, case):
    """The fixture's values as one replica's column [PP_FIELDS + n_dc + PP_BINS]."""
    n_dc = doc["scenario"]["n_dc"]
    col = np.zeros(NF + n_dc + S.PP_BINS)
    for i, f in enumerate(E.PP_FIELDS):
        col[i] = float.fromhex(case["fields"][f])
    col[NF:NF + n_dc] = [float.fromhex(x) for x in case["dc_peak_w"]]
    for k, v in case["bins"].items():
        col[NF + n_dc + int(k)] = float.fromhex(v)
    return col


def run_case(doc, case, **kw):
    rng = 1 if case["rng"] == "mt" else 0
    return H.run_batch(SC.to_spec(doc["scenario"]).to_bytes(), 1, case["seed"], threshold=threshold_of(doc),
                       rng_kind=rng, **kw)


def assert_bits(got, want, what):
    bad = np.nonzero(got.view(np.uint64) != want.view(np.uint64))[0]
    assert not len(bad), f"{what}: {len(bad)} values differ, first at {bad[0]}: {got[bad[0]]!r} != {want[bad[0]]!r}"


def test_fixture_set_covers_the_cases():
    """Crossing twice or more, never crossing, no threshold, an empty profile, and MT19937 runs are all pinned."""
    crossing = never = inf_case = empty = mt = False
    for name in FIXTURES:
        doc = load(name)
        thr = threshold_of(doc)
        for c in doc["cases"]:
            over, exc = float.fromhex(c["fields"]["over_s"]), float.fromhex(c["fields"]["excursions"])
            crossing |= over > 0 and exc >= 2
            never |= math.isfinite(thr) and over == 0 and c["levels"] > 0
            inf_case |= not math.isfinite(thr) and c["levels"] > 0
            empty |= c["levels"] == 0
            mt |= c["rng"] == "mt"
    assert crossing and never and inf_case and empty and mt
    assert len(FIXTURES) == 10


@pytest.mark.parametrize("name", FIXTURES)
def test_histogram_range_is_the_fixtures(name):
    doc = load(name)
    assert H.power_range(SC.to_spec(doc["scenario"]).to_bytes()).hex() == doc["hi"]


@pytest.mark.parametrize("uniform", [False, True], ids=["plain", "uniform_loop"])
@pytest.mark.parametrize("name", FIXTURES)
def test_host_build_equals_reference_fixture_bit_for_bit(name, uniform):
    doc = load(name)
    for case in doc["cases"]:
        got = run_case(doc, case, uniform=uniform)
        assert got["events"] == case["events"], (name, case["seed"], case["rng"])
        assert_bits(got["rows"][:, 0], expected_column(doc, case), f"{name} {case['rng']} {case['seed']}")


@pytest.mark.parametrize("name", ["cap_greedy_4x64", "cfg3_4x64_sinusoid_120s", "zero_xfer_4x64_sin10_60s"])
def test_chunked_and_head_staged_give_identical_rows(name, monkeypatch):
    doc = load(name)
    case = doc["cases"][0]
    one = run_case(doc, case)["rows"]
    for chunk in (13, 61):
        assert_bits(run_case(doc, case, chunk_events=chunk)["rows"], one, f"chunk {chunk}")
    monkeypatch.setenv("DCSIM_RECORDS", "global")
    assert_bits(run_case(doc, case, chunk_events=61, uniform=True)["rows"], one, "head-staged, chunked")


def test_summaries_do_not_depend_on_the_recorder():
    for name in ("cap_greedy_4x64", "sweep_joint_nf", "ragged_3dc_12_5_40"):
        blob = SC.to_spec(SC.BY_NAME[name]).to_bytes()
        on = H.run_batch(blob, 3, 123, threshold=20000.0)
        off = H.run_batch(blob, 3, 123, record=False)
        assert_bits(on["summary"].ravel(), off["summary"].ravel(), name)


def check_identities(rows, summary, hi, n_dc, what):
    """Each replica: the bins sum to profile_s; the total energy lies between the bins' lower- and upper-edge energies
    and below peak x profile_s; the peak lies in range and below the sum of the DC peaks; out_of_range is zero."""
    prof = rows[S.PP_PROFILE_S]
    bins = rows[NF + n_dc:]
    assert np.all(rows[S.PP_OUT_OF_RANGE] == 0), what
    assert np.allclose(bins.sum(axis=0), prof, rtol=1e-12, atol=1e-12), what
    energy = summary[:, S.S_TOTAL_ENERGY_J]
    width = hi / S.PP_BINS
    lo_e = (bins * (np.arange(S.PP_BINS) * width)[:, None]).sum(axis=0)
    hi_e = (bins * ((np.arange(S.PP_BINS) + 1) * width)[:, None]).sum(axis=0)
    assert np.all(lo_e <= energy * (1 + 1e-12) + 1e-9) and np.all(energy <= hi_e * (1 + 1e-12) + 1e-9), what
    has = prof > 0
    assert np.all(rows[S.PP_PEAK_W][has] * prof[has] >= energy[has] * (1 - 1e-12)), what      # peak >= mean power
    assert np.all(rows[S.PP_PEAK_W] <= hi), what
    assert np.all(rows[S.PP_OVER_S] <= prof * (1 + 1e-12)), what
    assert np.all(rows[S.PP_LONGEST_OVER_S] <= rows[S.PP_OVER_S] * (1 + 1e-12) + 1e-12), what
    dc_sum = rows[NF:NF + n_dc].sum(axis=0)
    assert np.all(rows[S.PP_PEAK_W] <= dc_sum * (1 + 1e-12)), what


def test_identities_on_random_scenarios():
    from conftest import load_fuzz_reference
    cases = load_fuzz_reference()
    assert len(cases) >= 160
    for c in cases:
        sc = c["scenario"]
        blob = SC.to_spec(sc).to_bytes()
        hi = H.power_range(blob)
        thr = sc["power_cap"] if sc.get("power_cap", 0) > 0 else hi / 4
        got = H.run_batch(blob, 2, c["run"]["seed"], threshold=thr)
        assert np.all(got["summary"][:, S.S_STATUS] == 0), sc["name"]
        check_identities(got["rows"], got["summary"], hi, sc["n_dc"], sc["name"])


def test_one_level_profile_carries_the_reference_energy():
    """all_off has one constant idle level: its power times profile_s is the reference's total energy (the generator
    checks sum of level power x length against it for every fixture)."""
    doc = load("all_off_2x8")
    for case in doc["cases"]:
        got = run_case(doc, case)
        peak, prof = got["rows"][S.PP_PEAK_W, 0], got["rows"][S.PP_PROFILE_S, 0]
        e = float.fromhex(case["total_energy_j"])
        assert abs(peak * prof - e) <= 1e-12 * e


def brute_force_stats(rows, good, qs):
    x = rows[:, good]
    out = {"n": np.full(rows.shape[0], x.shape[1]), "sum": x.sum(axis=1), "min": x.min(axis=1), "max": x.max(axis=1)}
    out["std"] = x.std(axis=1, ddof=1)
    out["q"] = np.quantile(x, qs, axis=1, method="inverted_cdf")
    return out


def test_numpy_mirror_matches_brute_force():
    blob = SC.to_spec(SC.BY_NAME["ragged_3dc_12_5_40"]).to_bytes()
    n_dc, R = 3, 40
    hi = H.power_range(blob)
    got = H.run_batch(blob, R, 500, threshold=6000.0)
    rows, summary = got["rows"], got["summary"].copy()
    summary[[3, 17], S.S_STATUS] = 4.0                  # two replicas left out
    good = summary[:, S.S_STATUS] == 0
    res = E.power_profile_from_rows(rows, summary, hi, 6000.0)
    ref = brute_force_stats(rows[:NF + n_dc], good, res.q)
    c = NF + n_dc
    assert np.array_equal(res.n, ref["n"][:c]) and np.array_equal(res.min, ref["min"]) and np.array_equal(res.max, ref["max"])
    assert np.allclose(res.mean, ref["sum"] / good.sum(), rtol=1e-12)
    assert np.allclose(res.std, ref["std"], rtol=1e-9)
    for i in (S.PP_EXCURSIONS, S.PP_OUT_OF_RANGE):       # unit bins: exact quantiles
        assert np.array_equal(res.quantiles[:, i], ref["q"][:, i])
    width = E.bin_widths_for(res.min, res.max, E._pp_integral(c))
    assert np.all(np.abs(res.quantiles - ref["q"]) <= width[None, :] + 1e-9)
    curve = rows[c:, good].sum(axis=1)
    assert np.allclose(res.duration_curve[1], curve, rtol=1e-12, atol=0)
    assert np.allclose(res.pooled_time_s, rows[S.PP_PROFILE_S, good].sum(), rtol=1e-12)
    energy = summary[good, S.S_TOTAL_ENERGY_J].sum()
    assert res.mean_power_w == pytest.approx(energy / rows[S.PP_PROFILE_S, good].sum(), rel=1e-12)
    # power levels exceeded for a share of the time: within one bin width of the exact answer from the sorted bins
    edges = res.duration_curve[0]
    for share, level in zip((0.5, 0.1, 0.01), res.time_quantiles([0.5, 0.1, 0.01])):
        above = curve[edges[:-1] >= level - (edges[1] - edges[0])].sum()
        assert above >= share * curve.sum() * (1 - 1e-12)
    assert 0.0 <= res.over_share <= 1.0


def test_csv_layout(tmp_path):
    blob = SC.to_spec(SC.BY_NAME["eco_route_cap_2x16"]).to_bytes()
    got = H.run_batch(blob, 8, 7, threshold=1000.0)
    hi = H.power_range(blob)
    for thr in (1000.0, None):
        res = E.power_profile_from_rows(got["rows"], got["summary"], hi, thr)
        p = tmp_path / "pp.csv"
        res.to_csv(str(p), ["dc-a", "dc-b"])
        lines = p.read_text().splitlines()
        assert lines[0] == "dc,field,n,mean,std,min,p05,p25,p50,p75,p95,p99,max"
        body = [ln.split(",") for ln in lines[1:]]
        assert [r[1] for r in body] == list(E.PP_FIELDS) + ["dc_peak_w", "dc_peak_w", "power_w_time"]
        assert [r[0] for r in body[NF:NF + 2]] == ["dc-a", "dc-b"]
        over = body[E.PP_FIELDS.index("over_s")]
        assert (over[2] == "") == (thr is None)
        last = body[-1]
        assert last[2] == "8" and last[4] == "" and float(last[3]) == pytest.approx(res.mean_power_w)
        assert all(float(a) <= float(b) for a, b in zip(last[6:12], last[7:13]))


def test_abi_constants_agree():
    hdr = open(os.path.join(os.path.dirname(POWER_DIR), "..", "..", "include", "dcsim_b200.h")).read()
    assert "#define DCSIM_PP_BINS 1024" in hdr and "DCSIM_PP_FIELDS = 8" in hdr
    assert S.PP_BINS == E.PP_BINS == H.PP_BINS == 1024 and S.PP_FIELDS == len(E.PP_FIELDS) == H.PP_FIELDS


def test_cli_flags_and_compare_refusal():
    from distributed_cluster_gpus_b200 import run_sim_paper as R
    a = R.parse_args(["--power-profile-csv", "p.csv"])
    assert a.power_profile_csv == "p.csv" and R.power_threshold(a) is None
    assert R.power_threshold(R.parse_args(["--power-cap", "20000"])) == 20000.0
    assert R.power_threshold(R.parse_args(["--power-cap", "20000", "--power-threshold", "15000"])) == 15000.0
    for extra in (["--power-profile-csv", "p.csv"], ["--power-threshold", "100"]):
        with pytest.raises(SystemExit) as ei:
            R.main(["--compare-algos", "default_policy,cap_greedy"] + extra)
        assert "--power-profile-csv" in str(ei.value)
