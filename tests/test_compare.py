"""Policy comparisons on the CPU: the rule that lets batches share one arrival pre-pass (dcsim_arrival_inputs_equal)
against the lists the host build of the device source draws, the event loop of one spec on lists drawn under another
against the oracle and the reference's numbers, the numpy mirror of the paired reductions against numpy, its two-rank
all-reduce (gloo) against one rank, and the CSV."""
import csv
import ctypes as C
import itertools
import os
import sys

import numpy as np
import pytest
import torch.distributed as dist
import torch.multiprocessing as mp

import hostemu_pair_lib as HP
from conftest import ROOT, load_golden
from distributed_cluster_gpus_b200 import compare as CP, ensemble as EN, scenarios as SC, spec as S

SWEEP = ["sweep_default_energy_aware", "sweep_default_perf_first", "sweep_joint_nf", "sweep_carbon_cost", "sweep_debug_n2",
         "sweep_debug_n8_f08", "sweep_bandit"]
BASE = "sweep_default_energy_aware"


def _hand_picked():
    """Variants of the sweep scenario that change only what the event loop reads."""
    sc = SC.BY_NAME[BASE]
    return [SC.BY_NAME["cap_greedy_4x64"], dict(sc, name="cap_uniform_cap", algo="cap_uniform", power_cap=15000.0),
            dict(sc, name="debug_n4_f05", algo="debug", num_fixed_gpus=4, fixed_freq=0.5),
            dict(sc, name="perf_first_freq8", policy="perf_first", freq_levels=SC.FREQ8),
            dict(sc, name="carbon_cap", algo="carbon_cost", power_cap=9000.0)]


def _random_variants(n, seed):
    rnd = np.random.default_rng(seed)
    algos = ["default_policy", "joint_nf", "carbon_cost", "debug", "bandit", "cap_uniform", "cap_greedy"]
    out = []
    for i in range(n):
        algo = str(rnd.choice(algos))
        out.append(dict(SC.BY_NAME[BASE], name=f"random_{i}", algo=algo, policy=str(rnd.choice(["energy_aware", "perf_first"])),
                        power_cap=float(rnd.choice([0.0, 8000.0, 20000.0])) if algo.startswith("cap") else 0.0,
                        num_fixed_gpus=int(rnd.integers(1, 9)), fixed_freq=[None, 0.5, 0.8][int(rnd.integers(0, 3))],
                        freq_levels=[SC.FREQ3, SC.FREQ8][int(rnd.integers(0, 2))]))
    return out


OTHER_CAPS = {"cap_run": 9, "cap_q_inf": 7000, "cap_q_trn": 300, "cap_stale": 99, "cap_xfer": 40}


def _same_lists(a, b, n, seed, rng_kind=0):
    la, ha = HP.lists(a, n, seed, rng_kind)
    lb, hb = HP.lists(b, n, seed, rng_kind)
    if ha.tobytes() != hb.tobytes():
        return False
    return all(x.tobytes() == y.tobytes() for ra, rb in zip(la, lb) for x, y in zip(ra, rb))


@pytest.mark.parametrize("seed", load_golden(BASE)["meta"]["philox_seeds"])
def test_compatible_specs_draw_byte_identical_lists(seed):
    """Every pair the rule accepts has byte-identical lists and headers; the sweep, the hand-picked and the random
    variants are all accepted against each other (they differ in algo, policy, power cap, num_fixed_gpus, fixed_freq,
    the frequency ladder)."""
    specs = [SC.to_spec(SC.BY_NAME[k]).to_bytes() for k in SWEEP]
    specs += [SC.to_spec(sc).to_bytes() for sc in _hand_picked() + _random_variants(4, seed % 1000)]
    specs.append(SC.to_spec(SC.BY_NAME["sweep_joint_nf"], caps=OTHER_CAPS).to_bytes())   # other capacities, the same ring
    for a, b in itertools.combinations(specs, 2):
        eq, field = HP.compatible(a, b)
        assert eq and field == "", field
    ref_lists, ref_hdr = HP.lists(specs[0], 3, seed)
    assert np.all(ref_hdr["status"] == 0) and np.all(ref_hdr["ml_count"] > 0)
    for b in specs[1:]:
        assert _same_lists(specs[0], b, 3, seed)


def test_mersenne_twister_lists_are_shared_too():
    a = SC.to_spec(SC.BY_NAME[BASE]).to_bytes()
    b = SC.to_spec(SC.BY_NAME["cap_greedy_4x64"]).to_bytes()
    assert HP.compatible(a, b)[0] and _same_lists(a, b, 2, 123, rng_kind=1)


def test_eco_route_is_rejected_and_its_lists_differ():
    eco = SC.to_spec(SC.BY_NAME["sweep_eco_route"]).to_bytes()
    base = SC.to_spec(SC.BY_NAME[BASE]).to_bytes()
    eq, field = HP.compatible(base, eco)
    assert not eq and field == "route_rule"
    assert not _same_lists(base, eco, 2, 123)


def test_smaller_seq_ring_is_rejected_and_flagged_like_its_standalone_batch():
    """The merge flags an xfer overflow in the list header when a transfer lies further ahead than the seq ring holds: a
    spec whose cap_xfer implies another ring gets other headers, so it is not compatible (and a member on the owner's
    lists would run unflagged).  Its own run flags the overflow."""
    base = SC.to_spec(SC.BY_NAME[BASE]).to_bytes()
    small = SC.to_spec(SC.BY_NAME["sweep_joint_nf"], caps={"cap_xfer": 1}).to_bytes()
    eq, field = HP.compatible(base, small)
    assert not eq and field == "cap_xfer"
    _, h_base = HP.lists(base, 3, 123)
    _, h_small = HP.lists(small, 3, 123)
    assert np.all(h_base["status"] == 0) and np.all(h_small["status"] & S.ST_XFER_OVERFLOW)
    assert np.array_equal(h_base["max_ahead"], h_small["max_ahead"])
    assert np.all(HP.run(small, small, 3, 123)["summary"][:, S.S_STATUS].astype(int) & S.ST_XFER_OVERFLOW)
    with pytest.raises(ValueError):
        HP.run(base, small, 3, 123)


def _with(spec, mutate):
    sp = S.Spec.from_buffer_copy(spec.to_bytes())
    mutate(sp)
    return sp


LISTED = {
    "arr[0].rate": lambda s: setattr(s.arr[0], "rate", s.arr[0].rate * 1.5),
    "arr[0].amp": lambda s: setattr(s.arr[0], "amp", 0.3),
    "arr[0].period": lambda s: setattr(s.arr[0], "period", 1800.0),
    "arr[1].mode": lambda s: setattr(s.arr[1], "mode", 2),
    "arr[1].rate": lambda s: setattr(s.arr[1], "rate", 0.5),
    "n_ing": lambda s: setattr(s, "n_ing", s.n_ing - 1),
    "n_dc": lambda s: setattr(s, "n_dc", s.n_dc - 1),
    "end_time": lambda s: setattr(s, "end_time", s.end_time + 1.0),
    "pareto_xm": lambda s: setattr(s, "pareto_xm", s.pareto_xm * 2),
    "pareto_inv_alpha": lambda s: setattr(s, "pareto_inv_alpha", s.pareto_inv_alpha * 2),
    "lognorm_mu": lambda s: setattr(s, "lognorm_mu", s.lognorm_mu + 0.1),
    "lognorm_sigma": lambda s: setattr(s, "lognorm_sigma", s.lognorm_sigma + 0.1),
    "lognorm_floor": lambda s: setattr(s, "lognorm_floor", s.lognorm_floor * 2),
    "uniform_floor": lambda s: setattr(s, "uniform_floor", s.uniform_floor * 2),
    "nv_magicconst": lambda s: setattr(s, "nv_magicconst", np.nextafter(s.nv_magicconst, 2.0)),
    "two_pi": lambda s: setattr(s, "two_pi", np.nextafter(s.two_pi, 7.0)),
    "transfer_s": lambda s: s.transfer_s[1][2].__setitem__(0, s.transfer_s[1][2][0] + 0.01),
    "route_rule": lambda s: setattr(s, "route_rule", S.ROUTE_ECO),
    "cap_arrivals": lambda s: setattr(s, "cap_arrivals", s.cap_arrivals + 1),
    "cap_xfer": lambda s: setattr(s, "cap_xfer", s.cap_xfer * 2),   # twice the seq ring the merge checks against
}

UNLISTED = {
    "algo": lambda s: setattr(s, "algo", S.ALGO_IDS["joint_nf"]),
    "policy_name": lambda s: setattr(s, "policy_name", 1),
    "power_cap": lambda s: setattr(s, "power_cap", 1234.0),
    "cap_run": lambda s: setattr(s, "cap_run", s.cap_run + 3),
    "cap_q_inf": lambda s: setattr(s, "cap_q_inf", s.cap_q_inf * 2),
    "cap_xfer (the same seq ring)": lambda s: setattr(s, "cap_xfer", s.cap_xfer + 7),     # 48 -> 55: 128 entries either way
    "cap_stale": lambda s: setattr(s, "cap_stale", 77),
    "log_interval": lambda s: setattr(s, "log_interval", 2.0),
    "dvfs_low": lambda s: setattr(s, "dvfs_low", 0.1),
    "num_fixed_gpus": lambda s: setattr(s, "num_fixed_gpus", 5),
    "fixed_freq": lambda s: setattr(s, "fixed_freq", 0.8),
    "price_kwh": lambda s: s.dc[0].price_kwh.__setitem__(3, 9.0),
    "carbon_intensity": lambda s: setattr(s.dc[1], "carbon_intensity", 999.0),
    "coeffs": lambda s: setattr(s.dc[0].coeffs[1], "alpha_t", 3.0),
    "total_gpus": lambda s: setattr(s.dc[2], "total_gpus", 7),
    "freq_levels": lambda s: s.dc[0].freq_levels.__setitem__(0, 0.4),
    "nf_tables": lambda s: setattr(s.dc[0].nf_xfer[0][5], "n", 3),
    "eco_e_unit (random routing)": lambda s: s.dc[0].eco_e_unit.__setitem__(0, 1.0),
    "net_lat_s": lambda s: s.net_lat_s[0].__setitem__(1, 0.5),
}


@pytest.mark.parametrize("field", sorted(LISTED))
def test_each_listed_field_flips_the_answer(field):
    base = SC.to_spec(SC.BY_NAME[BASE])
    other = _with(base, LISTED[field])
    eq, named = HP.compatible(base.to_bytes(), bytes(other))
    assert not eq and named == field
    assert HP.compatible(bytes(other), bytes(other))[0]


@pytest.mark.parametrize("field", sorted(UNLISTED))
def test_unlisted_fields_do_not(field):
    base = SC.to_spec(SC.BY_NAME[BASE])
    assert HP.compatible(base.to_bytes(), bytes(_with(base, UNLISTED[field])))[0]


def test_eco_e_unit_counts_only_when_both_route_eco():
    eco = SC.to_spec(SC.BY_NAME["sweep_eco_route"])
    eq, field = HP.compatible(eco.to_bytes(), bytes(_with(eco, lambda s: s.dc[3].eco_e_unit.__setitem__(1, 1e-3))))
    assert not eq and field == "eco_e_unit"
    assert HP.compatible(eco.to_bytes(), bytes(_with(eco, lambda s: setattr(s, "algo", S.ALGO_IDS["default_policy"]))))[0]


def test_library_gives_the_host_builds_answers():
    from distributed_cluster_gpus_b200 import _native as N
    from distributed_cluster_gpus_b200.engine import arrivals_compatible
    base = SC.to_spec(SC.BY_NAME[BASE])
    others = [SC.to_spec(SC.BY_NAME[k]) for k in SWEEP + ["sweep_eco_route", "cap_greedy_4x64", "cfg3_4x64_sinusoid_120s"]]
    others += [_with(base, f) for f in list(LISTED.values()) + list(UNLISTED.values())]
    for o in others:
        assert arrivals_compatible(base, o) == HP.compatible(base.to_bytes(), bytes(o))[0]
    lib = N.load()
    eq = C.c_int(7)
    blob = base.to_bytes()
    assert lib.dcsim_arrivals_compatible(blob, len(blob) - 1, blob, len(blob), C.byref(eq)) == N.E_INVALID
    bad = bytearray(blob)
    bad[:8] = b"\0" * 8                                   # magic
    assert lib.dcsim_arrivals_compatible(blob, len(blob), bytes(bad), len(blob), C.byref(eq)) == N.E_INVALID


PINNED = [("sweep_joint_nf", BASE), ("sweep_bandit", "sweep_debug_n2"), ("cap_greedy_4x64", BASE),
          ("sweep_default_perf_first", "cap_greedy_4x64")]


@pytest.mark.parametrize("mode", ["one_shot", "chunks61", "uniform"])
@pytest.mark.parametrize("variant,owner", PINNED)
def test_variant_on_the_owners_lists_equals_oracle_and_reference(oracle, variant, owner, mode):
    """The event loop of the variant on lists drawn under the owner's spec: the oracle's own run of the variant (every
    count exact, every float bit-identical) and the reference's numbers of the variant's fixture."""
    from test_oracle_vs_reference import check_row_against_golden
    doc = load_golden(variant)
    sp_v, sp_o = SC.to_spec(doc["scenario"]).to_bytes(), SC.to_spec(SC.BY_NAME[owner]).to_bytes()
    kw = {"chunk_events": 61} if mode == "chunks61" else ({"uniform": True} if mode == "uniform" else {})
    for run in (r for r in doc["runs"] if r["rng"] == "philox"):
        got = HP.run(sp_o, sp_v, 1, run["seed"], **kw)
        want, events = oracle.run_batch(sp_v, 1, run["seed"])
        assert got["events"] == events
        assert np.array_equal(got["summary"][:, :S.S_MAX_XFER], want[:, :S.S_MAX_XFER])
        assert np.array_equal(got["summary"][:, S.S_UTIL_BEGIN:], want[:, S.S_UTIL_BEGIN:])
        check_row_against_golden(got["summary"][0], run, doc["scenario"]["n_dc"], [])


def test_variant_on_the_owners_lists_mersenne_twister(oracle):
    from test_oracle_vs_reference import check_row_against_golden
    doc = load_golden("sweep_carbon_cost")
    run = [r for r in doc["runs"] if r["rng"] == "mt"][0]
    sp_v, sp_o = SC.to_spec(doc["scenario"]).to_bytes(), SC.to_spec(SC.BY_NAME["sweep_bandit"]).to_bytes()
    got = HP.run(sp_o, sp_v, 1, run["seed"], chunk_events=61, rng_kind=1)
    want, events = oracle.run_batch(sp_v, 1, run["seed"], rng_kind=1)
    assert got["events"] == events == run["events"]
    assert np.array_equal(got["summary"][:, :S.S_MAX_XFER], want[:, :S.S_MAX_XFER])
    check_row_against_golden(got["summary"][0], run, doc["scenario"]["n_dc"], [])


def test_incompatible_pair_is_refused_by_the_host_run():
    with pytest.raises(ValueError):
        HP.run(SC.to_spec(SC.BY_NAME[BASE]).to_bytes(), SC.to_spec(SC.BY_NAME["sweep_eco_route"]).to_bytes(), 1, 5)


# ---- the numpy mirror of the paired reductions ------------------------------------------------------------------------
def _oracle_pair(oracle, n, first, duration=40.0, variant="sweep_joint_nf"):
    base, _ = oracle.run_batch(SC.to_spec(dict(SC.BY_NAME[BASE], duration=duration)).to_bytes(), n, 900, first)
    var, _ = oracle.run_batch(SC.to_spec(dict(SC.BY_NAME[variant], duration=duration)).to_bytes(), n, 900, first)
    return base, var


def _direct(base, var, n_dc):
    """Per metric: (values of base, of variant, defined) straight from the summary columns."""
    def vals(s):
        fin, fi, ft = s[:, S.S_JOBS_FINISHED], s[:, S.S_FIN_INF], s[:, S.S_FIN_TRN]
        g = [s[:, S.S_DC0 + d * S.S_DC_STRIDE:S.S_DC0 + (d + 1) * S.S_DC_STRIDE] for d in range(n_dc)]
        with np.errstate(invalid="ignore", divide="ignore"):
            v = [s[:, S.S_TOTAL_ENERGY_J], s[:, S.S_TOTAL_ENERGY_J] / fin, fi, ft, s[:, S.S_LAT_SUM_INF] / fi,
                 s[:, S.S_LAT_SUM_TRN] / ft, sum(x[:, S.SD_Q_INF] + x[:, S.SD_Q_TRN] + x[:, S.SD_RUNNING] for x in g)]
        ok = [fin == fin, fin > 0, fin == fin, fin == fin, fi > 0, ft > 0, fin == fin]
        return v + [x[:, S.SD_ENERGY_J] for x in g], ok + [fin == fin] * n_dc
    vb, okb = vals(base)
    vv, okv = vals(var)
    good = (base[:, S.S_STATUS] == 0) & (var[:, S.S_STATUS] == 0)
    return [(b, v, good & ob & ov) for b, v, ob, ov in zip(vb, vv, okb, okv)]


def numpy_pair_check(st, base, var, n_dc, quantiles=EN.DEFAULT_QUANTILES):
    for i, (b, v, ok) in enumerate(_direct(base, var, n_dc)):
        b, v = b[ok], v[ok]
        d = v - b
        assert st.n[i] == ok.sum()
        if not ok.any():
            assert np.isnan(st.diff_mean[i])
            continue
        assert st.frac_lower[i] == np.sum(v < b) / st.n[i] and st.frac_higher[i] == np.sum(v > b) / st.n[i]
        np.testing.assert_allclose([st.base_mean[i], st.variant_mean[i], st.diff_mean[i]], [b.mean(), v.mean(), d.mean()],
                                   rtol=1e-12, atol=1e-12 * max(1.0, np.abs(b).max()))
        if d.size > 1:
            np.testing.assert_allclose(st.diff_std[i], d.std(ddof=1), rtol=1e-12, atol=1e-12 * max(1.0, np.abs(b).max()))
            vb, vv, vd = b.var(ddof=1), v.var(ddof=1), d.var(ddof=1)
            if vb + vv > 0:
                np.testing.assert_allclose(st.var_ratio[i], vd / (vb + vv), rtol=1e-9)
            half = 1.96 * d.std(ddof=1) / np.sqrt(d.size)
            np.testing.assert_allclose([st.diff_ci95_lo[i], st.diff_ci95_hi[i]], [d.mean() - half, d.mean() + half],
                                       rtol=1e-9, atol=1e-12 * max(1.0, np.abs(b).max()))
        np.testing.assert_allclose(st.rel_change[i], v.mean() / b.mean() - 1.0, rtol=1e-9, atol=1e-15)
        integral = i in CP.INTEGER_METRICS
        for j, q in enumerate(quantiles):
            want = np.quantile(d, q, method="inverted_cdf")
            if integral and d.max() - d.min() + 1 <= EN.BINS:
                assert st.diff_quantiles[j, i] == want, (i, q)
            else:
                assert abs(st.diff_quantiles[j, i] - want) <= (d.max() - d.min()) / EN.BINS * (1 + 1e-12) + (1.0 if integral else 0.0)


def test_host_mirror_equals_numpy(oracle):
    base, var = _oracle_pair(oracle, 24, 50)
    var[[4, 9], S.S_STATUS] = S.ST_QUEUE_OVERFLOW        # two replicas that stopped: left out of every column
    base[[9, 17], S.S_STATUS] = S.ST_RUN_OVERFLOW
    st = CP.paired_from_summaries(base, var)
    assert st.metrics == CP.metric_names(4) and st.n[0] == 21
    numpy_pair_check(st, base, var, 4)
    assert np.any(st.frac_lower > 0) and np.any(st.var_ratio < 1.0)


def test_delta_method_ci_of_the_relative_change():
    rnd = np.random.default_rng(3)
    base = np.zeros((400, S.SUMMARY_K))
    base[:, S.S_TOTAL_ENERGY_J] = rnd.normal(1000.0, 50.0, 400)
    var = base.copy()
    var[:, S.S_TOTAL_ENERGY_J] = 0.9 * base[:, S.S_TOTAL_ENERGY_J] + rnd.normal(0.0, 5.0, 400)
    base[:, S.S_DC0 + S.SD_CURRENT_FREQ] = var[:, S.S_DC0 + S.SD_CURRENT_FREQ] = 1.0
    st = CP.paired_from_summaries(base, var)
    b, v = base[:, S.S_TOTAL_ENERGY_J], var[:, S.S_TOTAL_ENERGY_J]
    mb, mv, n = b.mean(), v.mean(), b.size
    cov = np.cov(b, v, ddof=1)[0, 1]
    se = np.sqrt((v.var(ddof=1) / mb ** 2 - 2 * mv * cov / mb ** 3 + mv ** 2 * b.var(ddof=1) / mb ** 4) / n)
    np.testing.assert_allclose([st.rel_ci95_lo[0], st.rel_ci95_hi[0]], [mv / mb - 1 - 1.96 * se, mv / mb - 1 + 1.96 * se], rtol=1e-9)
    assert st.var_ratio[0] < 0.05 and st.frac_lower[0] == 1.0 and st.n[0] == 400


def _comparison(st, shared=True):
    return CP.PairedComparison(baseline="default_policy", variants=("joint_nf",), n_dc=4, stats={"joint_nf": st},
                               shared_arrivals={"joint_nf": shared}, summaries={})


def test_to_csv_header_and_rows(tmp_path, oracle):
    base, var = _oracle_pair(oracle, 6, 10, duration=20.0)
    p = tmp_path / "cmp.csv"
    _comparison(CP.paired_from_summaries(base, var)).to_csv(str(p), ["a", "b", "c", "d"])
    with open(p) as f:
        rows = list(csv.reader(f))
    assert ",".join(rows[0]) == ("variant,baseline,metric,dc,n,base_mean,variant_mean,diff_mean,diff_std,diff_ci95_lo,"
                                 "diff_ci95_hi,rel_change,rel_ci95_lo,rel_ci95_hi,frac_lower,frac_higher,diff_p05,diff_p25,"
                                 "diff_p50,diff_p75,diff_p95,var_ratio,shared_arrivals")
    assert len(rows) == 1 + len(CP.METRICS) + 4
    assert [r[2] for r in rows[1:]] == list(CP.METRICS) + ["dc_energy_j"] * 4
    assert [r[3] for r in rows[1:]] == [""] * len(CP.METRICS) + ["a", "b", "c", "d"]
    assert all(r[0] == "joint_nf" and r[1] == "default_policy" and r[-1] == "True" for r in rows[1:])
    assert rows[1][4] == "6" and all(int(r[4]) <= 6 for r in rows[1:])


def _gloo_worker(rank, world, port, n_total, out_path):
    for p in (ROOT, os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests")):
        if p not in sys.path:
            sys.path.insert(0, p)
    import oracle_lib
    from distributed_cluster_gpus_b200 import sharding
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        first, count = sharding.shard(n_total, rank, world)
        base, var = _oracle_pair(oracle_lib, count, first, duration=30.0)
        st = CP.paired_from_summaries(base, var)
        if rank == 0:
            np.savez(out_path, **{k: getattr(st, k) for k in ("n", "base_mean", "variant_mean", "diff_mean", "diff_std",
                                                              "frac_lower", "frac_higher", "diff_quantiles", "hist")})
    finally:
        dist.destroy_process_group()


def test_two_rank_gloo_matches_one_rank(tmp_path, oracle):
    n_total = 13
    out = str(tmp_path / "pair.npz")
    mp.spawn(_gloo_worker, args=(2, 29500 + (os.getpid() + 1733) % 2000, n_total, out), nprocs=2, join=True)
    got = np.load(out)
    base, var = _oracle_pair(oracle, n_total, 0, duration=30.0)
    one = CP.paired_from_summaries(base, var)
    for k in ("n", "frac_lower", "frac_higher", "diff_quantiles", "hist"):
        assert np.array_equal(got[k], getattr(one, k), equal_nan=True), k
    for k in ("base_mean", "variant_mean", "diff_mean"):
        np.testing.assert_allclose(got[k], getattr(one, k), rtol=1e-12)
    np.testing.assert_allclose(got["diff_std"], one.diff_std, rtol=1e-12, atol=1e-12 * np.nanmax(np.abs(one.base_mean)))
