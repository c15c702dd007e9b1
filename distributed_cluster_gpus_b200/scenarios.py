"""Named synthetic scenarios (SURVEY.md §8(d)) shared by the golden generator, the parity tests and bench.py.

A scenario is a plain JSON-able dict; ``to_spec`` expands it through the package's own builders and flattening
(the golden fixtures under tests/golden/ were produced by feeding the SAME dicts to the unmodified reference,
so they pin builders + flattening against it).
"""
from . import spec as _spec
from .configs import paper_config as _pc
from .simcore.arrivals import ArrivalConfig

FREQ8 = [0.3, 0.4, 0.5, 0.6, 0.7, 0.8, 0.9, 1.0]
FREQ3 = [0.5, 0.8, 1.0]
SIN10 = dict(mode="sinusoid", rate=10.0, amp=0.6, period=3600.0)
SIN6 = dict(mode="sinusoid", rate=6.0, amp=0.6, period=3600.0)
POI = lambda r: dict(mode="poisson", rate=float(r), amp=0.0, period=3600.0)  # noqa: E731
OFF = dict(mode="off", rate=0.0, amp=0.0, period=3600.0)
ZERO_WAN = dict(latency_ms=0.0, capacity_gbps=0.0)
SLOW_WAN = dict(capacity_gbps=1.0)


def scenario(name, n_dc, gpus_per_dc, inf, trn, duration, freq_levels=None, algo="default_policy",
             policy="energy_aware", log_interval=5.0, power_cap=0.0, num_fixed_gpus=1, fixed_freq=None,
             gpus_list=None, wan=None, energy_price=None):
    sc = {"name": name, "n_dc": n_dc, "gpus_per_dc": gpus_per_dc, "gpus_list": gpus_list,
          "freq_levels": list(freq_levels or FREQ8), "inf": dict(inf), "trn": dict(trn),
          "duration": float(duration), "algo": algo, "policy": policy, "log_interval": float(log_interval),
          "power_cap": float(power_cap), "num_fixed_gpus": int(num_fixed_gpus), "fixed_freq": fixed_freq}
    if wan is not None:   # only when given: every scenario without it keeps the reference's own WAN (and its fixture)
        sc["wan"] = {k: float(v) for k, v in wan.items()}
    if energy_price is not None:  # a per-DC tariff {dc: {hour: USD/kWh}} in place of paper_config's; hours as strings (JSON)
        sc["energy_price"] = {dc: {str(h): float(p) for h, p in hours.items()} for dc, hours in energy_price.items()}
    return sc


def energy_price_of(sc):
    """The tariff a scenario runs under: its own per-DC map (SIM:986-1005's {dc: {hour: price}} form) or paper_config's."""
    if "energy_price" not in sc:
        return _pc.build_energy_price()
    return {dc: {int(h): float(p) for h, p in hours.items()} for dc, hours in sc["energy_price"].items()}


# BASELINE.json configs, with the durations fixed once here (SURVEY.md §8(d) caveat iii)
CFG1 = scenario("cfg1_1x4_poisson_5000s", 1, 4, POI(1.0), OFF, 5000.0)
CFG2 = scenario("cfg2_1x64_poisson_600s", 1, 64, POI(10.0), POI(1.0), 600.0)
CFG3 = scenario("cfg3_4x64_sinusoid_120s", 4, 64, SIN10, POI(1.0), 120.0)
CFG3_LONG = scenario("cfg3_4x64_sinusoid_600s", 4, 64, SIN10, POI(1.0), 600.0)
CFG5 = scenario("cfg5_8x256_sinusoid_60s", 8, 256, SIN10, dict(mode="sinusoid", rate=1.0, amp=0.0, period=3600.0), 60.0)

GOLDEN_SCENARIOS = [
    CFG1, CFG2, CFG3, CFG3_LONG, CFG5,
    scenario("kat_4x64_sin6_600s", 4, 64, SIN6, POI(0.3), 600.0),
    scenario("kat_8x256_sin10_poitrn_60s", 8, 256, SIN10, POI(1.0), 60.0),
    # policy sweep (cfg 4)
    scenario("sweep_default_energy_aware", 4, 64, SIN10, POI(1.0), 120.0, FREQ3),
    scenario("sweep_default_perf_first", 4, 64, SIN10, POI(1.0), 120.0, FREQ3, policy="perf_first"),
    scenario("sweep_joint_nf", 4, 64, SIN10, POI(1.0), 120.0, FREQ3, algo="joint_nf"),
    scenario("sweep_carbon_cost", 4, 64, SIN10, POI(1.0), 120.0, FREQ3, algo="carbon_cost"),
    scenario("sweep_eco_route", 4, 64, SIN10, POI(1.0), 120.0, FREQ3, algo="eco_route"),
    scenario("sweep_debug_n2", 4, 64, SIN10, POI(1.0), 120.0, FREQ3, algo="debug", num_fixed_gpus=2),
    scenario("sweep_debug_n8_f08", 4, 64, SIN10, POI(1.0), 120.0, FREQ3, algo="debug", num_fixed_gpus=8, fixed_freq=0.8),
    scenario("sweep_bandit", 4, 64, SIN10, POI(1.0), 120.0, FREQ3, algo="bandit"),
    # cold rows / edges
    scenario("cap_greedy_4x64", 4, 64, SIN10, POI(1.0), 120.0, FREQ8, algo="cap_greedy", power_cap=20000.0),
    scenario("cap_uniform_4x64", 4, 64, SIN10, POI(1.0), 60.0, FREQ8, algo="cap_uniform", power_cap=20000.0),
    scenario("eco_route_cap_2x16", 2, 16, POI(2.0), POI(0.2), 300.0, FREQ8, algo="eco_route", power_cap=1000.0),
    scenario("carbon_cost_8h_2x16", 2, 16, POI(0.02), POI(0.002), 30000.0, FREQ8, algo="carbon_cost", log_interval=600.0),
    scenario("ragged_3dc_12_5_40", 3, None, POI(3.0), POI(0.4), 200.0, FREQ8, gpus_list=[12, 5, 40]),
    scenario("trn_only_2x8", 2, 8, OFF, POI(0.5), 400.0, FREQ8),
    scenario("underloaded_1x64", 1, 64, POI(0.5), OFF, 600.0, FREQ8),
    scenario("all_off_2x8", 2, 8, OFF, OFF, 100.0, FREQ8),
    scenario("short_0p3s_4x64", 4, 64, SIN10, POI(1.0), 0.3, FREQ8),
    # |amp| > 1 is NOT a valid scenario: lambda(t) clips to 0 and the reference's non-advancing "thinning"
    # (arrivals.py:41-45) then never accepts — the reference spins for ever.  amp = 1.0 is the edge that still ends.
    scenario("full_swing_sinusoid_amp1", 2, 32, dict(mode="sinusoid", rate=4.0, amp=1.0, period=60.0), POI(0.3), 300.0, FREQ8),
    scenario("negative_amp_sinusoid", 2, 32, dict(mode="sinusoid", rate=4.0, amp=-0.5, period=45.0), dict(mode="sinusoid", rate=0.3, amp=0.3, period=100.0), 200.0, FREQ8),
    scenario("no_inf_priority_perf_first", 2, 16, POI(4.0), POI(0.5), 200.0, FREQ8, policy="perf_first"),
    # what `python run_sim_paper.py` runs with its own defaults (run_sim_paper.py:18-112, paper_config.py:39-64):
    # all 8 DCs with their own GPU counts, sinusoid inference 6/s amp 0.6 period 300 s, Poisson training 0.3/s, 180 s
    scenario("cli_defaults_8dc_180s", 8, None, dict(mode="sinusoid", rate=6.0, amp=0.6, period=300.0),
             dict(mode="poisson", rate=0.3, amp=0.0, period=3600.0), 180.0, FREQ8, gpus_list=[16, 32, 256, 16, 128, 16, 512, 512]),
    scenario("cli_defaults_8dc_joint_nf_60s", 8, None, dict(mode="sinusoid", rate=6.0, amp=0.6, period=300.0),
             dict(mode="poisson", rate=0.3, amp=0.0, period=3600.0), 60.0, FREQ8, algo="joint_nf", gpus_list=[16, 32, 256, 16, 128, 16, 512, 512]),
    # WAN overrides (paper_config.build_scenario `wan`).  Zero latency and no bandwidth term: transfer_s == 0, so every
    # arrival ties with the xfer_done it pushes at its own instant.  1 Gbps links: a training job's 5 GB
    # take 5 s (SIM:489), hundreds of arrivals lie within one max_transfer and the list merge leaves its shared-memory ring.
    scenario("zero_xfer_4x64_sin10_60s", 4, 64, SIN10, POI(1.0), 60.0, FREQ8, wan=ZERO_WAN),
    scenario("slow_wan_1g_4x64_sin10_60s", 4, 64, SIN10, POI(1.0), 60.0, FREQ8, wan=SLOW_WAN),
    scenario("zero_xfer_cap_greedy_4x64_60s", 4, 64, SIN10, POI(1.0), 60.0, FREQ8, algo="cap_greedy", power_cap=20000.0,
             wan=ZERO_WAN),
]
BY_NAME = {s["name"]: s for s in GOLDEN_SCENARIOS}

# scenarios whose reference-written CSV files are kept under tests/golden/csv/ (wire-format tests)
CSV_SCENARIOS = {
    "ragged_3dc_12_5_40": BY_NAME["ragged_3dc_12_5_40"],
    "csv_joint_nf_4x64_20s": scenario("csv_joint_nf_4x64_20s", 4, 64, SIN10, POI(1.0), 20.0, FREQ3, algo="joint_nf", log_interval=2.0),
    "csv_carbon_cost_2x16": scenario("csv_carbon_cost_2x16", 2, 16, POI(2.0), POI(0.1), 90.0, FREQ8, algo="carbon_cost"),
}


def build_inputs(sc):
    """Scenario -> kwargs of MultiIngressPaperSimulator / spec.flatten (product builders)."""
    ingresses, dcs, graph, coeffs = _pc.build_scenario(sc["n_dc"], sc["gpus_per_dc"], sc["freq_levels"], sc.get("gpus_list"),
                                                       sc.get("wan"))
    return dict(ingresses=ingresses, dcs=dcs, graph=graph, arrival_inf=ArrivalConfig(**sc["inf"]),
                arrival_train=ArrivalConfig(**sc["trn"]), coeffs_map=coeffs,
                carbon_intensity=_pc.build_carbon_intensity(), energy_price=energy_price_of(sc),
                policy=_pc.build_policy(name=sc["policy"]))


def to_spec(sc, caps=None):
    kw = build_inputs(sc)
    return _spec.flatten(kw["ingresses"], kw["dcs"], kw["graph"], kw["arrival_inf"], kw["arrival_train"],
                         kw["coeffs_map"], kw["policy"], carbon_intensity=kw["carbon_intensity"],
                         energy_price=kw["energy_price"], sim_duration=sc["duration"], log_interval=sc["log_interval"],
                         algo=sc["algo"], power_cap=sc["power_cap"], num_fixed_gpus=sc["num_fixed_gpus"],
                         fixed_freq=sc["fixed_freq"], caps=caps)
