"""Scenario constants and builders — drop-in for the reference's configs/paper_config.py.

Same builder names, arguments and return types (build_dcs :20, build_arrivals :67, build_policy :74,
build_paper_coeffs :81, build_ingresses_and_topology :182, build_carbon_intensity :280,
build_router_policy :289, build_energy_price :294, plus the single-DC debug pair build_dc :10 /
build_ingress_and_topology :171).  The numbers are the reference's scenario data; here they live in tables
that the builders expand, and ``build_scenario`` adds the (D, G) sub-setting rule of SURVEY.md §8(d) that the
reference CLI cannot express (run_sim_paper.py:119 hard-wires all 8 DCs).
"""
from typing import Dict, Iterable, Optional, Sequence

from ..simcore.arrivals import ArrivalConfig
from ..simcore.coeffs import TrainLatencyCoeffs, TrainPowerCoeffs
from ..simcore.models import DataCenter, GPUType
from ..simcore.network import Graph, Ingress
from ..simcore.policy import PolicyConfig
from ..simcore.router import RouterPolicy

FREQ_LEVELS_8 = (0.3, 0.4, 0.5, 0.6, 0.7, 0.8, 0.9, 1.0)

# name: (p_idle W, p_peak W, p_sleep W); alpha = 3.0 throughout
GPU_TABLE = {
    "A100-SXM4": (50.0, 400.0, 30.0), "A100-PCIe": (45.0, 300.0, 28.0),
    "H100-SXM5": (55.0, 700.0, 35.0), "H100-PCIe": (45.0, 350.0, 28.0),
    "H200-SXM": (60.0, 700.0, 38.0), "H200-PCIe": (55.0, 600.0, 35.0),
    "L4": (15.0, 72.0, 8.0), "T4": (10.0, 70.0, 6.0),
    "A10": (20.0, 150.0, 10.0), "A30": (25.0, 165.0, 12.0), "A40": (40.0, 300.0, 25.0),
    "L40": (35.0, 300.0, 20.0), "L40S": (40.0, 350.0, 25.0),
}

# DC name -> (GPU model, GPU count, region tag of its gateway); insertion order is the DC order everywhere
DC_TABLE = {
    "us-west": ("H100-PCIe", 16, "US"),
    "us-east": ("A100-PCIe", 32, "US"),
    "eu-west": ("L40S", 256, "EU"),
    "eu-central": ("H100-SXM5", 16, "EU"),
    "ap-southeast": ("L4", 128, "APAC"),
    "ap-northeast": ("H200-PCIe", 16, "APAC"),
    "sa-east": ("A30", 512, "SA"),
    "me-central": ("A10", 512, "ME"),
}

# DC -> {jtype: ((alpha_p, beta_p, gamma_p), (alpha_t, beta_t, gamma_t))}
COEFF_TABLE = {
    "us-west": {"training": ((75.0, 80.0, 110.0), (0.0045, 0.032, 0.0012)),
                "inference": ((95.0, 20.0, 97.0), (0.0090, 0.0018, 0.0007))},
    "us-east": {"training": ((65.0, 60.0, 90.0), (0.0050, 0.038, 0.0014)),
                "inference": ((85.0, 18.0, 80.0), (0.0080, 0.0020, 0.0009))},
    "eu-west": {"training": ((55.0, 40.0, 70.0), (0.0060, 0.045, 0.0018)),
                "inference": ((70.0, 15.0, 60.0), (0.0050, 0.020, 0.0010))},
    "eu-central": {"training": ((90.0, 85.0, 120.0), (0.0042, 0.030, 0.0011)),
                   "inference": ((100.0, 22.0, 100.0), (0.0085, 0.0017, 0.0007))},
    "ap-southeast": {"training": ((45.0, 20.0, 40.0), (0.0065, 0.060, 0.0022)),
                     "inference": ((40.0, 12.0, 35.0), (0.0045, 0.025, 0.0012))},
    "ap-northeast": {"training": ((95.0, 90.0, 125.0), (0.0040, 0.029, 0.0010)),
                     "inference": ((105.0, 25.0, 105.0), (0.0080, 0.0016, 0.0006))},
    "sa-east": {"training": ((50.0, 35.0, 65.0), (0.0062, 0.050, 0.0019)),
                "inference": ((65.0, 14.0, 55.0), (0.0055, 0.022, 0.0011))},
    "me-central": {"training": ((40.0, 25.0, 50.0), (0.0068, 0.055, 0.0023)),
                   "inference": ((55.0, 12.0, 45.0), (0.0050, 0.023, 0.0012))},
}

# gateway of DC x -> [(peer DC, one-way latency ms)], listed in the order the reference adds the edges.
# Every link is added gateway->DC then DC->gateway, except that gw-us-west -> eu-central is added twice
# forward before its return edge (paper_config.py:205-207); the duplicate is kept so the adjacency lists match.
WAN_TABLE = {
    "us-west": [("us-west", 12), ("us-east", 70), ("eu-central", 110), ("ap-southeast", 150)],
    "us-east": [("us-east", 10), ("us-west", 70), ("eu-west", 90), ("sa-east", 110)],
    "eu-west": [("eu-west", 10), ("eu-central", 20), ("us-east", 90), ("ap-northeast", 190)],
    "eu-central": [("eu-central", 10), ("me-central", 60), ("ap-southeast", 170)],
    "ap-southeast": [("ap-southeast", 8), ("ap-northeast", 60), ("eu-central", 170)],
    "ap-northeast": [("ap-northeast", 8), ("us-west", 130), ("eu-west", 190)],
    "sa-east": [("sa-east", 12), ("us-east", 110), ("eu-west", 150)],
    "me-central": [("me-central", 10), ("eu-central", 60), ("ap-southeast", 120)],
}
_DUPLICATED_FORWARD_EDGES = {("gw-us-west", "eu-central")}

CARBON_G_PER_KWH = {"us-west": 350.0, "eu-central": 220.0, "ap-southeast": 500.0}
PRICE_BANDS_USD_PER_KWH = ((0, 7, 0.12), (7, 19, 0.20), (19, 24, 0.16))  # [from hour, to hour) -> price


def _gpu(model: str) -> GPUType:
    p_idle, p_peak, p_sleep = GPU_TABLE[model]
    return GPUType(model, p_idle=p_idle, p_peak=p_peak, p_sleep=p_sleep, alpha=3.0)


def _datacenter(name: str, model: str, count: int, freq_levels: Sequence[float] = FREQ_LEVELS_8) -> DataCenter:
    return DataCenter(name, gpu_type=_gpu(model), total_gpus=count, freq_levels=list(freq_levels),
                      default_freq=1.0, power_gating=True)


def build_dc():
    """Single-DC debug scenario (reference :10-17)."""
    return {"us-west": _datacenter("us-west", "H100-PCIe", 128)}


def build_dcs():
    return {name: _datacenter(name, model, count) for name, (model, count, _) in DC_TABLE.items()}


def build_arrivals(inf_mode="sinusoid", inf_rate=6.0, inf_amp=0.6, inf_period=300.0,
                   trn_mode="poisson", trn_rate=0.3):
    # The training stream gets no amp/period (reference :70): a 'sinusoid' training stream is flat-rate.
    return (ArrivalConfig(mode=inf_mode, rate=inf_rate, amp=inf_amp, period=inf_period),
            ArrivalConfig(mode=trn_mode, rate=trn_rate))


def build_policy(name="energy_aware", max_gpus_per_job=8, inf_priority=True, dvfs_low=0.6, dvfs_high=1.0,
                 train_scale_out_low_freq=True, reserve_inf_gpus=0):
    return PolicyConfig(name=name, max_gpus_per_job=max_gpus_per_job, inf_priority=inf_priority,
                        dvfs_low=dvfs_low, dvfs_high=dvfs_high,
                        train_scale_out_low_freq=train_scale_out_low_freq, reserve_inf_gpus=reserve_inf_gpus)


def build_paper_coeffs(dcs) -> Dict[tuple, tuple]:
    """(dc name, jtype) -> (TrainPowerCoeffs, TrainLatencyCoeffs) for all eight DCs, like the reference."""
    table = {}
    for dc_name, per_type in COEFF_TABLE.items():
        for jtype in ("training", "inference"):
            power, latency = per_type[jtype]
            table[(dc_name, jtype)] = (TrainPowerCoeffs(*power), TrainLatencyCoeffs(*latency))
    return table


def build_ingress_and_topology():
    """Single-gateway debug topology (reference :171-180)."""
    g = Graph()
    g.add_edge("gw-us-west", "us-west", 12)
    g.add_edge("us-west", "gw-us-west", 12)
    return {"gw-us-west": Ingress("gw-us-west", region="US")}, g


def build_ingresses_and_topology():
    ingresses = {f"gw-{name}": Ingress(f"gw-{name}", region=region) for name, (_, _, region) in DC_TABLE.items()}
    g = Graph()
    for home, links in WAN_TABLE.items():
        gw = f"gw-{home}"
        for peer, ms in links:
            g.add_edge(gw, peer, ms)
            if (gw, peer) in _DUPLICATED_FORWARD_EDGES:
                g.add_edge(gw, peer, ms)
            g.add_edge(peer, gw, ms)
    return ingresses, g


def build_carbon_intensity():
    return dict(CARBON_G_PER_KWH)


def build_router_policy():
    return RouterPolicy(w_energy=1.0, w_latency=0.5, w_carbon=0.0, d_choices=0)


def build_energy_price():
    return {h: price for lo, hi, price in PRICE_BANDS_USD_PER_KWH for h in range(lo, hi)}


# Labels used by the reference's plot scripts
dc_gpus_dict = {name: f"{count} x {'H100-SXM' if model == 'H100-SXM5' else model}"
                for name, (model, count, _) in DC_TABLE.items()}
gw_alphabet_dict = dict(zip((f"gw-{n}" for n in ("us-west", "us-east", "eu-west", "eu-central", "ap-southeast",
                                                 "ap-northeast", "sa-east", "me-central")), "ABEFGHCD"))


def build_scenario(n_dc: int = 8, gpus_per_dc: Optional[int] = None, freq_levels: Optional[Iterable[float]] = None,
                   gpus_list: Optional[Sequence[int]] = None, wan: Optional[Dict[str, float]] = None):
    """The (D, G) sub-setting rule of SURVEY.md §8(d).

    Keeps the first ``n_dc`` DCs of build_dcs() (dict order) with their GPUType, overrides ``total_gpus``
    (``gpus_per_dc`` for all, or ``gpus_list`` per DC) and ``freq_levels``, keeps the gateways ``gw-<dc>`` of
    those DCs and the WAN edges with both endpoints kept.  Returns (ingresses, dcs, graph, coeffs_map).

    ``wan`` (optional) overrides every kept edge: ``latency_ms`` and/or ``capacity_gbps``.  A finite capacity adds
    payload / capacity to every transfer (SIM:487-495: 5 GB of training data over 1 Gbps is 5 s); latency 0 with
    capacity 0 (no bandwidth term) makes every transfer instantaneous, so each xfer_done falls on its arrival's instant.
    """
    wan = dict(wan or {})
    if set(wan) - {"latency_ms", "capacity_gbps"}:
        raise ValueError(f"wan: unknown keys {sorted(set(wan) - {'latency_ms', 'capacity_gbps'})}")
    if not 1 <= n_dc <= len(DC_TABLE):
        raise ValueError(f"n_dc must be in 1..{len(DC_TABLE)}")
    levels = list(freq_levels) if freq_levels is not None else list(FREQ_LEVELS_8)
    kept = list(DC_TABLE)[:n_dc]
    dcs = {}
    for i, name in enumerate(kept):
        model, count, _ = DC_TABLE[name]
        if gpus_list is not None:
            count = int(gpus_list[i])
        elif gpus_per_dc is not None:
            count = int(gpus_per_dc)
        dcs[name] = _datacenter(name, model, count, levels)
    all_ing, full = build_ingresses_and_topology()
    ingresses = {f"gw-{name}": all_ing[f"gw-{name}"] for name in kept}
    nodes = set(kept) | set(ingresses)
    graph = Graph()
    for u, edges in full.adj.items():
        if u in nodes:
            for e in edges:
                if e.to in nodes:
                    graph.add_edge(u, e.to, wan.get("latency_ms", e.latency_ms), wan.get("capacity_gbps", e.capacity_gbps),
                                   e.cost_per_GB)
    return ingresses, dcs, graph, build_paper_coeffs(dcs)
