"""TEST INFRASTRUCTURE — not product code.  Runs ONLY where a reference checkout is named by $DCSIM_REFERENCE_ROOT.

Drives the *unmodified* reference simulator (simcore/simulator_paper_multi.py) programmatically on
the synthetic scenarios of SURVEY.md §8(d) and captures in-memory results (the CSVs round:
latency_s ``.6f`` simulator_paper_multi.py:820, energy_kJ ``.4f`` :948).

Two RNG modes:
  * ``mt``      the reference untouched: process-global Mersenne Twister seeded at :71.
                Reproduces the survey's known-answer values (SURVEY.md App. C) -> proves the harness neutral.
  * ``philox``  the five module attributes the reference looks up at call time
                (random.seed/random/expovariate/lognormvariate/choice; arrivals.py:8,11,15,44 and
                simulator_paper_multi.py:71,576) are re-bound to one PhiloxRandom instance.

Nothing under the product package is imported here.
"""
import contextlib
import logging
import os
import random
import sys
import tempfile
import time

REFERENCE_ROOT = os.environ.get("DCSIM_REFERENCE_ROOT", "")

_HERE = os.path.dirname(os.path.abspath(__file__))
if _HERE not in sys.path:
    sys.path.insert(0, _HERE)
from philox_random import PhiloxRandom  # noqa: E402

FREQ8 = [0.3, 0.4, 0.5, 0.6, 0.7, 0.8, 0.9, 1.0]


def scenario(name, n_dc, gpus_per_dc, inf, trn, duration, freq_levels=None, algo="default_policy",
             policy="energy_aware", log_interval=5.0, power_cap=0.0, num_fixed_gpus=1, fixed_freq=None,
             gpus_list=None):
    """A JSON-able scenario descriptor (shared with tests/ and bench.py through tests/golden/*.json)."""
    return {
        "name": name, "n_dc": n_dc, "gpus_per_dc": gpus_per_dc, "gpus_list": gpus_list,
        "freq_levels": list(freq_levels or FREQ8),
        "inf": dict(inf), "trn": dict(trn), "duration": float(duration), "algo": algo, "policy": policy,
        "log_interval": float(log_interval), "power_cap": float(power_cap),
        "num_fixed_gpus": int(num_fixed_gpus), "fixed_freq": fixed_freq,
    }


def _import_reference():
    if not os.path.isdir(REFERENCE_ROOT):
        raise RuntimeError(f"reference tree not found at {REFERENCE_ROOT!r}; set DCSIM_REFERENCE_ROOT to a checkout of "
                           "the reference to regenerate the goldens")
    if REFERENCE_ROOT not in sys.path:
        sys.path.insert(0, REFERENCE_ROOT)
    from simcore.simulator_paper_multi import MultiIngressPaperSimulator
    from simcore.arrivals import ArrivalConfig
    from simcore.network import Graph
    from configs import paper_config as pc
    return MultiIngressPaperSimulator, ArrivalConfig, Graph, pc


@contextlib.contextmanager
def _patched_random(inst):
    names = ("seed", "random", "expovariate", "lognormvariate", "choice")
    saved = {n: getattr(random, n) for n in names}
    try:
        for n in names:
            setattr(random, n, getattr(inst, n))
        yield
    finally:
        for n, v in saved.items():
            setattr(random, n, v)


def build_reference_inputs(sc):
    """Scenario -> the reference's own dataclasses, per SURVEY.md §8(d)."""
    _, ArrivalConfig, Graph, pc = _import_reference()
    all_dcs = pc.build_dcs()
    keep = list(all_dcs)[: sc["n_dc"]]
    dcs = {}
    for i, k in enumerate(keep):
        dc = all_dcs[k]
        dc.total_gpus = int(sc["gpus_list"][i]) if sc.get("gpus_list") else int(sc["gpus_per_dc"])
        dc.freq_levels = list(sc["freq_levels"])
        assert dc.default_freq in dc.freq_levels
        dcs[k] = dc
    all_ing, full_graph = pc.build_ingresses_and_topology()
    ingresses = {f"gw-{k}": all_ing[f"gw-{k}"] for k in keep}
    nodes = set(keep) | set(ingresses)
    graph = Graph()
    for u, edges in full_graph.adj.items():
        if u not in nodes:
            continue
        for e in edges:
            if e.to in nodes:
                graph.add_edge(u, e.to, e.latency_ms, e.capacity_gbps, e.cost_per_GB)
    arr_inf = ArrivalConfig(**sc["inf"])
    arr_trn = ArrivalConfig(**sc["trn"])
    return dict(
        ingresses=ingresses, dcs=dcs, graph=graph, arrival_inf=arr_inf, arrival_train=arr_trn,
        router_policy=pc.build_router_policy(), coeffs_map=pc.build_paper_coeffs(dcs),
        carbon_intensity=pc.build_carbon_intensity(), energy_price=pc.build_energy_price(),
        policy=pc.build_policy(name=sc["policy"]),
    )


def run_reference(sc, seed, rng="philox", trace_events=0, log_dir=None):
    """One reference run. Returns a dict of exact (hex-float) results plus capacity statistics."""
    Sim, _, _, _ = _import_reference()
    inputs = build_reference_inputs(sc)
    logger = logging.getLogger("dcsim-ref-harness")
    logger.addHandler(logging.NullHandler())
    logger.propagate = False
    logger.setLevel(logging.CRITICAL)

    inst = PhiloxRandom(0) if rng == "philox" else None
    ctx = _patched_random(inst) if inst is not None else contextlib.nullcontext()
    tmp = None
    if log_dir is None:
        tmp = tempfile.TemporaryDirectory(prefix="dcsim_ref_", dir="/dev/shm" if os.path.isdir("/dev/shm") else None)
        log_dir = tmp.name
    st = {"events": 0, "by_type": {}, "lat_sum": 0.0, "lat_sum_inf": 0.0, "lat_sum_trn": 0.0,
          "n_fin": 0, "n_fin_inf": 0, "n_fin_trn": 0, "max_heap": 0, "max_run": 0, "max_qinf": 0,
          "max_qtrn": 0, "max_xfer": 0, "trace": [], "last_t": 0.0}
    with ctx:
        sim = Sim(logger=logger, sim_duration=sc["duration"], log_interval=sc["log_interval"], log_path=log_dir,
                  rng_seed=seed, algo=sc["algo"], power_cap=sc["power_cap"], show_progress=False,
                  num_fixed_gpus=sc["num_fixed_gpus"], fixed_freq=sc["fixed_freq"], **inputs)
        orig_pop = sim._pop
        orig_fin = sim._handle_job_finish
        dcs = sim.dcs

        def counting_pop():
            st["max_heap"] = max(st["max_heap"], len(sim.event_q))
            nx = sum(1 for e in sim.event_q if e[2] == "xfer_done") if (st["events"] % 64 == 0) else 0
            st["max_xfer"] = max(st["max_xfer"], nx)
            ev = orig_pop()
            if ev is not None and ev[0] <= sim.end_time:
                st["events"] += 1
                st["by_type"][ev[2]] = st["by_type"].get(ev[2], 0) + 1
                st["last_t"] = ev[0]
                if len(st["trace"]) < trace_events:
                    st["trace"].append([ev[0].hex(), ev[1], ev[2]])
            for dc in dcs.values():
                st["max_run"] = max(st["max_run"], len(dc.running_jobs))
                st["max_qinf"] = max(st["max_qinf"], len(dc.q_inf))
                st["max_qtrn"] = max(st["max_qtrn"], len(dc.q_train))
            return ev

        def capturing_finish(dc_name, jid):
            tup = dcs[dc_name].running_jobs.get(jid)
            orig_fin(dc_name, jid)
            if tup:
                job = tup[0]
                lat = job.finish_time - job.start_time          # what job_log.csv calls latency_s (:820)
                st["lat_sum"] += lat                            # plain left-to-right accumulation
                st["n_fin"] += 1
                if job.jtype == "inference":
                    st["lat_sum_inf"] += lat
                    st["n_fin_inf"] += 1
                else:
                    st["lat_sum_trn"] += lat
                    st["n_fin_trn"] += 1

        sim._pop = counting_pop
        sim._handle_job_finish = capturing_finish
        t0 = time.perf_counter()
        sim.run()
        wall = time.perf_counter() - t0
    if tmp is not None:
        tmp.cleanup()

    total_e = 0.0
    for dc in dcs.values():
        total_e += dc.energy_joules                             # left-to-right, DC dict order
    out = {
        "seed": seed, "rng": rng, "events": st["events"], "by_type": st["by_type"],
        "jobs_finished": st["n_fin"], "jobs_finished_inf": st["n_fin_inf"], "jobs_finished_trn": st["n_fin_trn"],
        "jobs_created": next(sim.jid_counter) - 1,
        "seq_pushed": next(sim.seq),
        "total_energy_j": total_e.hex(), "total_energy_repr": repr(total_e),
        # builtin sum() is Neumaier-compensated since CPython 3.12; this is the figure SURVEY.md App. C quotes
        "total_energy_builtin_sum_repr": repr(sum(dc.energy_joules for dc in dcs.values())),
        "latency_sum_s": st["lat_sum"].hex(), "latency_sum_inf_s": st["lat_sum_inf"].hex(),
        "latency_sum_trn_s": st["lat_sum_trn"].hex(),
        "mean_latency_s": (st["lat_sum"] / st["n_fin"]).hex() if st["n_fin"] else None,
        "last_event_t": float(st["last_t"]).hex(),
        "dc": [
            {"name": dc.name, "energy_j": dc.energy_joules.hex(), "util_gpu_time": float(dc.util_gpu_time).hex(),
             "acc_job_unit": float(dc.accumulated_job_unit).hex(), "busy": dc.busy_gpus,
             "current_freq": float(dc.current_freq).hex(), "q_inf": len(dc.q_inf), "q_train": len(dc.q_train),
             "running": len(dc.running_jobs)}
            for dc in dcs.values()
        ],
        "caps": {"max_heap": st["max_heap"], "max_running_per_dc": st["max_run"], "max_q_inf": st["max_qinf"],
                 "max_q_train": st["max_qtrn"], "max_xfer_sampled": st["max_xfer"]},
        "ref_wall_s": wall,
    }
    if inst is not None:
        out["rng_words"] = inst.words_consumed
        out["n_random"] = inst.n_random
        out["n_getrandbits"] = inst.n_getrandbits
    if trace_events:
        out["trace"] = st["trace"]
    return out
