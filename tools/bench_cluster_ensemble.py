#!/usr/bin/env python
"""Cost of the cluster-log ensemble (or, with --recorder job / power / waits / occupancy / tail / resources / cost, the
job-log ensemble / the power profile / the waiting-time recorder on top of the job ensemble / the occupancy recorder / the
per-run tail-latency recorder / the job-resources recorder on top of the job ensemble / the energy-cost recorder) at bench size: the event loop with the recorder off and on, the two reduction kernels, the recorder's bytes per
replica.  One JSON line on stdout; writes nothing else.

    python tools/bench_cluster_ensemble.py [--recorder cluster|job|power|waits|occupancy|tail|resources|cost] [--replicas 65536] [--scenario cfg3_4x64_sinusoid_120s]
                                           [--rounds 3]

Each batch runs on a fresh engine (two bench-size batches do not fit beside each other), the arms alternate
(off on / on off / ...), the seeds are the same, times are CUDA events on the launching stream (bench.timed_batch: one
warm-up batch, then one timed).  The reductions are timed on their second pass; the moments pass includes the capacity
check's host round trip (the job-log ensemble has none).  For the tail recorder the first moments pass also runs the
selection pass (with its all-done check): `selection_ms` is that first pass less the second.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

# --recorder -> the recorder's name in engine.RECORDERS
RECORDERS = {"cluster": "cluster_ensemble", "job": "job_ensemble", "power": "power_profile", "waits": "job_waits",
             "occupancy": "occupancy", "tail": "tail_latency", "resources": "job_resources", "cost": "energy_cost"}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--replicas", type=int, default=65536)
    ap.add_argument("--scenario", default="cfg3_4x64_sinusoid_120s")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--recorder", choices=list(RECORDERS), default="cluster")
    args = ap.parse_args()

    import torch
    from bench import timed_batch
    from distributed_cluster_gpus_b200 import ensemble as EN, scenarios as SC, spec as S
    from distributed_cluster_gpus_b200.engine import BatchedEngine

    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    sp = SC.to_spec(SC.BY_NAME[args.scenario])
    n, seed = args.replicas, 123
    stream = torch.cuda.Stream()
    torch.cuda.set_stream(stream)

    def make(arm):
        e = BatchedEngine(sp, n, base_seed=seed, cuda_stream=stream.cuda_stream)
        if args.recorder in ("waits", "resources"):  # their own cost: both arms run the job ensemble they need
            e.enable_job_ensemble()
            if arm == "on":
                e.enable_job_waits() if args.recorder == "waits" else e.enable_job_resources()
        elif arm == "on" and args.recorder == "job":
            e.enable_job_ensemble()
        elif arm == "on" and args.recorder == "power":
            e.enable_power_profile(sp.power_cap if sp.power_cap > 0 else None)
        elif arm == "on" and args.recorder == "occupancy":
            e.enable_occupancy()
        elif arm == "on" and args.recorder == "tail":
            e.enable_tail_latency(0.5)
        elif arm == "on" and args.recorder == "cost":
            e.enable_energy_cost()
        elif arm == "on":
            e.enable_cluster_ensemble()
        return e

    loop_ms = {"off": [], "on": []}
    for i in range(args.rounds):
        for arm in ("off", "on") if i % 2 == 0 else ("on", "off"):
            e = make(arm)
            try:
                loop_ms[arm].append(timed_batch(torch, None, e, stream, 1, seed, 0)[2])
            finally:
                e.close()

    on = make("on")
    stats = None
    try:
        on.advance(0)
        events = float(on.summary()[:, S.S_EVENTS].sum())
        recorder = RECORDERS[args.recorder]
        cols, spread_cols = on.stat_columns(recorder)
        if args.recorder == "power":
            rows, recorder_bytes = cols, cols * 8 + 20 * 8      # columns + the working row (DCSIM_PPW_N doubles)
        elif args.recorder == "occupancy":
            rows, recorder_bytes = cols + 1, (cols + 1) * 8 + sp.n_dc * 11 * 8   # columns + working rows (DCSIM_OCCW_N)
        elif args.recorder == "cost":
            rows, recorder_bytes = cols, S.cost_bytes_per_replica(sp.n_dc)   # columns + working rows (3 doubles per DC)
            stats = EN.energy_cost(on).pooled()
        elif args.recorder == "tail":
            cap = sp.cap_arrivals if sp.cap_arrivals > 0 else 16384
            rows, recorder_bytes = cols, cols * 8 + cap * 16     # columns + the slot buffer (16 B per arrival slot)
        elif args.recorder == "waits":
            rows, recorder_bytes = on.job_ensemble_windows + 1, ((on.job_ensemble_windows + 1) * 3 * sp.n_dc * 2 * 8
                                                                 + sp.n_dc * 2 * 2 * EN.LAT_BINS * 4)
            summ = on.summary()
            stats = EN.job_waits(on).pooled()
            for jt, name in enumerate(EN.JOB_TYPES):   # the service latency the summaries report, beside the waits
                fin = summ[:, S.S_FIN_INF if jt == 0 else S.S_FIN_TRN].sum()
                lat = summ[:, S.S_LAT_SUM_INF if jt == 0 else S.S_LAT_SUM_TRN].sum()
                stats[name]["mean_service_s"] = float(lat / fin) if fin else float("nan")
        elif args.recorder == "resources":
            win = on.job_ensemble_windows + 1
            rows, recorder_bytes = win, win * 3 * sp.n_dc * 2 * 8 + (cols - spread_cols) * 4   # sums + u32 counts
            stats = EN.job_resources(on).pooled()
        elif args.recorder == "job":
            rows, recorder_bytes = on.job_ensemble_windows + 1, ((on.job_ensemble_windows + 1) * 2 * sp.n_dc * 2 * 8
                                                                 + sp.n_dc * 2 * EN.LAT_BINS * 4)
        else:
            rows, recorder_bytes = on.cluster_ensemble_capacity, cols * 8
        mom = torch.zeros((4, cols), dtype=torch.float64, device="cuda")
        m2 = torch.zeros(spread_cols, dtype=torch.float64, device="cuda")
        hist = torch.zeros((spread_cols, EN.BINS), dtype=torch.int64, device="cuda")
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
        first_moments_ms = None
        for _ in range(2):
            torch.cuda.synchronize()
            ev[0].record(stream)
            on.stat_moments_into(recorder, mom.data_ptr())
            ev[1].record(stream)
            cnt = mom[0]
            mean = torch.where(cnt > 0, mom[1] / cnt.clamp(min=1.0), torch.zeros_like(cnt)).contiguous()
            lo, hi = mom[2].contiguous(), mom[3].contiguous()
            torch.cuda.synchronize()
            ev[2].record(stream)
            on.stat_spread_into(recorder, mean.data_ptr(), lo.data_ptr(), hi.data_ptr(), m2.data_ptr(), hist.data_ptr())
            ev[3].record(stream)
            torch.cuda.synchronize()
            first_moments_ms = ev[0].elapsed_time(ev[1]) if first_moments_ms is None else first_moments_ms
        if args.recorder == "tail":
            stats = EN.tail_latency(on).pooled()
        moments_ms, spread_ms = ev[0].elapsed_time(ev[1]), ev[2].elapsed_time(ev[3])
    finally:
        on.close()

    try:
        gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception:
        gpu = torch.cuda.get_device_name()
    med = lambda xs: float(np.median(xs))  # noqa: E731
    print(json.dumps({"gpu": gpu, "recorder": args.recorder, "scenario": args.scenario, "replicas": n, "rounds_alternated": args.rounds,
                      "events": events, "event_loop_ms_off": loop_ms["off"], "event_loop_ms_on": loop_ms["on"],
                      "events_per_s_off": events / (med(loop_ms["off"]) / 1e3),
                      "events_per_s_on": events / (med(loop_ms["on"]) / 1e3),
                      "slowdown_on_vs_off": med(loop_ms["on"]) / med(loop_ms["off"]) - 1.0,
                      "rows": rows, "bytes_per_replica": recorder_bytes, "bytes_total": recorder_bytes * n,
                      "moments_ms": moments_ms, "spread_ms": spread_ms,
                      **({"waits": stats} if args.recorder == "waits" else {}),
                      **({"resources": stats} if args.recorder == "resources" else {}),
                      **({"cost": stats} if args.recorder == "cost" else {}),
                      **({"selection_ms": first_moments_ms - moments_ms, "tail": stats} if args.recorder == "tail" else {})}),
          flush=True)


if __name__ == "__main__":
    main()
