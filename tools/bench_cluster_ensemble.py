#!/usr/bin/env python
"""Cost of the cluster-log ensemble (or, with --recorder job, the job-log ensemble) at bench size: the event loop with
the recorder off and on, the two reduction kernels, the recorder's bytes per replica.  One JSON line on stdout; writes
nothing else.

    python tools/bench_cluster_ensemble.py [--recorder cluster|job] [--replicas 65536] [--scenario cfg3_4x64_sinusoid_120s]
                                           [--rounds 3]

Each batch runs on a fresh engine (two bench-size batches do not fit beside each other), the arms alternate
(off on / on off / ...), the seeds are the same, times are CUDA events on the launching stream (bench.timed_batch: one
warm-up batch, then one timed).  The reductions are timed on their second pass; the moments pass includes the capacity
check's host round trip (the job-log ensemble has none).
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--replicas", type=int, default=65536)
    ap.add_argument("--scenario", default="cfg3_4x64_sinusoid_120s")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--recorder", choices=["cluster", "job"], default="cluster")
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
        if arm == "on" and args.recorder == "job":
            e.enable_job_ensemble()
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
    try:
        on.advance(0)
        events = float(on.summary()[:, S.S_EVENTS].sum())
        if args.recorder == "job":
            cols = (on.job_ensemble_windows + 1) * len(EN.JOB_FIELDS) * sp.n_dc * 2
            moments_into, spread_into = on.job_ensemble_moments_into, on.job_ensemble_spread_into
            rows, recorder_bytes = on.job_ensemble_windows + 1, ((on.job_ensemble_windows + 1) * 2 * sp.n_dc * 2 * 8
                                                                 + sp.n_dc * 2 * EN.LAT_BINS * 4)
        else:
            cols = on.cluster_ensemble_capacity * len(EN.FIELDS) * sp.n_dc
            moments_into, spread_into = on.ensemble_moments_into, on.ensemble_spread_into
            rows, recorder_bytes = on.cluster_ensemble_capacity, cols * 8
        mom = torch.zeros((4, cols), dtype=torch.float64, device="cuda")
        m2 = torch.zeros(cols, dtype=torch.float64, device="cuda")
        hist = torch.zeros((cols, EN.BINS), dtype=torch.int64, device="cuda")
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
        for _ in range(2):
            torch.cuda.synchronize()
            ev[0].record(stream)
            moments_into(mom.data_ptr())
            ev[1].record(stream)
            cnt = mom[0]
            mean = torch.where(cnt > 0, mom[1] / cnt.clamp(min=1.0), torch.zeros_like(cnt)).contiguous()
            lo, hi = mom[2].contiguous(), mom[3].contiguous()
            torch.cuda.synchronize()
            ev[2].record(stream)
            spread_into(mean.data_ptr(), lo.data_ptr(), hi.data_ptr(), m2.data_ptr(), hist.data_ptr())
            ev[3].record(stream)
            torch.cuda.synchronize()
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
                      "moments_ms": moments_ms, "spread_ms": spread_ms}), flush=True)


if __name__ == "__main__":
    main()
