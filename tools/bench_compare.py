#!/usr/bin/env python
"""Policy comparison at bench size: the BASELINE config 4 variants (4 DC x 64, freq {0.5, 0.8, 1.0}, 120 s) on the same
replica keys, in two arms that alternate round by round:

  separate  one batch per variant, each with its own arrival pre-pass (what tools/policy_sweep.py does)
  shared    one group: the baseline owns the pre-pass, every other variant is a member on its lists (compare.py)

Per arm: device time of the pre-passes and of the event loops (CUDA events on the stream the engines launch on), the
device memory each creation took (cudaMemGetInfo before / after) next to launch_info's byte counts, and whether every
variant's summary rows are bit-identical between the arms.  The shared arm also reports var_ratio per metric (var of the
paired difference over the sum of the two variances: how much pairing narrows the CI of a difference).  One JSON line.

    python tools/bench_compare.py --replicas 65536 --rounds 2
"""
import argparse
import hashlib
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
import torch  # noqa: E402

from distributed_cluster_gpus_b200 import compare as CP, scenarios as SC, spec as S  # noqa: E402
from distributed_cluster_gpus_b200.engine import BatchedEngine  # noqa: E402

VARIANTS = [("default_policy", "energy_aware", {}), ("default_policy", "perf_first", {}), ("joint_nf", "energy_aware", {}),
            ("carbon_cost", "energy_aware", {}), ("bandit", "energy_aware", {}), ("debug", "energy_aware", {"num_fixed_gpus": 2}),
            ("cap_greedy", "energy_aware", {"power_cap": 20000.0})]


def _specs(duration):
    out = {}
    for algo, policy, extra in VARIANTS:
        name = f"{algo}/{policy}" + "".join(f"/{k}={v:g}" for k, v in extra.items())
        out[name] = SC.to_spec(SC.scenario(name, 4, 64, SC.SIN10, SC.POI(1.0), duration, SC.FREQ3, algo=algo, policy=policy, **extra))
    return out


def _free():
    torch.cuda.synchronize()
    return torch.cuda.mem_get_info()[0]


def _timed(eng, stream):
    """(pre-pass ms, event-loop ms, summary rows) of one batch on `stream`."""
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
    with torch.cuda.stream(stream):
        ev[0].record(stream)
        eng.prepare()
        ev[1].record(stream)
        eng.advance(0, sync=False)
        ev[2].record(stream)
    summ = eng.summary()
    torch.cuda.synchronize()
    return ev[0].elapsed_time(ev[1]), ev[1].elapsed_time(ev[2]), summ


def _arm(specs, n, seed, shared, stream, want_pairs):
    names = list(specs)
    res = {"prepass_ms": 0.0, "event_loop_ms": 0.0, "created_bytes": {}, "launch_info_bytes": {}, "digest": {}}
    t0 = time.perf_counter()
    owner, pairs = None, {}
    try:
        for name in names:
            free0 = _free()
            if shared and owner is not None:
                eng = BatchedEngine.shared(specs[name], owner)
            else:
                eng = BatchedEngine(specs[name], n, seed)
                eng.set_stream(stream.cuda_stream)
            res["created_bytes"][name] = free0 - _free()
            li = eng.launch_info()
            res["launch_info_bytes"][name] = li["hbm_bytes_state"] + li["hbm_bytes_queues"] + li["hbm_bytes_arrivals"]
            pre, loop, summ = _timed(eng, stream)
            res["prepass_ms"] += pre
            res["event_loop_ms"] += loop
            assert np.all(summ[:, S.S_STATUS] == 0), (name, int(np.bitwise_or.reduce(summ[:, S.S_STATUS].astype(np.int64))))
            res["digest"][name] = hashlib.sha256(summ.tobytes()).hexdigest()
            if shared and owner is None:
                owner = eng                                # stays: the group's lists and the base of the reductions
                continue
            if want_pairs and owner is not None:
                pairs[name] = CP._paired_on_device(owner, torch.from_numpy(summ).cuda(), 4, torch.device("cuda"),
                                                   CP.EN.DEFAULT_QUANTILES)
            eng.close()
    finally:
        if owner is not None:
            owner.close()
    res["wall_s"] = time.perf_counter() - t0
    res["device_ms"] = res["prepass_ms"] + res["event_loop_ms"]
    return res, pairs


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--replicas", type=int, default=65536)
    ap.add_argument("--duration", type=float, default=120.0)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--seed", type=int, default=123)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_compare needs a CUDA device")
    specs = _specs(args.duration)
    stream = torch.cuda.Stream()
    _arm({k: specs[k] for k in list(specs)[:2]}, min(args.replicas, 4096), args.seed, True, stream, False)   # warm-up
    rounds = {"separate": [], "shared": []}
    var_ratio = None
    for r in range(args.rounds):
        for arm in (("separate", "shared") if r % 2 == 0 else ("shared", "separate")):
            res, pairs = _arm(specs, args.replicas, args.seed, arm == "shared", stream, var_ratio is None and arm == "shared")
            rounds[arm].append(res)
            if pairs:
                names = CP.metric_names(4)
                var_ratio = {v: {m + (f"[{i - len(CP.METRICS)}]" if m == CP.DC_METRIC else ""): float(st.var_ratio[i])
                                 for i, m in enumerate(names)} for v, st in pairs.items()}
    identical = all(a["digest"] == rounds["shared"][0]["digest"] for arm in rounds.values() for a in arm)
    try:
        gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception:
        gpu = torch.cuda.get_device_name()
    med = lambda arm, k: float(np.median([x[k] for x in rounds[arm]]))  # noqa: E731
    summary = {arm: {k: med(arm, k) for k in ("device_ms", "prepass_ms", "event_loop_ms", "wall_s")} for arm in rounds}
    for arm in rounds:
        first = rounds[arm][0]
        summary[arm]["created_bytes"] = first["created_bytes"]
        summary[arm]["launch_info_bytes"] = first["launch_info_bytes"]
        summary[arm]["peak_created_bytes"] = (first["created_bytes"][list(specs)[0]] + max(list(first["created_bytes"].values())[1:])
                                              if arm == "shared" else max(first["created_bytes"].values()))
        summary[arm]["rounds_device_ms"] = [x["device_ms"] for x in rounds[arm]]
    print(json.dumps({"gpu": gpu, "replicas": args.replicas, "duration_s": args.duration, "variants": list(specs),
                      "rounds_alternated": args.rounds, "arms": summary,
                      "saving_device_ms": summary["separate"]["device_ms"] - summary["shared"]["device_ms"],
                      "summaries_bit_identical": identical, "var_ratio": var_ratio}), flush=True)


if __name__ == "__main__":
    main()
