#!/usr/bin/env python
"""Throughput of every BASELINE.json config on one GPU at its per-GPU replica count (not bench lines: context).

    python tools/config_sweep.py > config_sweep.json
"""
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
import torch  # noqa: E402

from distributed_cluster_gpus_b200 import scenarios as SC, spec as S  # noqa: E402
from distributed_cluster_gpus_b200.engine import BatchedEngine  # noqa: E402

CASES = [("cfg1_1x4_poisson_5000s", 65536), ("cfg2_1x64_poisson_600s", 65536), ("cfg3_4x64_sinusoid_120s", 65536),
         ("cfg3_4x64_sinusoid_600s", 16384), ("cfg5_8x256_sinusoid_60s", 131072),
         ("sweep_default_perf_first", 32768), ("sweep_joint_nf", 32768), ("sweep_carbon_cost", 32768),
         ("sweep_eco_route", 32768), ("sweep_debug_n2", 32768), ("sweep_bandit", 32768), ("cap_greedy_4x64", 32768)]
stream = torch.cuda.Stream()
torch.cuda.set_stream(stream)
out = []
for name, n in CASES:
    sc = SC.BY_NAME[name]
    sp = SC.to_spec(sc)
    eng = BatchedEngine(sp, n, 123, cuda_stream=stream.cuda_stream)
    eng.advance(0)                                                  # warm-up
    eng.reset(999)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record(stream)
    eng.advance(0, sync=False)
    e1.record(stream)
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1)
    s = eng.summary()
    info = eng.launch_info()
    eng.close()
    ev = float(s[:, S.S_EVENTS].sum())
    out.append({"scenario": name, "replicas": n, "events": ev, "kernel_ms": ms, "events_per_s": ev / (ms / 1e3),
                "failed": int(np.count_nonzero((s[:, S.S_STATUS] != 0) | (s[:, S.S_DONE] == 0))),
                "warps_per_sm": info["resident_warps_per_sm"], "regs": info["regs_per_thread"],
                "state_block_bytes": info["smem_bytes_per_cta"] // info["warps_per_cta"],
                "hbm_gb": (info["hbm_bytes_state"] + info["hbm_bytes_queues"]) / 1e9,
                "max_run": float(s[:, S.S_MAX_RUN].max()), "max_xfer": float(s[:, S.S_MAX_XFER].max()), "max_q": float(s[:, S.S_MAX_Q].max())})
    print(json.dumps(out[-1]), flush=True)
