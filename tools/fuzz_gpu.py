#!/usr/bin/env python
"""Differential fuzz on the GPU: the sm_90a kernels through the C-ABI against the C oracle on random scenarios
(the generator of tools/fuzz_core.py).  Counts must be exact, every float within 1e-9 relative (the parity bar);
capacity overflows go through engine.run_to_completion's retry like in production.

    python tools/fuzz_gpu.py --cases 300 --seed 7 > fuzz_gpu.json
"""
import argparse
import json
import os
import random
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import numpy as np  # noqa: E402

import hostemu_lib as hostemu  # noqa: E402  (conditioning probe only)
import oracle_lib as oracle  # noqa: E402
from fuzz_core import random_scenario  # noqa: E402
from distributed_cluster_gpus_b200 import scenarios as SC, spec as S  # noqa: E402
from distributed_cluster_gpus_b200.engine import BatchedEngine  # noqa: E402

COUNT_COLS = (S.S_STATUS, S.S_EVENTS, S.S_JOBS_FINISHED, S.S_JOBS_CREATED, S.S_FIN_INF, S.S_FIN_TRN, S.S_RNG_WORDS,
              S.S_SEQ, S.S_EV_ARRIVAL, S.S_EV_XFER, S.S_EV_FINISH, S.S_EV_LOG, S.S_DONE)
FLOAT_COLS = (S.S_TOTAL_ENERGY_J, S.S_LAT_SUM, S.S_LAT_SUM_INF, S.S_LAT_SUM_TRN, S.S_LAST_T)


def float_cols(n_dc):
    cols = list(FLOAT_COLS)
    for d in range(n_dc):
        b = S.S_DC0 + d * S.S_DC_STRIDE
        cols += [b + S.SD_ENERGY_J, b + S.SD_UTIL_GPU_TIME, b + S.SD_ACC_JOB_UNIT, b + S.SD_CURRENT_FREQ]
    return cols


def sensitivity(sp, n, seed, want, n_dc):
    """How far the scenario's floats move when every 5th pow() result of the HOST build is off by one ulp (no GPU
    involved): the scenario's own amplification of last-bit libm differences."""
    got = hostemu.run_batch(sp.to_bytes(), n, seed, perturbed=True)["summary"]
    worst = 0.0
    for col in float_cols(n_dc):
        denom = np.maximum(np.abs(want[:, col]), 1e-300)
        worst = max(worst, float(np.max(np.where(want[:, col] == got[:, col], 0.0, np.abs(got[:, col] - want[:, col]) / denom))))
    return worst


def compare(got, want, n_dc):
    for col in COUNT_COLS:
        if not np.array_equal(got[:, col], want[:, col]):
            return "count column %d: %s vs %s" % (col, got[:, col].tolist(), want[:, col].tolist()), 0.0
    cols = list(FLOAT_COLS)
    for d in range(n_dc):
        b = S.S_DC0 + d * S.S_DC_STRIDE
        cols += [b + S.SD_ENERGY_J, b + S.SD_UTIL_GPU_TIME, b + S.SD_ACC_JOB_UNIT, b + S.SD_CURRENT_FREQ]
        for k in (S.SD_BUSY, S.SD_Q_INF, S.SD_Q_TRN, S.SD_RUNNING):
            if not np.array_equal(got[:, b + k], want[:, b + k]):
                return "dc%d field %d" % (d, k), 0.0
    worst = 0.0
    for col in cols:
        denom = np.maximum(np.abs(want[:, col]), 1e-300)
        rel = float(np.max(np.where(want[:, col] == got[:, col], 0.0, np.abs(got[:, col] - want[:, col]) / denom)))
        worst = max(worst, rel)
    return (None if worst <= 1e-9 else "float rel err %.3e" % worst), worst


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--cases", type=int, default=300)
    ap.add_argument("--seed", type=int, default=7)
    ap.add_argument("--replicas", type=int, default=6)
    args = ap.parse_args()
    rnd = random.Random(args.seed)
    fails, ill, worst_all, events, t0, by_algo = [], [], 0.0, 0, time.time(), {}
    for case in range(args.cases):
        sc = random_scenario(rnd, case)
        seed = rnd.randrange(1, 2 ** 40)
        log_mode = case % 3  # 0: plain (lean records), 1: job+cluster log and trace on replica 1, 2: stepping in chunks
        sp = SC.to_spec(sc)
        want, want_total = oracle.run_batch(sp.to_bytes(), args.replicas, seed, 0, n_threads=8)
        try:
            with BatchedEngine(sp, args.replicas, seed, 0, 0) as eng:
                if log_mode == 1:
                    eng.set_logging(1, 60000, 4000); eng.set_trace(1, 4000)
                if log_mode == 2:
                    total = 0
                    while not eng.all_done():
                        total += eng.advance(997)
                else:
                    total = eng.advance(0)
                got = eng.summary()
                err, worst = compare(got, want, sc["n_dc"])
                if err is None and total != want_total:
                    err = "event total %d vs %d" % (total, want_total)
                if err is None and log_mode == 1:
                    sim = oracle.OracleSim(sp.to_bytes(), seed + 1, trace_cap=4000, joblog_cap=60000, clog_cap=4000)
                    sim.advance(0)
                    tr, wt = eng.trace(), sim.trace()
                    jl, wj = eng.job_log(), sim.job_log()
                    if len(tr) != len(wt) or not np.array_equal(tr["seq"], wt["seq"]) or not np.array_equal(tr["kind"], wt["kind"]):
                        err = "trace differs"
                    elif len(jl) != len(wj) or not np.array_equal(jl["jid"], wj["jid"]):
                        err = "job log differs"
                    sim.close()
        except Exception as e:
            err, worst = "EXC %s: %s" % (type(e).__name__, str(e)[:200]), 0.0
        by_algo[sc["algo"]] = by_algo.get(sc["algo"], 0) + 1
        if err and err.startswith("float rel err"):
            # counts are exact; is the scenario itself that sensitive to last-bit differences?  (host-only probe)
            probe = sensitivity(sp, args.replicas, seed, want, sc["n_dc"])
            if probe > 1e-10 and worst <= 1000.0 * probe:
                ill.append({"case": case, "gpu_rel_err": worst, "one_ulp_probe_rel_err": probe, "scenario": sc, "seed": seed})
                err, worst = None, 0.0
        worst_all = max(worst_all, worst)
        events += int(want_total)
        if err:
            fails.append({"case": case, "mode": log_mode, "error": err, "scenario": sc, "seed": seed})
            print("FAIL", case, log_mode, err, sc, seed, file=sys.stderr, flush=True)
    print(json.dumps({"cases": args.cases, "replicas_per_case": args.replicas, "generator_seed": args.seed, "events_compared": events,
                      "failures": len(fails), "worst_float_rel_err": worst_all,
                      "ill_conditioned": ill, "cases_by_algo": by_algo,
                      "seconds": round(time.time() - t0, 1), "failed": fails[:20]}))
    sys.exit(1 if fails else 0)
