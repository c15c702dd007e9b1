#!/usr/bin/env python
"""Re-runs the cases a GPU fuzz flagged under several builds / launch shapes: is a mismatch a property of the SCENARIO
(every build disagrees with the oracle on it, each in its own way: ill-conditioned) or of one build?

    python tools/fuzz_recheck.py failed_cases.json label[:lib=path][:ENV=val] ...
"""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CHILD = r'''
import sys, json
sys.path.insert(0, %r)
from distributed_cluster_gpus_b200 import scenarios as SC, spec as S
from distributed_cluster_gpus_b200.engine import BatchedEngine
case = json.loads(sys.argv[1]); n = int(sys.argv[2])
sp = SC.to_spec(case["scenario"])
with BatchedEngine(sp, n, case["seed"], 0, 0) as e:
    e.advance(0)
    s = e.summary()
    print(json.dumps({"events": s[:, S.S_EVENTS].astype(int).tolist(), "status": s[:, S.S_STATUS].astype(int).tolist(),
                      "energy": s[:, S.S_TOTAL_ENERGY_J].tolist(), "lanes": e.launch_info().get("lanes_per_replica")}))
''' % ROOT


def main():
    spec = json.load(open(sys.argv[1]))
    sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "oracle"))
    import oracle_lib as oracle
    from distributed_cluster_gpus_b200 import scenarios as SC, spec as S
    n = spec["replicas"]
    for case in spec["cases"]:
        sp = SC.to_spec(case["scenario"])
        want, _ = oracle.run_batch(sp.to_bytes(), n, case["seed"], 0, n_threads=8)
        ref = want[:, S.S_EVENTS].astype(int).tolist()
        print(json.dumps({"case": case["case"], "variant": "oracle", "events": ref}), flush=True)
        for v in sys.argv[2:]:
            parts = v.split(":")
            env = {}
            for kv in parts[1:]:
                k, val = kv.split("=", 1)
                env["DCSIM_B200_LIB" if k == "lib" else k] = os.path.abspath(val) if k == "lib" else val
            try:
                r = subprocess.run([sys.executable, "-c", CHILD, json.dumps(case), str(n)], env=dict(os.environ, **env),
                                   capture_output=True, text=True, timeout=300)
                row = json.loads(r.stdout.strip().splitlines()[-1]) if r.returncode == 0 and r.stdout.strip() else {"error": (r.stderr or "")[-400:]}
            except Exception as e:  # noqa: BLE001
                row = {"error": repr(e)}
            if "events" in row:
                row["differs_in_replicas"] = [i for i, (a, b) in enumerate(zip(row["events"], ref)) if a != b]
                row["energy_rel_err"] = [abs(a - b) / abs(b) for a, b in zip(row.pop("energy"), want[:, S.S_TOTAL_ENERGY_J].tolist())]
            print(json.dumps(dict({"case": case["case"], "variant": parts[0]}, **row)), flush=True)


if __name__ == "__main__":
    main()
