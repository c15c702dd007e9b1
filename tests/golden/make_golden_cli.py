"""Golden files written by the reference's OWN command line, untouched: `python $DCSIM_REFERENCE_ROOT/run_sim_paper.py
<flags>` (its process-global Mersenne Twister, its default 8-DC scenario).  The product's CLI with the same flags
plus `--rng mt19937` must write the same files.  Needs a reference checkout.   python tests/golden/make_golden_cli.py"""
import json
import os
import shutil
import subprocess
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
REFERENCE_ROOT = os.environ.get("DCSIM_REFERENCE_ROOT", "")

CASES = {
    "defaults_12s_seed7": ["--duration", "12", "--seed", "7"],
    "carbon_cost_poisson_10s_seed5": ["--duration", "10", "--seed", "5", "--algo", "carbon_cost", "--inf-mode", "poisson",
                                      "--inf-rate", "3", "--trn-rate", "0.2", "--log-interval", "2"],
    "perf_first_debug_n4_8s_seed99": ["--duration", "8", "--seed", "99", "--algo", "debug", "--num_fixed_gpus", "4",
                                      "--fixed_freq", "0.8", "--policy", "perf_first"],
}

if __name__ == "__main__":
    if not os.path.isfile(os.path.join(REFERENCE_ROOT, "run_sim_paper.py")):
        raise SystemExit(f"reference tree not found at {REFERENCE_ROOT!r}; set DCSIM_REFERENCE_ROOT to a checkout of the "
                         "reference to regenerate the CLI goldens")
    out = os.path.join(HERE, "cli")
    os.makedirs(out, exist_ok=True)
    for name, flags in CASES.items():
        with tempfile.TemporaryDirectory() as tmp:
            logs = os.path.join(tmp, "logs", "x")
            subprocess.run([sys.executable, os.path.join(REFERENCE_ROOT, "run_sim_paper.py"), "--log-path", logs] + flags,
                           cwd=tmp, check=True, capture_output=True, timeout=600)
            for f in ("cluster_log.csv", "job_log.csv"):
                shutil.copy(os.path.join(logs, f), os.path.join(out, f"{name}_{f}"))
        print(name, "ok", os.path.getsize(os.path.join(out, f"{name}_job_log.csv")), "bytes of job log")
    with open(os.path.join(out, "cases.json"), "w") as f:
        json.dump(CASES, f, indent=1)
