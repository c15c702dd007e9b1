"""Regenerates tests/golden/fuzz_reference.json: RANDOM scenarios (generator of tools/fuzz_core.py, fixed seed) run
through the UNMODIFIED reference — once with the Philox stream injected (oracle/ref_harness.py) and once exactly as
shipped, on its own Mersenne Twister ("run_mt") — only possible where
$DCSIM_REFERENCE_ROOT names a reference checkout.  The fixture pins the oracle (tests/test_oracle_vs_reference.py) and, through it, the
device path on parameter combinations nobody picked by hand.  Usage: python tests/golden/make_golden_fuzz.py [cases]
"""
import json
import os
import platform
import random
import signal
import sys
import time

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
for p in (ROOT, os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tools"), os.path.join(ROOT, "tests")):
    sys.path.insert(0, p)

from distributed_cluster_gpus_b200 import scenarios as S  # noqa: E402
from fuzz_core import random_scenario  # noqa: E402
from ref_harness import run_reference  # noqa: E402

GENERATOR_SEED = 20260924
EVENT_BUDGET = 4000  # the Python reference does ~1e4 events/s


class _Timeout(Exception):
    pass


def _alarm(signum, frame):
    raise _Timeout()


def bounded(sc):
    """Shortens the scenario so that the reference finishes in about a second."""
    n_ing = len(S.build_inputs(sc)["ingresses"])
    rate = sum(a["rate"] for a in (sc["inf"], sc["trn"]) if a["mode"] != "off")
    est = 3.0 * n_ing * rate * sc["duration"]
    if est > EVENT_BUDGET:
        sc = dict(sc, duration=round(sc["duration"] * EVENT_BUDGET / est, 3))
    return sc


def main():
    n_cases = int(sys.argv[1]) if len(sys.argv) > 1 else 160
    rnd = random.Random(GENERATOR_SEED)
    signal.signal(signal.SIGALRM, _alarm)
    cases, skipped, t0 = [], 0, time.time()
    for case in range(n_cases):
        sc = bounded(random_scenario(rnd, case))
        seed = rnd.randrange(1, 2 ** 40)
        signal.alarm(40)
        try:
            run = run_reference(sc, seed, rng="philox")
            run_mt = run_reference(sc, seed, rng="mt")      # the reference exactly as shipped (its own MT19937)
        except _Timeout:
            skipped += 1
            print("case", case, "skipped: reference did not finish in 40 s", sc, flush=True)
            continue
        finally:
            signal.alarm(0)
        run.pop("ref_wall_s", None)
        run_mt.pop("ref_wall_s", None)
        cases.append({"scenario": sc, "run": run, "run_mt": run_mt})
        if case % 20 == 0:
            print(case, sc["algo"], run["events"], "events", "%.0f s" % (time.time() - t0), flush=True)
    doc = {"meta": {"generated_by": "tests/golden/make_golden_fuzz.py", "reference": "filrg/distributed_cluster_GPUs @ 9e78013",
                    "python": platform.python_version(), "libc": " ".join(platform.libc_ver()), "machine": platform.machine(),
                    "generator_seed": GENERATOR_SEED, "skipped": skipped},
           "cases": cases}
    with open(os.path.join(HERE, "fuzz_reference.json"), "w") as f:
        json.dump(doc, f, separators=(",", ":"))
    print(len(cases), "cases,", sum(c["run"]["events"] for c in cases), "events,", skipped, "skipped, %.0f s" % (time.time() - t0))


if __name__ == "__main__":
    main()
