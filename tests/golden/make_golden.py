"""Regenerates tests/golden/*.json by running the UNMODIFIED reference (only possible where
$DCSIM_REFERENCE_ROOT names a reference checkout).  Usage:  python tests/golden/make_golden.py [name-substring ...]

For every scenario of distributed_cluster_gpus_b200.scenarios.GOLDEN_SCENARIOS:
  * rng = "mt"     seed 123                 — the reference exactly as shipped (global Mersenne Twister);
  * rng = "philox" seeds 123, 124, 2**40+7  — the reference with oracle/philox_random.PhiloxRandom injected.
Floats are stored as float.hex() so comparisons can be bit-exact.  kat.json additionally records the survey's
known-answer strings (SURVEY.md App. C) that the "mt" runs must reproduce — the proof that the harness does
not perturb the reference.
"""
import json
import os
import platform
import sys
import time

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))

from distributed_cluster_gpus_b200 import scenarios as S  # noqa: E402
from ref_harness import run_reference  # noqa: E402

PHILOX_SEEDS = [123, 124, 2**40 + 7]
TRACE_EVENTS = {"cfg3_4x64_sinusoid_120s": 600, "cfg1_1x4_poisson_5000s": 200, "sweep_joint_nf": 300,
                "cap_greedy_4x64": 300}

# SURVEY.md App. C: unmodified reference, MT19937, seed 123
SURVEY_KAT = {
    "cfg1_1x4_poisson_5000s": {"events": 15940, "total_energy_repr": "587568.6274574532", "jobs": 4980},
    "cfg2_1x64_poisson_600s": {"events": 18312, "total_energy_repr": "6672749.673869186", "jobs": 5022},
    "kat_4x64_sin6_600s": {"events": 67057, "total_energy_repr": "23186546.067431837", "jobs": 19653},
    "cfg3_4x64_sinusoid_600s": {"events": 117152, "total_energy_repr": "23375474.435973424", "jobs": 35061},
    "cfg3_4x64_sinusoid_120s": {"events": 17050, "total_energy_repr": "4557619.181151763"},
    "kat_8x256_sin10_poitrn_60s": {"events": 20764, "total_energy_repr": "12561052.820839519"},
    "sweep_joint_nf": {"events": 21559, "total_energy_repr": "4360415.220138516"},
}


def main():
    want = sys.argv[1:]
    meta = {"generated_by": "tests/golden/make_golden.py", "reference": "filrg/distributed_cluster_GPUs @ 9e78013",
            "python": platform.python_version(), "libc": " ".join(platform.libc_ver()),
            "machine": platform.machine(), "philox_seeds": PHILOX_SEEDS}
    kat_seen = {}
    for sc in S.GOLDEN_SCENARIOS:
        if want and not any(w in sc["name"] for w in want):
            continue
        t0 = time.time()
        runs = [run_reference(sc, 123, rng="mt")]
        if sc["name"] in SURVEY_KAT:
            k = SURVEY_KAT[sc["name"]]
            got = runs[0]
            ok = got["events"] == k["events"] and got["total_energy_builtin_sum_repr"] == k["total_energy_repr"] and \
                ("jobs" not in k or got["jobs_finished"] == k["jobs"])
            kat_seen[sc["name"]] = {"expected": k, "events": got["events"], "total_energy_repr": got["total_energy_builtin_sum_repr"],
                                    "jobs": got["jobs_finished"], "ok": ok}
            if not ok:
                raise SystemExit(f"harness is NOT neutral on {sc['name']}: {kat_seen[sc['name']]}")
        for i, seed in enumerate(PHILOX_SEEDS):
            runs.append(run_reference(sc, seed, rng="philox", trace_events=TRACE_EVENTS.get(sc["name"], 0) if i == 0 else 0))
        doc = {"meta": meta, "scenario": sc, "runs": runs}
        with open(os.path.join(HERE, sc["name"] + ".json"), "w") as f:
            json.dump(doc, f, indent=1)
        evs = sum(r["events"] for r in runs)
        wall = sum(r["ref_wall_s"] for r in runs)
        print(f"{sc['name']:40s} {len(runs)} runs {evs:8d} events  ref {wall:6.1f}s ({evs / max(wall, 1e-9):8.0f} ev/s)  total {time.time() - t0:5.1f}s",
              flush=True)
    write_kat(meta)


def write_kat(meta):
    """kat.json: the "mt" run of every scenario SURVEY.md App. C quotes, next to the quoted strings."""
    seen = {}
    for name, k in SURVEY_KAT.items():
        path = os.path.join(HERE, name + ".json")
        if not os.path.exists(path):
            continue
        with open(path) as f:
            got = [r for r in json.load(f)["runs"] if r["rng"] == "mt"][0]
        ok = got["events"] == k["events"] and got["total_energy_builtin_sum_repr"] == k["total_energy_repr"] and \
            ("jobs" not in k or got["jobs_finished"] == k["jobs"])
        seen[name] = {"expected": k, "events": got["events"], "total_energy_repr": got["total_energy_builtin_sum_repr"],
                      "jobs": got["jobs_finished"], "ok": ok}
    with open(os.path.join(HERE, "kat.json"), "w") as f:
        json.dump({"meta": meta, "survey_known_answers": seen}, f, indent=1)


if __name__ == "__main__":
    main()
