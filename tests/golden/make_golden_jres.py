"""Golden job-resources cells from the UNMODIFIED reference, for tests/test_job_resources.py and its GPU twin.

The reference runs through oracle/ref_harness.run_reference with ``_handle_job_finish`` wrapped at run time: for every
job that finished it records, unrounded, the GPU count g and f_used of its running entry, its size, its finish instant
and E_pred — the first ``energy_tuple`` the handler evaluates (SIM:716), before any job it dequeues starts.  The
expected cells then come from the plain loops below, written from the definition in include/dcsim_b200.h (not from
the package): per finish window of log_interval seconds and for the whole run, sums in finish order of g, f and
E_job = E_pred * size; the (g, f) mix; the quarter-octave energy histogram from 1 J.  Floats are float.hex strings.

Build-container only (needs the reference tree):   DCSIM_REFERENCE_ROOT=... python tests/golden/make_golden_jres.py
"""
import json
import math
import os
import sys
from fractions import Fraction

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))
from distributed_cluster_gpus_b200 import scenarios as S  # noqa: E402
import ref_harness  # noqa: E402

CASES = [S.BY_NAME[n] for n in ("cfg3_4x64_sinusoid_120s", "sweep_joint_nf", "sweep_bandit", "cap_greedy_4x64",
                                 "ragged_3dc_12_5_40", "all_off_2x8", "underloaded_1x64")]
RUNS = [(123, "philox"), (124, "philox")]
MT_SCENARIOS = ("ragged_3dc_12_5_40", "cap_greedy_4x64")
TYPES = ("inference", "training")
MAX_FREQ, EBINS = 16, 128


def reference_jobs(sc, seed, rng):
    """-> ([(dc, jtype, g, f_used, E_pred, size, finish)] in finish order, reference result)."""
    ref_harness._import_reference()
    import simcore.simulator_paper_multi as M
    jobs, grab = [], []
    orig_fin, orig_et = M.MultiIngressPaperSimulator._handle_job_finish, M.energy_tuple

    def energy_tuple(*a, **kw):
        out = orig_et(*a, **kw)
        if grab and grab[-1] is None:
            grab[-1] = out
        return out

    def finish(self, dc_name, jid):
        dc = self.dcs[dc_name]
        tup = dc.running_jobs.get(jid)
        f_used = float(getattr(tup[0], "f_used", dc.current_freq)) if tup else None
        grab.append(None)
        orig_fin(self, dc_name, jid)
        got = grab.pop()
        if tup:
            job, g = tup
            jobs.append((list(self.dcs.keys()).index(dc_name), TYPES.index(job.jtype), int(g), f_used, float(got[2]),
                         float(job.size), float(job.finish_time)))

    M.MultiIngressPaperSimulator._handle_job_finish, M.energy_tuple = finish, energy_tuple
    try:
        res = ref_harness.run_reference(sc, seed, rng=rng)
    finally:
        M.MultiIngressPaperSimulator._handle_job_finish, M.energy_tuple = orig_fin, orig_et
    return jobs, res


def energy_bin(e):
    """clamp(floor(4 * log2(e)), 0, EBINS - 1), exactly (rational comparisons of e^4 with powers of two)."""
    if not e >= 1.0:
        return 0
    x, b = Fraction(e) ** 4, 0
    while b < EBINS - 1 and x >= 2 ** (b + 1):
        b += 1
    return b


def expected(jobs, sc):
    sp = S.to_spec(sc)                                 # (the scenario's levels and max_gpus_per_job as the library has them)
    n_dc = sp.n_dc
    bin_s, end = float(sc["log_interval"]), float(sc["duration"])
    W = max(1, math.ceil(end / bin_s))
    G = min(max(int(sp.max_gpus_per_job), 1), 32)
    levels = [[float(sp.dc[d].freq_levels[q]) for q in range(sp.dc[d].n_freq)] for d in range(n_dc)]
    rows = [[[[0.0, 0.0] for _ in range(n_dc)] for _ in range(3)] for _ in range(W + 1)]
    mix = [[[0] * (G * MAX_FREQ + 1) for _ in range(2)] for _ in range(n_dc)]
    hist = [[[0] * EBINS for _ in range(2)] for _ in range(n_dc)]
    for d, jt, g, f, e_pred, size, fin in jobs:
        e_job = e_pred * size
        k = min(math.floor(fin / bin_s), W - 1)
        for row in (k, W):
            rows[row][0][d][jt] += float(g)
            rows[row][1][d][jt] += f
            rows[row][2][d][jt] += e_job
        col = G * MAX_FREQ
        for q, lv in enumerate(levels[d]):
            if lv == f:
                col = (min(g, G) - 1) * MAX_FREQ + q
                break
        mix[d][jt][col] += 1
        hist[d][jt][energy_bin(e_job)] += 1
    hexed = [[[[v.hex() for v in c] for c in f] for f in r] for r in rows]
    return hexed, mix, hist


def main():
    out_dir = os.path.join(HERE, "jres")
    os.makedirs(out_dir, exist_ok=True)
    for sc in CASES:
        runs = list(RUNS) + ([(123, "mt")] if sc["name"] in MT_SCENARIOS else [])
        cases = []
        for seed, rng in runs:
            jobs, res = reference_jobs(sc, seed, rng)
            assert len(jobs) == res["jobs_finished"]
            rows, mix, hist = expected(jobs, sc)
            cases.append({"seed": seed, "rng": rng, "jobs_finished": res["jobs_finished"], "rows": rows, "mix": mix,
                          "hist": hist})
            print(f"{sc['name']:30s} {rng:6s} {seed}: finished {res['jobs_finished']:6d}")
        doc = {"meta": {"generator": "tests/golden/make_golden_jres.py",
                        "source": "unmodified reference, _handle_job_finish and energy_tuple wrapped"},
               "scenario": sc, "cases": cases}
        with open(os.path.join(out_dir, sc["name"] + ".json"), "w") as fh:
            json.dump(doc, fh, separators=(",", ":"))


if __name__ == "__main__":
    main()
