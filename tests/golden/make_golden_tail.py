"""Golden per-run tail-latency columns from the UNMODIFIED reference, for tests/test_tail_latency.py.

The reference runs through oracle/ref_harness.run_reference with three things wrapped at run time: the simulator
module's ``Job`` (every created job, its type and its ingress arrival instant — taken here because
``_handle_transfer_done`` overwrites ``job.arrival_time`` with the xfer_done instant, SIM:599), ``_schedule`` (the
xfer_done instant and the DC the arrival routed the job to, also when the instant lies past the end and the event is
dropped) and ``_handle_job_finish`` (start and finish of every job that finished).  The expected columns then come from
the plain loops below, written from the definition in include/dcsim_b200.h (not from the package): the q-quantile of n
values is the k-th smallest, k = max(ceil(n * q), 1).  Values are float.hex strings; NaN columns are null.

Build-container only (needs the reference tree):   DCSIM_REFERENCE_ROOT=... python tests/golden/make_golden_tail.py
"""
import json
import math
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))
from distributed_cluster_gpus_b200 import scenarios as S  # noqa: E402
import ref_harness  # noqa: E402

SLA_S = 0.5
QUANTILES = (0.5, 0.95, 0.99, 0.999)
CASES = [S.BY_NAME[n] for n in ("cfg3_4x64_sinusoid_120s", "short_0p3s_4x64", "underloaded_1x64", "all_off_2x8",
                                 "ragged_3dc_12_5_40", "cap_greedy_4x64", "sweep_eco_route")]
RUNS = [(123, "philox"), (124, "philox")]
MT_SCENARIOS = ("ragged_3dc_12_5_40", "cap_greedy_4x64")
TYPES = ("inference", "training")


def reference_jobs(sc, seed, rng):
    """-> ({jid: [jtype, dc, arrival, xfer_done, start, finish]} of every created job, reference result)."""
    ref_harness._import_reference()
    import simcore.simulator_paper_multi as M
    jobs = {}
    orig_job, orig_sched, orig_fin = M.Job, M.MultiIngressPaperSimulator._schedule, M.MultiIngressPaperSimulator._handle_job_finish

    def job(*a, **kw):
        j = orig_job(*a, **kw)
        jobs[j.jid] = [TYPES.index(j.jtype), None, float(j.arrival_time), math.inf, None, None]
        return j

    def schedule(self, t, etype, payload):
        if etype == "xfer_done":
            rec = jobs[payload["jid"]]
            rec[1], rec[3] = list(self.dcs.keys()).index(payload["dc"]), float(t)
        return orig_sched(self, t, etype, payload)

    def finish(self, dc_name, jid):
        tup = self.dcs[dc_name].running_jobs.get(jid)
        orig_fin(self, dc_name, jid)
        if tup:
            jobs[jid][4], jobs[jid][5] = float(tup[0].start_time), float(tup[0].finish_time)

    M.Job, M.MultiIngressPaperSimulator._schedule, M.MultiIngressPaperSimulator._handle_job_finish = job, schedule, finish
    try:
        res = ref_harness.run_reference(sc, seed, rng=rng)
    finally:
        M.Job, M.MultiIngressPaperSimulator._schedule, M.MultiIngressPaperSimulator._handle_job_finish = orig_job, orig_sched, orig_fin
    return jobs, res


def kth(values, q):
    v = sorted(values)
    return v[max(math.ceil(len(v) * q), 1) - 1]


def expected(jobs, n_dc):
    """The library's columns of one replica (DCSIM_TAIL_* order), None for NaN."""
    cols = []
    p99 = {}
    for jt in range(2):
        for dc in range(-1, n_dc):
            mine = [j for j in jobs.values() if j[0] == jt and (dc < 0 or j[1] == dc)]
            done = [j for j in mine if j[5] is not None]
            cols += [float(len(done)), float(len(mine) - len(done))]
            kinds = ([j[5] - j[4] for j in done], [j[4] - j[3] for j in done], [j[5] - j[2] for j in done])
            for k, vals in enumerate(kinds):
                if not vals:
                    cols += [None] * (len(QUANTILES) + 1)
                    continue
                cols += [kth(vals, q) for q in QUANTILES] + [max(vals)]
                if dc < 0:
                    p99[(k, jt)] = kth(vals, 0.99)
    for k in range(3):
        for jt in range(2):
            cols.append(None if (k, jt) not in p99 else (1.0 if p99[(k, jt)] <= SLA_S else 0.0))
    return cols


def main():
    out_dir = os.path.join(HERE, "tail")
    os.makedirs(out_dir, exist_ok=True)
    unfinished = empty = 0
    for sc in CASES:
        runs = list(RUNS) + ([(123, "mt")] if sc["name"] in MT_SCENARIOS else [])
        cases = []
        for seed, rng in runs:
            jobs, res = reference_jobs(sc, seed, rng)
            assert len(jobs) == res["jobs_created"]
            assert sum(j[5] is not None for j in jobs.values()) == res["jobs_finished"]
            assert all(j[1] is not None for j in jobs.values()), "a job without a routed DC"
            cols = expected(jobs, sc["n_dc"])
            unfinished += res["jobs_created"] - res["jobs_finished"]
            empty += sum(c is None for c in cols)
            cases.append({"seed": seed, "rng": rng, "jobs_created": res["jobs_created"],
                          "jobs_finished": res["jobs_finished"], "cols": [None if c is None else c.hex() for c in cols]})
            print(f"{sc['name']:30s} {rng:6s} {seed}: created {res['jobs_created']:6d} finished {res['jobs_finished']:6d}")
        doc = {"meta": {"generator": "tests/golden/make_golden_tail.py", "sla_s": SLA_S,
                        "source": "unmodified reference, Job / _schedule / _handle_job_finish wrapped"},
               "scenario": sc, "cases": cases}
        with open(os.path.join(out_dir, sc["name"] + ".json"), "w") as fh:
            json.dump(doc, fh, indent=1)
    assert unfinished > 0, "no run left a job unfinished"
    assert empty > 0, "no empty group"


if __name__ == "__main__":
    main()
