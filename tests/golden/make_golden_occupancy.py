"""Golden occupancy rows from the UNMODIFIED reference, for tests/test_occupancy.py.

The reference runs through oracle/ref_harness.run_reference with DataCenter.accrue_energy wrapped at run time (as
make_golden_power.py does): every call that accrues sees the DC's state before the event — len(q_inf), len(q_train),
len(running_jobs), busy_gpus — over (last_energy_time, now], tail included.  The expected columns then come from the
plain loop over levels below, written from the definition in include/dcsim_b200.h (not from the package).  Values are
float.hex strings; bins are stored sparse ({column: seconds}).

Build-container only (needs the reference tree):   DCSIM_REFERENCE_ROOT=... python tests/golden/make_golden_occupancy.py
"""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))
from distributed_cluster_gpus_b200 import scenarios as S  # noqa: E402
import ref_harness  # noqa: E402

F, B = 8, 128
EMPTY = dict(S.BY_NAME["cfg3_4x64_sinusoid_120s"], name="cfg3_ends_before_first_event", duration=1e-4)
CASES = [S.BY_NAME[n] for n in ("cfg1_1x4_poisson_5000s", "ragged_3dc_12_5_40", "cap_greedy_4x64", "eco_route_cap_2x16",
                                 "sweep_default_perf_first", "no_inf_priority_perf_first", "zero_xfer_4x64_sin10_60s",
                                 "underloaded_1x64", "all_off_2x8")] + [EMPTY]
# (ragged_3dc_12_5_40 and cap_greedy_4x64 hold queues far past bin 127: the generator asserts time in the last bin)
RUNS = [(123, "philox"), (124, "philox")]
MT_SCENARIOS = ("ragged_3dc_12_5_40", "cap_greedy_4x64")


def reference_intervals(sc, seed, rng):
    """-> (groups, reference result): groups = [(t_prev, t, [(qi, qt, n, b) per DC in DC order])]."""
    ref_harness._import_reference()
    from simcore.models import DataCenter
    calls = []
    orig = DataCenter.accrue_energy

    def recording(self, now, power_fn=None):
        last = getattr(self, "last_energy_time", 0.0)
        if last != 0.0:
            calls.append((last, now, (len(self.q_inf), len(self.q_train), len(self.running_jobs), self.busy_gpus)))
        return orig(self, now, power_fn)

    DataCenter.accrue_energy = recording
    try:
        res = ref_harness.run_reference(sc, seed, rng=rng)
    finally:
        DataCenter.accrue_energy = orig
    n_dc = sc["n_dc"]
    assert len(calls) % n_dc == 0
    groups = []
    for g in range(0, len(calls), n_dc):
        grp = calls[g:g + n_dc]
        assert all(c[0] == grp[0][0] and c[1] == grp[0][1] for c in grp), "the DCs of one accrual disagree on instants"
        groups.append((grp[0][0], grp[0][1], [c[2] for c in grp]))
    return groups, res


def expected(groups, end_time, totals):
    """The library's column [1 + 8 D + 256 D] of one replica, from levels of Qi, Qt, N, Q, B per DC."""
    D = len(totals)
    col = [0.0] * (1 + F * D + 2 * B * D)
    merged_b = 0                                       # intervals of B merged into a level that began earlier
    for d in range(D):
        w = (totals[d] + 1 + B - 1) // B
        fns = []
        for a, b, st in groups:
            if b > a:
                qi, qt, n, busy = st[d]
                fns.append((a, b, (qi, qt, n, qi + qt, busy)))
        for k in range(5):
            levels = []
            for a, b, v in fns:
                if levels and levels[-1][2] == v[k]:
                    levels[-1][1] = b
                else:
                    levels.append([a, b, v[k]])
            for s, e, v in levels:
                L = e - s
                if k == 0:
                    col[1 + 0 * D + d] += v * L
                    col[1 + 3 * D + d] = max(col[1 + 3 * D + d], float(v))
                elif k == 1:
                    col[1 + 1 * D + d] += v * L
                    col[1 + 4 * D + d] = max(col[1 + 4 * D + d], float(v))
                elif k == 2:
                    col[1 + 2 * D + d] += v * L
                elif k == 3:
                    if v > 0:
                        col[1 + 5 * D + d] += L
                    col[1 + F * D + d * B + min(v, B - 1)] += L
                else:
                    if v == totals[d]:
                        col[1 + 6 * D + d] += L
                    if v == 0:
                        col[1 + 7 * D + d] += L
                    col[1 + F * D + (D + d) * B + v // w] += L
            if k == 4:
                merged_b += len(fns) - len(levels)
    if groups:
        col[0] = end_time - groups[0][0]
    return col, merged_b


def main():
    out_dir = os.path.join(HERE, "occupancy")
    os.makedirs(out_dir, exist_ok=True)
    last_bin = merged = empty = 0
    for sc in CASES:
        runs = list(RUNS) + ([(123, "mt")] if sc["name"] in MT_SCENARIOS else [])
        sp = S.to_spec(sc)
        totals = [sp.dc[d].total_gpus for d in range(sc["n_dc"])]
        cases = []
        for seed, rng in runs:
            groups, res = reference_intervals(sc, seed, rng)
            col, mb = expected(groups, sc["duration"], totals)
            D = len(totals)
            last_bin += sum(col[1 + F * D + d * B + B - 1] > 0 for d in range(D))
            merged += mb
            empty += col[0] == 0.0
            for d in range(D):                         # each DC's queue and busy bins sum to PROFILE_S
                for o in (1 + F * D + d * B, 1 + F * D + (D + d) * B):
                    assert abs(sum(col[o:o + B]) - col[0]) <= 1e-9 * max(col[0], 1.0)
            cases.append({"seed": seed, "rng": rng, "events": res["events"],
                          "profile_s": col[0].hex(), "fields": [x.hex() for x in col[1:1 + F * D]],
                          "bins": {str(i): x.hex() for i, x in enumerate(col) if i >= 1 + F * D and x != 0.0}})
            print(f"{sc['name']:30s} {rng:6s} {seed}: profile {col[0]:9.3f} q_max {[col[1 + 3 * D + d] for d in range(D)]}")
        doc = {"meta": {"generator": "tests/golden/make_golden_occupancy.py",
                        "source": "unmodified reference, accrue_energy wrapped"}, "scenario": sc, "cases": cases}
        with open(os.path.join(out_dir, sc["name"] + ".json"), "w") as fh:
            json.dump(doc, fh, indent=1)
    assert last_bin > 0, "no queue reached the last bin"
    assert merged > 0, "no level of busy GPUs spans more than one inter-event interval"
    assert empty > 0, "no empty profile"


if __name__ == "__main__":
    main()
