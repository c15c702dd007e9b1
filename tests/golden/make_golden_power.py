"""Golden power profiles from the UNMODIFIED reference, for tests/test_power_profile*.py.

The reference runs through oracle/ref_harness.run_reference with DataCenter.accrue_energy wrapped at run time (as the
harness wraps _pop and _handle_job_finish): the wrapper records (last_energy_time, now, p) of every call that accrues,
i.e. exactly the power the reference integrates, tail included.  The expected fields and bins then come from the plain
loop below, written from the definition in include/dcsim_b200.h (not from the package's numpy mirror).  The histogram
range hi is the library's (dcsim_pp_range through the host build); it is stored so the tests also pin it.  Values are
float.hex strings; bins are stored sparse ({index: seconds}).

Build-container only (needs the reference tree):   DCSIM_REFERENCE_ROOT=... python tests/golden/make_golden_power.py
"""
import json
import math
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
from distributed_cluster_gpus_b200 import scenarios as S  # noqa: E402
import ref_harness  # noqa: E402
import hostemu_pp_lib  # noqa: E402

FIELDS = ["profile_s", "peak_w", "t_peak_s", "over_s", "over_j", "excursions", "longest_over_s", "out_of_range"]
BINS = 1024
INF = float("inf")
EMPTY = dict(S.BY_NAME["all_off_2x8"], name="all_off_2x8_1s_empty", duration=1.0)  # ends before the first log tick

# (scenario, threshold rule): "cap" = the scenario's power cap; ("level", q) = halfway between two adjacent distinct
# level powers around quantile q of the first run; "above" = 5 % over that run's peak (never crossed); "inf" = none
CASES = [
    (S.BY_NAME["cfg3_4x64_sinusoid_120s"], ("level", 0.8)),
    (S.BY_NAME["cap_greedy_4x64"], "cap"),
    (S.BY_NAME["cap_uniform_4x64"], "cap"),
    (S.BY_NAME["eco_route_cap_2x16"], "cap"),
    (S.BY_NAME["sweep_joint_nf"], ("level", 0.9)),
    (S.BY_NAME["ragged_3dc_12_5_40"], ("level", 0.5)),
    (S.BY_NAME["zero_xfer_4x64_sin10_60s"], ("level", 0.75)),
    (S.BY_NAME["short_0p3s_4x64"], "above"),
    (S.BY_NAME["all_off_2x8"], "inf"),
    (EMPTY, 1000.0),
]
RUNS = [(123, "philox"), (124, "philox")]
MT_SCENARIOS = ("cfg3_4x64_sinusoid_120s", "cap_greedy_4x64")


def reference_intervals(sc, seed, rng):
    """-> (groups, reference result): groups = [(t_prev, t, [p_d in DC order])], one per accruing event and the tail."""
    ref_harness._import_reference()
    from simcore.models import DataCenter
    calls = []
    orig = DataCenter.accrue_energy

    def recording(self, now, power_fn=None):
        last = getattr(self, "last_energy_time", 0.0)
        if last != 0.0:
            p = power_fn(self) if power_fn else self.instantaneous_power_w()
            calls.append((self.name, last, now, p))
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
        assert all(c[1] == grp[0][1] and c[2] == grp[0][2] for c in grp), "the DCs of one accrual disagree on instants"
        groups.append((grp[0][1], grp[0][2], [c[3] for c in grp]))
    return groups, res


def levels_of(groups):
    lv = []
    for a, b, ps in groups:
        if not b > a:
            continue
        p = 0.0
        for x in ps:
            p += x
        if lv and lv[-1][2].hex() == p.hex():
            lv[-1][1] = b
        else:
            lv.append([a, b, p])
    return lv


def expected(groups, end_time, n_dc, hi, thr):
    lv = levels_of(groups)
    dc_peak = [0.0] * n_dc
    first = True
    for a, b, ps in groups:
        if not b > a:
            continue
        for d in range(n_dc):
            if first or ps[d] > dc_peak[d]:
                dc_peak[d] = ps[d]
        first = False
    f = dict.fromkeys(FIELDS, 0.0)
    bins = [0.0] * BINS
    run_s = None
    width = hi / BINS
    for i, (s, e, p) in enumerate(lv):
        L = e - s
        k = math.floor(p / width)
        b = min(BINS - 1, max(0, k))
        if not (0.0 <= p <= hi):
            f["out_of_range"] += 1.0
        bins[b] += L
        if i == 0 or p > f["peak_w"]:
            f["peak_w"], f["t_peak_s"] = p, s
        if p > thr:
            f["over_s"] += L
            f["over_j"] += (p - thr) * L
            if run_s is None:
                run_s = s
                f["excursions"] += 1.0
        elif run_s is not None:
            f["longest_over_s"] = max(f["longest_over_s"], s - run_s)
            run_s = None
    if lv and run_s is not None:
        f["longest_over_s"] = max(f["longest_over_s"], lv[-1][1] - run_s)
    if groups:
        f["profile_s"] = end_time - groups[0][0]
    return f, dc_peak, bins, lv


def pick_threshold(rule, sc, lv):
    if rule == "cap":
        return float(sc["power_cap"])
    if rule == "inf":
        return INF
    if rule == "above":
        return max(p for _, _, p in lv) * 1.05
    if isinstance(rule, float):
        return rule
    q = rule[1]
    ps = sorted({p for _, _, p in lv})
    i = min(len(ps) - 2, int(q * (len(ps) - 1)))
    return 0.5 * (ps[i] + ps[i + 1])


def main():
    out_dir = os.path.join(HERE, "power")
    os.makedirs(out_dir, exist_ok=True)
    crossing = never = inf_case = False
    for sc, rule in CASES:
        spec = S.to_spec(sc).to_bytes()
        hi = hostemu_pp_lib.power_range(spec)
        runs = list(RUNS) + ([(123, "mt")] if sc["name"] in MT_SCENARIOS else [])
        thr = None
        cases = []
        for seed, rng in runs:
            groups, res = reference_intervals(sc, seed, rng)
            lv = levels_of(groups)
            if thr is None:
                thr = pick_threshold(rule, sc, lv)
            f, dc_peak, bins, lv = expected(groups, sc["duration"], sc["n_dc"], hi, thr)
            # no level within 1e-9 of the threshold, and a peak no other level comes within 1e-9 of: the last bits of
            # libdevice vs glibc cannot flip a comparison on the GPU
            for _, _, p in lv:
                assert thr == INF or abs(p - thr) > 1e-9 * abs(thr), (sc["name"], seed, rng, "level at the threshold")
                assert p.hex() == f["peak_w"].hex() or p < f["peak_w"] * (1 - 1e-9), (sc["name"], seed, rng, "peak not unique")
            energy = float.fromhex(res["total_energy_j"])
            lsum = math.fsum(p * (e - s) for s, e, p in lv)
            assert abs(lsum - energy) <= 1e-12 * max(abs(energy), 1.0), (sc["name"], seed, rng, lsum, energy)
            assert abs(math.fsum(bins) - f["profile_s"]) <= 1e-12 * max(f["profile_s"], 1.0)
            crossing |= f["over_s"] > 0 and f["excursions"] >= 2
            never |= thr != INF and f["over_s"] == 0.0 and bool(lv)
            inf_case |= thr == INF and bool(lv)
            cases.append({"seed": seed, "rng": rng, "levels": len(lv), "events": res["events"],
                          "fields": {k: v.hex() for k, v in f.items()}, "dc_peak_w": [x.hex() for x in dc_peak],
                          "bins": {str(i): x.hex() for i, x in enumerate(bins) if x != 0.0},
                          "total_energy_j": res["total_energy_j"]})
            print(f"{sc['name']:28s} {rng:6s} {seed}: levels {len(lv):6d} peak {f['peak_w']:10.1f} over_s {f['over_s']:8.3f} "
                  f"excursions {int(f['excursions'])}")
        if sc["name"] == "cap_greedy_4x64":
            assert any(float.fromhex(c["fields"]["over_s"]) > 0 and float.fromhex(c["fields"]["excursions"]) >= 2
                       for c in cases), "cap_greedy_4x64 never crossed its cap twice"
        doc = {"meta": {"generator": "tests/golden/make_golden_power.py", "source": "unmodified reference, accrue_energy wrapped"},
               "scenario": sc, "threshold": thr.hex() if thr != INF else "inf", "hi": hi.hex(), "cases": cases}
        with open(os.path.join(out_dir, sc["name"] + ".json"), "w") as fh:
            json.dump(doc, fh, indent=1)
    assert crossing and never and inf_case, (crossing, never, inf_case)


if __name__ == "__main__":
    main()
