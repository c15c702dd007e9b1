"""Golden energy cost and carbon from the UNMODIFIED reference, for tests/test_energy_cost*.py.

The reference runs through oracle/ref_harness.run_reference with DataCenter.accrue_energy wrapped at run time, exactly as
make_golden_power.py does (its reference_intervals): every call that accrues records (last_energy_time, now, p) per DC,
i.e. the power the reference integrates, tail included.  The tariff and carbon intensity come from the reference too:
its own _price_kwh resolved at every hour of the day and carbon.get(name, 0.0) (SIM:625).  The expected columns then
come from the plain loop below, written from the definition in include/dcsim_b200.h (not from the package's mirror).
A scenario with an "energy_price" key runs the reference under that per-DC tariff instead of paper_config's.  Values are
float.hex strings.

It also writes the CSVs of the numpy mirror (ensemble.energy_cost_from_rows) on seeded rows, CSV_CASES, which
tests/test_energy_cost.py pins byte for byte; `--csv` writes only those (no reference needed).

Build-container only (needs the reference tree):   DCSIM_REFERENCE_ROOT=... python tests/golden/make_golden_cost.py
"""
import json
import math
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))
sys.path.insert(0, HERE)
from distributed_cluster_gpus_b200 import ensemble as EN, scenarios as S, spec as SP  # noqa: E402
import ref_harness  # noqa: E402
from make_golden_power import EMPTY, reference_intervals  # noqa: E402

HOURS = 24
# a light load over more than a day: its hours fold across days
LIGHT_27H = S.scenario("light_2x8_27h", 2, 8, S.POI(0.004), S.POI(0.0004), 97200.0, S.FREQ8, log_interval=1800.0)
# a per-DC tariff: hourly prices for us-west, a few hours for us-east (the others 0.0), none for eu-west
TARIFF = S.scenario("tariff_per_dc_3dc_3h", 3, None, S.POI(0.3), S.POI(0.03), 10800.0, S.FREQ8, algo="carbon_cost",
                    log_interval=600.0, gpus_list=[12, 5, 40],
                    energy_price={"us-west": {h: 0.05 + 0.01 * h for h in range(HOURS)},
                                  "us-east": {0: 0.30, 1: 0.07, 2: 0.11}})
CASES = [
    S.BY_NAME["carbon_cost_8h_2x16"],     # crosses the 07:00 tariff step; log ticks land on hour boundaries
    LIGHT_27H,
    TARIFF,
    S.BY_NAME["cap_greedy_4x64"],         # the controller's DF_POWER writes
    S.BY_NAME["cfg3_4x64_sinusoid_120s"],  # shorter than one hour
    S.BY_NAME["short_0p3s_4x64"],
    EMPTY,                                # ends before the first event
]
RUNS = [(123, "philox"), (124, "philox")]
MT_SCENARIOS = ("carbon_cost_8h_2x16", "cap_greedy_4x64")


def reference_tables(sc):
    """-> (price [n_dc][24], carbon [n_dc], DC names) as the reference resolves them."""
    Sim = ref_harness._import_reference()[0]
    kw = ref_harness.build_reference_inputs(sc)
    names = list(kw["dcs"])
    price = []
    for name in names:
        row = []
        for h in range(HOURS):
            stub = types.SimpleNamespace(energy_price=kw["energy_price"], now=3600.0 * h)
            stub._current_hour = types.MethodType(Sim._current_hour, stub)
            row.append(Sim._price_kwh(stub, name))
        price.append(row)
    carbon = [(kw["carbon_intensity"] or {}).get(name, 0.0) for name in names]
    return price, carbon, names


def window(a):
    k = math.floor(a / 3600.0)
    if 3600.0 * k > a:
        k -= 1
    elif 3600.0 * (k + 1) <= a:
        k += 1
    return k


def expected(groups, n_dc, price, carbon):
    """The columns of include/dcsim_b200.h from the per-DC accruals: levels, hour pieces, sums in the stated orders."""
    E = [[0.0] * HOURS for _ in range(n_dc)]
    n_levels = [0] * n_dc
    pieces_per_hour = [0] * HOURS
    for d in range(n_dc):
        levels = []
        for a, b, ps in groups:
            if not b > a:
                continue
            p = ps[d]
            if levels and levels[-1][2].hex() == p.hex():
                levels[-1][1] = b
            else:
                levels.append([a, b, p])
        n_levels[d] = len(levels)
        for s, e, p in levels:
            k, a = window(s), s
            while True:
                b = 3600.0 * (k + 1)
                cut = b < e
                E[d][k % HOURS] += p * ((b if cut else e) - a)
                pieces_per_hour[k % HOURS] += 1
                if not cut:
                    break
                a, k = b, k + 1
    cols = {"hour_j": E, "energy_j": [], "cost_usd": [], "carbon_g": []}
    tot = [0.0, 0.0, 0.0]
    for d in range(n_dc):
        ej = usd = 0.0
        for h in range(HOURS):
            ej += E[d][h]
            usd += (E[d][h] / 3.6e6) * price[d][h]
        g = (ej / 3.6e6) * carbon[d]
        cols["energy_j"].append(ej)
        cols["cost_usd"].append(usd)
        cols["carbon_g"].append(g)
        tot[0] += ej
        tot[1] += usd
        tot[2] += g
    cols["total_j"], cols["total_usd"], cols["total_g"] = tot
    return cols, n_levels, pieces_per_hour


def _hex(x):
    return [_hex(v) for v in x] if isinstance(x, list) else x.hex()


def _mirror_csv(path, good):
    """Seeded per-replica columns of 3 DCs (the second absent from the carbon map), derived as the header states,
    replicas with good == False failed -> the mirror's CSV."""
    rng = np.random.default_rng(31)
    n_dc, R = 3, len(good)
    price = [[0.12 if h < 7 else 0.20 if h < 19 else 0.16 for h in range(HOURS)], [0.10] * HOURS,
             [0.05 + 0.01 * h for h in range(HOURS)]]
    carbon = [350.0, 0.0, 220.0]
    rows = np.zeros((SP.cost_cols(n_dc), R))
    for r in range(R):
        E = rng.uniform(0.0, 2e6, size=(n_dc, HOURS)) * (rng.uniform(size=(n_dc, HOURS)) < 0.8)
        tot = [0.0, 0.0, 0.0]
        for d in range(n_dc):
            ej = usd = 0.0
            for h in range(HOURS):
                rows[SP.cost_hour_j(n_dc, d, h), r] = E[d, h]
                ej += E[d, h]
                usd += (E[d, h] / 3.6e6) * price[d][h]
            g = (ej / 3.6e6) * carbon[d]
            rows[[SP.cost_energy_j(n_dc, d), SP.cost_usd(n_dc, d), SP.cost_carbon_g(n_dc, d)], r] = ej, usd, g
            tot = [tot[0] + ej, tot[1] + usd, tot[2] + g]
        rows[list(SP.cost_totals(n_dc)), r] = tot
    status = np.where(good, 0, 4)
    EN.energy_cost_from_rows(rows, status, price, carbon).to_csv(path, ["us-west", "us-east", "eu-west"])


CSV_CASES = {
    "energy_cost_mixed.csv": lambda p: _mirror_csv(p, np.array([1, 1, 0, 1, 1, 1, 0, 1, 1], dtype=bool)),
    "energy_cost_one_replica.csv": lambda p: _mirror_csv(p, np.arange(9) == 4),
    "energy_cost_no_replica.csv": lambda p: _mirror_csv(p, np.zeros(9, dtype=bool)),
}


def write_csvs(out_dir):
    os.makedirs(out_dir, exist_ok=True)
    for name, fn in CSV_CASES.items():
        fn(os.path.join(out_dir, name))


def main():
    orig_inputs = ref_harness.build_reference_inputs

    def with_tariff(sc):
        kw = orig_inputs(sc)
        if "energy_price" in sc:
            kw["energy_price"] = S.energy_price_of(sc)
        return kw

    ref_harness.build_reference_inputs = with_tariff
    out_dir = os.path.join(HERE, "cost")
    os.makedirs(out_dir, exist_ok=True)
    for sc in CASES:
        price, carbon, names = reference_tables(sc)
        runs = list(RUNS) + ([(123, "mt")] if sc["name"] in MT_SCENARIOS else [])
        cases = []
        for seed, rng in runs:
            groups, res = reference_intervals(sc, seed, rng)
            cols, n_levels, pieces = expected(groups, sc["n_dc"], price, carbon)
            for d in range(sc["n_dc"]):
                ref_j = float.fromhex(res["dc"][d]["energy_j"])
                assert abs(cols["energy_j"][d] - ref_j) <= 1e-10 * max(abs(ref_j), 1.0), (sc["name"], seed, rng, d)
            cases.append({"seed": seed, "rng": rng, "events": res["events"], "levels": n_levels,
                          "hours_reached": [h for h in range(HOURS) if pieces[h]],
                          "dc_energy_j": [dc["energy_j"] for dc in res["dc"]],
                          "cols": {k: _hex(v) for k, v in cols.items()}})
            print(f"{sc['name']:28s} {rng:6s} {seed}: events {res['events']:7d} levels {n_levels} "
                  f"hours {len(cases[-1]['hours_reached']):2d} USD {cols['total_usd']:.6f} g {cols['total_g']:.3f}")
        doc = {"meta": {"generator": "tests/golden/make_golden_cost.py",
                        "source": "unmodified reference, accrue_energy wrapped; _price_kwh and carbon.get per DC"},
               "scenario": sc, "dc_names": names, "price_kwh": _hex(price), "carbon_intensity": _hex(carbon),
               "cases": cases}
        with open(os.path.join(out_dir, sc["name"] + ".json"), "w") as fh:
            json.dump(doc, fh, indent=1)


if __name__ == "__main__":
    write_csvs(os.path.join(HERE, "cost"))
    if "--csv" not in sys.argv:
        main()
