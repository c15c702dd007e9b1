"""The arrival pre-pass and the list merge, entry by entry, on the host build of the device core.

The event loop reads nothing about jobs and transfers but what these two write: each replica's arrivals (arr_t,
arr_raw, arr_meta, arr_pred), the time-ordered {arrival, xfer_done} list (ml_t, ml_aux, ml_meta) and the header
(count, first_mask, rng_words, status, ml_count, max_ahead).  Two independent references pin them:

  * tests/list_reference.py builds the list from the heap's (t, push rank) rule, given the build's own arrivals.  The
    list must equal it byte for byte, header included.
  * tests/oracle_jobs/oracle_lists.c steps the C oracle one event at a time and records every arrival it processes.
    The arrivals must equal it bit for bit (the host build and the oracle use the same libm).

Each case checks from the reference data that it reaches the edge it is there for.  Run on the plain, warp-uniform and
small-ring (DCSIM_MERGE_RING = 32: every scan that leaves the chunk reads HBM) host builds.  tests/
test_arrival_lists_gpu.py holds the device to the same references."""
import ctypes as C
import os

import numpy as np
import pytest

import hostemu_lib as H
import list_reference as LR
import oracle_probes_lib as OP
from conftest import ROOT
from distributed_cluster_gpus_b200 import _native, scenarios as SC, spec as S

NO_PRED = LR.NO_PRED
ST_ARRIVALS_OVERFLOW = 32  # DCSIM_ST_ARRIVALS_OVERFLOW
MERGE_RING = 128           # DCSIM_MERGE_RING of the product build


def _short(name, duration=30.0, **kw):
    sc = dict(SC.BY_NAME[name])
    sc.update(kw)
    sc["duration"] = min(sc["duration"], duration)
    return sc


def huge_transfer_spec():
    """A finite transfer time far above any run (5e300 s) for one (DC, job type) of every ingress: such an xfer_done is
    scheduled by nobody and listed nowhere (SIM:161), like +inf."""
    sp = SC.to_spec(SC.scenario("mixed", 2, 8, SC.POI(2.0), SC.POI(0.5), 30.0))
    for i in range(sp.n_ing):
        sp.transfer_s[i][1][1] = 5e300
    return sp


def _end_on_grid(sp, end):
    sp.end_time = end
    return sp


# name -> (spec factory, replicas, key of replica 0, rng kind, time quantum)
CASES = {
    "cfg3": (lambda: SC.to_spec(_short("cfg3_4x64_sinusoid_120s")), 5, 123, 0, 0.0),
    "mt19937": (lambda: SC.to_spec(_short("cfg3_4x64_sinusoid_120s")), 3, 77, 1, 0.0),
    "eco_route": (lambda: SC.to_spec(_short("sweep_eco_route")), 3, 5, 0, 0.0),
    "zero_wan": (lambda: SC.to_spec(_short("cfg3_4x64_sinusoid_120s", wan=SC.ZERO_WAN)), 3, 9, 0, 0.0),
    "wan_1g": (lambda: SC.to_spec(_short("cfg3_4x64_sinusoid_120s", wan=SC.SLOW_WAN), caps={"cap_xfer": 4096}), 2, 31, 0, 0.0),
    "wan_0p075g": (lambda: SC.to_spec(_short("cfg3_4x64_sinusoid_120s", 120.0, wan=dict(capacity_gbps=0.075)),
                                      caps={"cap_xfer": 8192}), 2, 31, 0, 0.0),
    # the same lists against a 128-entry seq ring: the merge flags DCSIM_ST_XFER_OVERFLOW
    "xfer_ring_overflow": (lambda: SC.to_spec(_short("cfg3_4x64_sinusoid_120s", 30.0, wan=dict(capacity_gbps=0.075)),
                                              caps={"cap_xfer": 64}), 2, 31, 0, 0.0),
    "quantum_end_on_grid": (lambda: _end_on_grid(SC.to_spec(_short("cfg3_4x64_sinusoid_120s"), caps={"cap_xfer": 4096}), 30.0),
                            4, 900, 0, 0.25),
    "quantum_end_below_grid": (lambda: _end_on_grid(SC.to_spec(_short("cfg3_4x64_sinusoid_120s"), caps={"cap_xfer": 4096}),
                                                    30.0 - 0.5e-9), 8, 900, 0, 0.25),
    "huge_transfer": (huge_transfer_spec, 4, 123, 0, 0.0),
}


def list_ties(ml_t, ml_meta):
    """Adjacent list entries at the same instant, by class."""
    same = ml_t[1:] == ml_t[:-1]
    x0, x1 = (ml_meta[:-1] & 1) == 1, (ml_meta[1:] & 1) == 1
    return {"arrival_arrival": int(np.sum(same & ~x0 & ~x1)), "arrival_xfer": int(np.sum(same & (x0 != x1))),
            "xfer_xfer": int(np.sum(same & x0 & x1))}


def edge_reached(name, sp, lists, rows):
    """Asserts from the reference data that case `name` reaches its edge.  lists[r]: reference list of replica r; rows[r]:
    the oracle's arrivals."""
    end = sp.end_time
    if name == "eco_route":
        return
    if name == "xfer_ring_overflow":
        assert all(l["status"] == LR.ST_XFER_OVERFLOW for l in lists)
    if name == "zero_wan":
        assert all(np.array_equal(r["tx"], r["t"]) for r in rows), "every xfer_done at its arrival's instant"
    elif name in ("wan_1g", "wan_0p075g"):
        ahead = max(l["max_ahead"] for l in lists)
        tr = np.ctypeslib.as_array(sp.transfer_s)[:sp.n_ing, :sp.n_dc]
        tmax = float(tr[np.isfinite(tr)].max())
        window = max(int(np.max(np.searchsorted(r["t"], r["t"] + tmax, side="right") - np.arange(len(r)))) for r in rows)
        assert window > 2 * MERGE_RING, "stage 1 runs past the ring: at[k_last] comes from HBM"
        assert ahead >= (1000 if name == "wan_0p075g" else 200), ahead
    elif name.startswith("quantum"):
        ties = [list_ties(l["ml_t"], l["ml_meta"]) for l in lists]
        assert all(sum(t[k] for t in ties) > 0 for k in ties[0]), ties
        if name == "quantum_end_on_grid":
            assert any(np.any(l["ml_t"] == end) for l in lists), "instants exactly at end_time"
        else:
            grid = end + 0.5e-9
            late_x = sum(int(np.sum((r["tx"] == grid))) for r in rows)
            late_a = sum(int(np.sum(r["next"][r["t"] < grid] == 1)) - int(np.sum(r["pred"] != NO_PRED)) for r in rows)
            assert late_x > 0, "an xfer_done in (end, end + 1e-9]: it takes a seq but is not listed"
            assert late_a > 0, "an arrival in (end, end + 1e-9]: it takes a seq but is not listed"
    elif name == "huge_transfer":
        assert all(np.any(np.isinf(r["tx"]) & (r["dc"] < 0)) for r in rows)


def check_lists(sp, d, replicas, quantum):
    """The lists of `replicas` (rows of d) equal list_reference built from the same arrivals, byte for byte.  -> refs."""
    refs = []
    for r in replicas:
        h = d["hdr"][r]
        c, m = int(h["count"]), int(h["ml_count"])
        ref = LR.merge_spec(sp, d["arr_t"][r, :c], d["arr_meta"][r, :c], d["arr_pred"][r, :c], d["arr_raw"][r, :c], quantum)
        assert m == ref["ml_count"], (r, m, ref["ml_count"])
        for f in ("ml_t", "ml_aux"):
            got = d[f][r, :m].view(np.uint64)
            bad = np.flatnonzero(got != ref[f].view(np.uint64))
            assert len(bad) == 0, (r, f, bad[:5], got[bad[:5]], ref[f].view(np.uint64)[bad[:5]])
        bad = np.flatnonzero(d["ml_meta"][r, :m] != ref["ml_meta"])
        assert len(bad) == 0, (r, "ml_meta", bad[:5], d["ml_meta"][r, bad[:5]], ref["ml_meta"][bad[:5]])
        assert np.array_equal(d["arr_tx"][r, :c].view(np.uint64), ref["tx"].view(np.uint64)), r
        assert int(h["max_ahead"]) == ref["max_ahead"], r
        assert (int(h["status"]) & LR.ST_XFER_OVERFLOW) == ref["status"], r
        refs.append(ref)
    return refs


def ulp_distance(a, b):
    """Units in the last place between positive doubles."""
    return np.abs(a.view(np.int64) - b.view(np.int64))


def check_arrivals(sp, d, replicas, seed0, rng_kind, quantum, t_rtol=0.0, size_ulp=0):
    """Arrivals of `replicas` against the stepped oracle: meta, pred, next bit, count, first_mask and rng_words exact;
    t within t_rtol (0: bit for bit), sizes within size_ulp.  -> (oracle rows, worst t deviation, worst size ulp)."""
    out, worst_t, worst_ulp = [], 0.0, 0
    end_eps = sp.end_time + 1e-9
    for r in replicas:
        rows, first_mask, rng_words = OP.arrivals(sp.to_bytes(), seed0 + r, rng_kind, quantum)
        h = d["hdr"][r]
        c = int(h["count"])
        if int(h["status"]) & ST_ARRIVALS_OVERFLOW:
            assert c == sp.cap_arrivals and len(rows) > c, r     # the oracle's prefix
            rows = rows[:c]
        else:
            assert c == len(rows), (r, c, len(rows))
            assert int(h["rng_words"]) == rng_words, r
        assert int(h["first_mask"]) == first_mask, r
        meta, pred = d["arr_meta"][r, :c], d["arr_pred"][r, :c]
        assert np.array_equal(meta & 15, rows["stream"]), r
        assert np.array_equal(pred, rows["pred"]), r
        assert np.array_equal((meta >> 7) & 1, rows["next"]), r
        known = rows["dc"] >= 0
        assert np.array_equal(((meta >> 4) & 7)[known], rows["dc"][known]), r
        assert np.all(((meta >> 8) & 1) == int(sp.route_rule == S.ROUTE_ECO)), r   # the size was drawn before routing
        assert np.all(meta >> 9 == 0), r
        t = d["arr_t"][r, :c]
        if t_rtol == 0.0:
            assert np.array_equal(t, rows["t"]), r
        else:
            np.testing.assert_allclose(t, rows["t"], rtol=t_rtol, atol=0)
        if c:
            worst_t = max(worst_t, float(np.max(np.abs(t - rows["t"]) / np.maximum(rows["t"], 1e-300))))
            ulp = int(np.max(ulp_distance(d["arr_raw"][r, :c], rows["size"])))
            worst_ulp = max(worst_ulp, ulp)
            assert ulp <= size_ulp, (r, ulp)
        tx = d["arr_tx"][r, :c]
        pushed = (tx != np.inf) & ~(tx > end_eps)           # the merge's ML_A_XSCHED rule
        assert np.array_equal(pushed, np.isfinite(rows["tx"])), r
        np.testing.assert_allclose(tx[pushed], rows["tx"][pushed], rtol=t_rtol, atol=0)
        out.append(rows)
    return out, worst_t, worst_ulp


@pytest.mark.parametrize("variant", H.VARIANTS)
@pytest.mark.parametrize("name", list(CASES))
def test_lists_and_arrivals_match_references(name, variant):
    make, n, seed, rng, q = CASES[name]
    sp = make()
    d = H.prepass(sp.to_bytes(), n, seed, rng, variant, q)
    assert np.all((d["hdr"]["status"] | LR.ST_XFER_OVERFLOW) == LR.ST_XFER_OVERFLOW)
    refs = check_lists(sp, d, range(n), q)
    rows, _, _ = check_arrivals(sp, d, range(n), seed, rng, q)
    edge_reached(name, sp, refs, rows)
    print(f"{name} {variant}: counts {d['hdr']['count'].tolist()} max_ahead {d['hdr']['max_ahead'].tolist()}")


def test_eco_route_carries_sizes():
    """eco_route draws the size before routing and keeps it (meta bit 0x100); random routing keeps the raw draw."""
    for name, bit in (("eco_route", 1), ("cfg3", 0)):
        make, n, seed, rng, q = CASES[name]
        d = H.prepass(make().to_bytes(), n, seed, rng, "plain", q)
        for r in range(n):
            c = int(d["hdr"]["count"][r])
            assert c > 0 and np.all(((d["arr_meta"][r, :c] >> 8) & 1) == bit), name


def test_huge_finite_transfer_matches_oracle_end_to_end(oracle):
    """A finite transfer time above 1e300 s is left out of max_transfer; the merge must not count it as a listed
    transfer either.  Events, counts and floats equal the oracle."""
    sp = huge_transfer_spec()
    blob = sp.to_bytes()
    want, total = oracle.run_batch(blob, 4, 123, 0)
    for uniform in (False, True):
        got = H.run_batch(blob, 4, 123, uniform=uniform)
        assert got["events"] == total
        assert np.array_equal(got["summary"][:, S.S_EVENTS], want[:, S.S_EVENTS])
        assert np.all(got["summary"][:, S.S_STATUS] == 0)


COUNT_EDGES = (0, 1, 31, 32, 33, 127, 128, 129)


def count_edge_specs():
    """Low-rate batches whose arrival counts fall on the list's chunk and ring edges: mean ~1, ~32 and ~128."""
    return [SC.to_spec(SC.scenario(f"lowrate_{rate}", 2, 8, SC.POI(rate), SC.OFF, 10.0)) for rate in (0.05, 1.6, 6.4)]


COUNT_EDGE_BATCH = ((0, 24), (1, 160), (2, 320))   # (spec, replicas)


def test_arrival_counts_at_chunk_edges():
    seen = set()
    for (i, n), sp in zip(COUNT_EDGE_BATCH, count_edge_specs()):
        d = H.prepass(sp.to_bytes(), n, 4000 + i, 0, "smallring")
        counts = d["hdr"]["count"]
        seen |= set(int(c) for c in counts)
        pick = [r for r in range(n) if counts[r] in COUNT_EDGES]
        check_lists(sp, d, pick, 0.0)
        check_arrivals(sp, d, pick, 4000 + i, 0, 0.0)
    assert set(COUNT_EDGES) <= seen, sorted(set(COUNT_EDGES) - seen)


def test_arrival_capacity_edge_keeps_neighbours():
    """cap_arrivals at exactly one replica's count: that one is fine, one with more arrivals stops with the status bit and
    keeps the oracle's prefix, and every other row equals the default-capacity run."""
    sc = _short("cfg3_4x64_sinusoid_120s", 10.0)
    n, seed = 12, 600
    full = H.prepass(SC.to_spec(sc).to_bytes(), n, seed)
    counts = full["hdr"]["count"].astype(int)
    cap = int(np.sort(counts)[n // 2])
    sp = SC.to_spec(sc, caps={"cap_arrivals": cap})
    d = H.prepass(sp.to_bytes(), n, seed)
    over = counts > cap
    assert np.any(counts == cap) and np.any(over)
    assert np.array_equal((d["hdr"]["status"] & ST_ARRIVALS_OVERFLOW) != 0, over)
    check_arrivals(sp, d, range(n), seed, 0, 0.0)
    check_lists(sp, d, range(n), 0.0)
    for r in np.flatnonzero(~over):
        c, m = counts[r], int(full["hdr"]["ml_count"][r])
        for f in ("arr_t", "arr_raw", "arr_meta", "arr_pred"):
            assert np.array_equal(d[f][r, :c], full[f][r, :c]), (r, f)
        for f in ("ml_t", "ml_aux", "ml_meta"):
            assert np.array_equal(d[f][r, :m].view(np.uint8), full[f][r, :m].view(np.uint8)), (r, f)


def test_prepass_hooks_only_in_the_test_build():
    """The GPU build with the hooks (tests/gpuhooks, -DDCSIM_TEST_HOOKS) exports the pre-pass poison and fetch entry points
    test_arrival_lists_gpu.py uses; the product library and its header have neither."""
    import __graft_entry__ as G
    if not os.path.exists(G.HOOK_LIB):
        G.build()
    product, hook = C.CDLL(_native.LIB_PATH), C.CDLL(G.HOOK_LIB)
    with open(os.path.join(ROOT, "include", "dcsim_b200.h")) as f:
        header = f.read()
    for sym in ("dcsim_test_poison_prepass", "dcsim_test_fetch_prepass"):
        assert not hasattr(product, sym), sym
        assert hasattr(hook, sym), sym
        assert sym not in header, sym
