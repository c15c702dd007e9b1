"""Capacities at their edge on the host build of the device core (plain and warp-uniform skeleton): a replica overflows
a capacity exactly when its need exceeds it, gets the status bit and stops undone, and every replica that fits is
bit-identical to the oracle and to the same batch at default capacities.

The need of each replica is read from sources independent of the capacity checks: the oracle's S_MAX_Q, S_MAX_RUN and
S_EV_ARRIVAL (equal, replica by replica, to the pre-pass header's arrival count) and the list merge's max_ahead.  The
scenarios below were picked on the host build so that each batch straddles the boundaries it tests."""
import os

import numpy as np
import pytest

import hostemu_pair_lib as HP
from distributed_cluster_gpus_b200 import scenarios as SC, spec as S
from test_device_core_hostemu import _same

N = 48
# one DC held near saturation by rare 8-GPU training jobs for 3000 s: queues peak at 147..335 entries while ~3100
# arrivals pass through them, so a ring sized at the need wraps about ten times
QUEUE_SC = SC.scenario("queue_1x64_3000s", 1, 64, SC.POI(1.0), SC.POI(0.03), 3000.0)
# lightly loaded: the running set peaks anywhere from 1 to 8 jobs, replicas needing exactly 4 and 5 among them
RUN_SC = SC.scenario("run_1x64_300s", 1, 64, SC.POI(1.0), SC.POI(0.01), 300.0)
ARR_SC = SC.BY_NAME["ragged_3dc_12_5_40"]
# seq ring: at seed 97 the batch's max_ahead is 11..16 with 6 replicas at exactly 15 and 5 at exactly 16 (ring 16: the
# former fit, the latter overflow by one)
RING_SC, RING_SEED = SC.BY_NAME["ragged_3dc_12_5_40"], 97
# cap_greedy on one DC under a tight cap: at cap_stale 4 half of the batch overflows its stale-event pool, at 8 none
STALE_SC = SC.scenario("stale_cap_greedy_1x64_600s", 1, 64, SC.POI(1.0), SC.POI(0.03), 600.0, algo="cap_greedy",
                       power_cap=8000.0)
# WAN links at 0.075 Gbps (12 s per GB): every replica's xfer_done lies 8845..9182 list entries past its arrival, so a
# cap_xfer of 2100 (ring 8192) overflows and its doubling (ring 16384) fits
SLOW_WAN_SC = SC.scenario("wan_0p075g_4x64_90s", 4, 64, SC.SIN10, SC.POI(1.0), 90.0, SC.FREQ8,
                          wan=dict(capacity_gbps=0.075))
SEED = 5

BITS = {"queue": S.ST_QUEUE_OVERFLOW, "run": S.ST_RUN_OVERFLOW, "arrivals": S.ST_ARRIVALS_OVERFLOW,
        "ring": S.ST_XFER_OVERFLOW, "stale": S.ST_STALE_OVERFLOW}
SCENARIOS = {"queue": (QUEUE_SC, SEED), "run": (RUN_SC, SEED), "arrivals": (ARR_SC, SEED), "ring": (RING_SC, RING_SEED),
             "stale": (STALE_SC, SEED)}


def caps_for(kind, c):
    return {"queue": {"cap_q_inf": c, "cap_q_trn": c}, "run": {"cap_run": c}, "arrivals": {"cap_arrivals": c},
            "ring": {"cap_xfer": c}, "stale": {"cap_stale": c}}[kind]


def largest_fit(kind, c):
    """The largest need that capacity value `c` holds: cap_run and cap_stale round up to a multiple of 4; the seq ring
    is the smallest power of two >= 2 cap_xfer (at least 8) and holds entries up to ring - 1 ahead."""
    if kind in ("run", "stale"):
        return (c + 3) & ~3
    if kind == "ring":
        ring = 8
        while ring < 2 * c:
            ring <<= 1
        return ring - 1
    return c


def needs(oracle, kind):
    """(oracle summaries at default capacities, per-replica need of `kind`)."""
    sc, seed = SCENARIOS[kind]
    blob = SC.to_spec(sc).to_bytes()
    want, _ = oracle.run_batch(blob, N, seed, 0, n_threads=os.cpu_count() or 1)
    assert np.all(want[:, S.S_STATUS] == 0)
    _, hdr = HP.lists(blob, N, seed)
    assert np.array_equal(hdr["count"], want[:, S.S_EV_ARRIVAL])      # two independent counts of the same arrivals
    need = {"queue": want[:, S.S_MAX_Q], "run": want[:, S.S_MAX_RUN], "arrivals": hdr["count"],
            "ring": hdr["max_ahead"], "stale": None}[kind]
    return want, (None if need is None else need.astype(np.int64))


def edge_caps(kind, need):
    """Capacity values: exact fit of the batch's largest need, one short of it, and one near the median need."""
    top, med = int(need.max()), int(np.median(need))
    if kind == "run":       # effective capacities are multiples of 4: 4 sits on the boundary between needs 4 and 5
        assert top % 4 == 0 and np.any(need == 4) and np.any(need == 5), need
        return [top, top - 3, 4, 1]     # top - 3 and 1 round up to top and 4
    if kind == "ring":      # smallest ring above the largest need, and the ring that the largest need overflows by one
        assert top == 16 and np.any(need == 15), need
        return [16, 8, 5]               # rings 32, 16, 16
    return [top, top - 1, med]


def flagged(summ, bit):
    return (summ[:, S.S_STATUS].astype(np.int64) & bit) != 0


def check_edge(got, want, need_fits, bit, what):
    """Exactly the replicas that do not fit carry the bit (and no other); the others equal `want`.  (S_DONE of a
    replica that overflowed is 0 unless its end_time came before the next status poll, at most 16 events later: the
    event loop then finishes it as usual, so the status bit, not S_DONE, is what marks it failed.)"""
    over = ~need_fits
    assert np.array_equal(flagged(got, bit), over), (what, np.flatnonzero(flagged(got, bit)), np.flatnonzero(over))
    assert np.all(got[over, S.S_STATUS] == bit), what
    assert _same(got[~over], want[~over]), (what, np.argwhere(got[~over] != want[~over])[:6])


@pytest.mark.parametrize("uniform", [False, True], ids=["plain", "uniform"])
@pytest.mark.parametrize("kind", ["queue", "run", "arrivals", "ring"])
def test_capacity_at_need(oracle, hostemu, kind, uniform):
    """Exact fit, one short, near the median: flagged set == {r : need[r] > capacity}, every other row == the oracle's
    and == the default-capacity run's, bit for bit."""
    sc, seed = SCENARIOS[kind]
    want, need = needs(oracle, kind)
    base = hostemu.run_batch(SC.to_spec(sc).to_bytes(), N, seed, uniform=uniform)["summary"]
    assert _same(base, want)
    seen_fit, seen_over = set(), set()
    for c in edge_caps(kind, need):
        fit = largest_fit(kind, c)
        res = hostemu.run_batch(SC.to_spec(sc, caps=caps_for(kind, c)).to_bytes(), N, seed, uniform=uniform)
        got = res["summary"]
        check_edge(got, want, need <= fit, BITS[kind], (kind, c))
        assert np.array_equal(got[need <= fit], base[need <= fit])
        if kind == "run":
            assert res["layout"]["cap_run"] == fit
        seen_fit |= set(np.flatnonzero(need == fit))
        seen_over |= set(np.flatnonzero(need == fit + 1))
    assert seen_fit and seen_over, "no replica sat exactly on a boundary"       # the off-by-one is observable


@pytest.mark.parametrize("uniform", [False, True], ids=["plain", "uniform"])
def test_queue_rings_wrap_at_exact_fit(oracle, hostemu, uniform):
    """The FIFO rings at exactly the batch's largest need go round many times (head + length past the end)."""
    want, need = needs(oracle, "queue")
    jobs = want[:, S.S_JOBS_CREATED]
    assert np.all(jobs > 8 * need.max()), "the rings would not wrap several times"
    got = hostemu.run_batch(SC.to_spec(QUEUE_SC, caps=caps_for("queue", int(need.max()))).to_bytes(), N, SEED,
                            chunk_events=997, uniform=uniform)["summary"]
    check_edge(got, want, np.ones(N, bool), BITS["queue"], "queue, chunked")


def test_stale_pool_edge(oracle, hostemu):
    """No need column for the stale-event pool: at cap_stale 4 (and 1, which rounds up to 4) both host builds flag the
    same replicas, about half of the batch; the rest equal the oracle.  At 8 nothing overflows."""
    want, _ = needs(oracle, "stale")
    sets = []
    for c in (4, 1, 8):
        blob = SC.to_spec(STALE_SC, caps=caps_for("stale", c)).to_bytes()
        plain = hostemu.run_batch(blob, N, SEED)["summary"]
        uni = hostemu.run_batch(blob, N, SEED, uniform=True)["summary"]
        over = flagged(plain, S.ST_STALE_OVERFLOW)
        check_edge(plain, want, ~over, S.ST_STALE_OVERFLOW, ("stale plain", c))
        check_edge(uni, want, ~over, S.ST_STALE_OVERFLOW, ("stale uniform", c))
        sets.append(over)
    assert np.array_equal(sets[0], sets[1]) and 8 <= sets[0].sum() <= N - 8 and not sets[2].any()


def test_slow_wan_ring_need_straddles_8192():
    """The scenario of the device's staged -> in-place XFER retry: every replica's seq-ring need is in [8192, 16384)."""
    _, hdr = HP.lists(SC.to_spec(SLOW_WAN_SC).to_bytes(), 8, 3)
    assert np.all(hdr["status"] == 0) and np.all((hdr["max_ahead"] >= 8192) & (hdr["max_ahead"] < 16384))
    assert largest_fit("ring", 2100) == 8191 and largest_fit("ring", 4200) == 16383
