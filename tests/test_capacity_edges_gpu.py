"""Capacities at their edge on the H100 (the scenarios and needs of tests/test_capacity_edges.py): mixed batches in
which some lane groups of a warp stop on a status bit while their warp-mates run on, on 8 and 32 lanes — the arrival
capacity also through the pre-pass's warp-staged flush — and the engine's capacity retry from a too-small value of each
capacity, including one XFER retry that takes an 8-lane launch from staged shared memory to in place."""
import numpy as np
import pytest

from conftest import has_cuda
from distributed_cluster_gpus_b200 import scenarios as SC, spec as S
from test_capacity_edges import (BITS, N, SCENARIOS, SLOW_WAN_SC, caps_for, edge_caps, flagged, largest_fit, needs)
from test_gpu_parity import assert_rows_match

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not has_cuda(), reason="needs a CUDA device")]

HIGH_WATER = (S.S_MAX_RUN, S.S_MAX_Q, S.S_UTIL_BEGIN)


def run(sp, n, seed):
    from distributed_cluster_gpus_b200.engine import BatchedEngine
    with BatchedEngine(sp, n, base_seed=seed) as eng:
        eng.advance(0)
        return eng.summary(), eng.launch_info()


def check_edge(got, want, base, over, bit, n_dc, what):
    """Exactly `over` carries the bit (and no other); every other replica equals the oracle (counts and high-water
    marks exact, floats within 1e-9) and the default-capacity batch bit for bit."""
    assert np.array_equal(flagged(got, bit), over), (what, np.flatnonzero(flagged(got, bit)), np.flatnonzero(over))
    assert np.all(got[over, S.S_STATUS] == bit), what
    ok = ~over
    assert_rows_match(got[ok], want[ok], n_dc)
    for col in HIGH_WATER:
        assert np.array_equal(got[ok, col], want[ok, col]), (what, col)
    assert np.array_equal(got[ok].view(np.uint64), base[ok].view(np.uint64)), what


@pytest.mark.parametrize("lanes", [8, 32])
@pytest.mark.parametrize("kind", ["queue", "run", "arrivals", "ring"])
def test_capacity_at_need(oracle, monkeypatch, kind, lanes):
    monkeypatch.setenv("DCSIM_GROUP", str(lanes))
    sc, seed = SCENARIOS[kind]
    want, need = needs(oracle, kind)
    base, info = run(SC.to_spec(sc), N, seed)
    assert info["lanes_per_replica"] == lanes
    check_edge(base, want, base, np.zeros(N, bool), BITS[kind], sc["n_dc"], (kind, "default"))
    for c in edge_caps(kind, need):
        got, _ = run(SC.to_spec(sc, caps=caps_for(kind, c)), N, seed)
        check_edge(got, want, base, need > largest_fit(kind, c), BITS[kind], sc["n_dc"], (kind, c))


@pytest.mark.parametrize("lanes", [8, 32])
def test_stale_pool_edge(oracle, hostemu, monkeypatch, lanes):
    """The flagged set is the host build's (warp-uniform skeleton) at the same capacity."""
    monkeypatch.setenv("DCSIM_GROUP", str(lanes))
    sc, seed = SCENARIOS["stale"]
    want, _ = needs(oracle, "stale")
    base, _ = run(SC.to_spec(sc), N, seed)
    for c in (4, 8):
        sp = SC.to_spec(sc, caps=caps_for("stale", c))
        over = flagged(hostemu.run_batch(sp.to_bytes(), N, seed, uniform=True)["summary"], S.ST_STALE_OVERFLOW)
        got, _ = run(sp, N, seed)
        check_edge(got, want, base, over, S.ST_STALE_OVERFLOW, sc["n_dc"], ("stale", c))


def _next_cap(kind, c):
    """raise_caps on one capacity: cap_run jumps to the largest DC's GPU count (64 here), cap_stale to 2 max(64, c),
    the others double."""
    return {"run": 64, "stale": 2 * max(64, c)}.get(kind, 2 * c)


@pytest.mark.parametrize("kind,start", [("queue", 40), ("run", 4), ("arrivals", 500), ("ring", 2), ("stale", 4)])
def test_retry_from_too_small(oracle, kind, start):
    """run_to_completion from a too-small capacity: one attempt per raise until the batch's largest need fits (stale:
    the host build's verdict), and the final summaries equal a default-capacity batch bit for bit."""
    from distributed_cluster_gpus_b200 import engine as E
    sc, seed = SCENARIOS[kind]
    want, need = needs(oracle, kind)
    if kind == "stale":
        expected = 2                               # 4 -> 128; the host build clears the batch from 8 up
    else:
        expected, c = 1, start
        while largest_fit(kind, c) < need.max():
            c, expected = _next_cap(kind, c), expected + 1
    assert expected >= 2
    attempts = []

    def factory(caps):
        attempts.append(dict(caps))
        return SC.to_spec(sc, caps={**caps_for(kind, start), **caps})
    E.free_cached_engine()
    eng, summ = E.run_to_completion(factory, N, seed, max_retries=8)
    eng.close()
    E.free_cached_engine()
    base, _ = run(SC.to_spec(sc), N, seed)
    assert len(attempts) == expected, attempts
    assert np.array_equal(summ.view(np.uint64), base.view(np.uint64))
    assert_rows_match(summ, want, sc["n_dc"])


def test_xfer_retry_crosses_from_staged_into_in_place(oracle, monkeypatch):
    """8 lanes, cap_xfer 2100 (ring 8192, four heads fit a CTA's shared memory) overflows on every replica (need
    8845..9182); the retry's 4200 (ring 16384, 64 kB per head) no longer fits and runs in place."""
    from distributed_cluster_gpus_b200 import engine as E
    monkeypatch.setenv("DCSIM_GROUP", "8")
    modes = []

    def factory(caps):
        return SC.to_spec(SLOW_WAN_SC, caps={"cap_xfer": 2100, **caps})
    E.free_cached_engine()
    eng, summ = E.run_to_completion(factory, 8, 3, configure=lambda e: modes.append(e.launch_info()["staging_mode"]))
    eng.close()
    E.free_cached_engine()
    assert modes[0] in (1, 2) and modes[1:] == [0], modes
    base, info = run(SC.to_spec(SLOW_WAN_SC), 8, 3)
    assert info["staging_mode"] == 0 and info["lanes_per_replica"] == 8
    assert np.array_equal(summ.view(np.uint64), base.view(np.uint64))
    want, _ = oracle.run_batch(SC.to_spec(SLOW_WAN_SC).to_bytes(), 8, 3)
    assert_rows_match(summ, want, 4)
