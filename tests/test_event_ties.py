"""Events at the SAME instant: the heap orders them by seq (SIM:163), i.e. by push order.

A continuous clock all but never produces such ties (two arrival streams landing on one double: ~ rate * ulp(t) per
arrival — rare per replica, not rare over 10^5 replicas x hours), so they are provoked here: a test hook in the oracle
and in the host build of the device core rounds every arrival and xfer_done instant up to a multiple of a quantum.
The oracle then resolves the ties with its heap; the device core has to reproduce that order from list indices alone —
in the arrival pre-pass (two streams due at the same instant) and in the list merge (arrival vs xfer_done, xfer_done
vs xfer_done).  Everything must stay bit-identical: summaries, the seq of every traced event, both logs."""
import os

import numpy as np
import pytest

from conftest import ROOT

from distributed_cluster_gpus_b200 import scenarios as SC, spec as S
from distributed_cluster_gpus_b200.engine import CLUSTER_DTYPE, JOB_DTYPE

HIGH_WATER = (S.S_MAX_XFER, S.S_MAX_RUN, S.S_MAX_Q)
CASES = ["cfg3_4x64_sinusoid_120s", "sweep_joint_nf", "sweep_eco_route", "ragged_3dc_12_5_40", "cap_greedy_4x64",
         "cfg5_8x256_sinusoid_60s", "no_inf_priority_perf_first", "cfg2_1x64_poisson_600s"]


@pytest.fixture
def quantum(oracle, hostemu):
    def set_q(q):
        oracle.set_test_time_quantum(q)
        hostemu.set_test_time_quantum(q)
    yield set_q
    set_q(0.0)


@pytest.mark.parametrize("name", CASES)
@pytest.mark.parametrize("q", [2.0 ** -5, 0.25, 1.0])
def test_same_instant_events_pop_in_push_order(oracle, hostemu, quantum, name, q):
    sc = dict(SC.BY_NAME[name])
    sc["duration"] = min(sc["duration"], 60.0)
    blob = SC.to_spec(sc, caps={"cap_xfer": 4096}).to_bytes()   # coarse clocks pile transfers up: give the seq ring room
    quantum(q)
    want, total = oracle.run_batch(blob, 3, 900, 0)
    got = hostemu.run_batch(blob, 3, 900, rec_replica=1, trace_cap=6000, job_dtype=JOB_DTYPE, jobs_cap=40000,
                            cluster_dtype=CLUSTER_DTYPE, cluster_cap=4000)
    assert np.all(got["summary"][:, S.S_STATUS] == 0)
    a, b = got["summary"].copy(), want.copy()
    a[:, HIGH_WATER] = b[:, HIGH_WATER] = 0
    assert got["events"] == total and np.array_equal(a, b), np.argwhere(a != b)[:8]
    sim = oracle.OracleSim(blob, 901, trace_cap=6000, joblog_cap=40000, clog_cap=4000)
    sim.advance(0)
    wt, wj, wc = sim.trace(), sim.job_log(), sim.cluster_log()
    assert len(got["trace"]) == len(wt)
    ties = int(np.count_nonzero(np.diff(wt["t"]) == 0.0))
    assert ties > 50, "the hook is supposed to make ties common"
    for f in ("t", "seq", "kind"):
        assert np.array_equal(got["trace"][f], wt[f]), f
    for f in JOB_DTYPE.names:
        assert np.array_equal(got["jobs"][f], wj[f]), f
    for f in CLUSTER_DTYPE.names:
        assert np.array_equal(got["cluster"][f], wc[f]), f
    sim.close()


def test_chunked_resume_with_ties(oracle, hostemu, quantum):
    sc = dict(SC.CFG3, duration=30.0)
    blob = SC.to_spec(sc, caps={"cap_xfer": 4096}).to_bytes()
    quantum(0.125)
    whole = hostemu.run_batch(blob, 2, 5)
    parts = hostemu.run_batch(blob, 2, 5, chunk_events=7)
    assert np.array_equal(whole["summary"], parts["summary"]) and whole["events"] == parts["events"]


@pytest.mark.parametrize("name", ["cfg3_4x64_sinusoid_120s", "cfg5_8x256_sinusoid_60s", "ragged_3dc_12_5_40", "sweep_eco_route",
                                  "slow_wan_1g_4x64_sin10_60s"])
@pytest.mark.parametrize("q", [0.0, 0.25])
def test_merge_fallback_paths(oracle, hostemu, quantum, name, q):
    """The list merge keeps a sliding window of arrivals in shared memory and reads HBM where a scan leaves it.  A host
    build with a ring of ONE chunk sends nearly every scan down that path; results must not change.  The slow WAN
    (5 s transfers, hundreds of arrivals per max_transfer) leaves the ring even at full size."""
    sc = dict(SC.BY_NAME[name])
    sc["duration"] = min(sc["duration"], 40.0)
    blob = SC.to_spec(sc, caps={"cap_xfer": 4096}).to_bytes()
    quantum(q)
    want, total = oracle.run_batch(blob, 2, 31, 0)
    got = hostemu.run_batch(blob, 2, 31, smallring=True)
    a, b = got["summary"].copy(), want.copy()
    a[:, HIGH_WATER] = b[:, HIGH_WATER] = 0
    assert got["events"] == total and np.array_equal(a, b)


def test_time_quantum_hook_only_in_the_test_build():
    """The GPU build with the hook (tests/gpuhooks, -DDCSIM_TEST_HOOKS) exports its setter; the product library does not."""
    import ctypes as C
    import __graft_entry__ as G
    from distributed_cluster_gpus_b200 import _native
    if not os.path.exists(G.HOOK_LIB):
        G.build()
    assert not hasattr(C.CDLL(_native.LIB_PATH), "dcsim_test_set_time_quantum")
    hook = C.CDLL(G.HOOK_LIB)
    assert hasattr(hook, "dcsim_test_set_time_quantum")
    with open(os.path.join(ROOT, "include", "dcsim_b200.h")) as f:
        assert "dcsim_test_set_time_quantum" not in f.read()
