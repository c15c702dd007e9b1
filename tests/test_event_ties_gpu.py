"""Same-instant events and the list merge's long-transfer path, on the device, against the oracle.

Both are pinned on the single-lane host build (test_event_ties.py), but the code that differs between that build and
the GPU's is exactly the code they depend on: the merge's ballot count of finite transfers and its 32-lane chunks over a
shared-memory ring, the pre-pass's warp-flushed stages, the lane-group pop-min with its cached minimum.

  * Zero transfer (WAN latency 0, no bandwidth term, a configuration the reference runs): every arrival ties with the
    xfer_done it pushes at its own instant.
  * Slow WAN (1 Gbps: a training job's 5 GB take 5 s): hundreds of arrivals lie within one max_transfer, so the merge
    leaves its DCSIM_MERGE_RING-entry ring and reads HBM (dcsim_merge_positions<true>, stage 2's out-of-ring reads,
    stage 1's stop test).  Each test checks from the oracle's arrival instants that this really happens.
  * The test-only hook build (-DDCSIM_TEST_HOOKS, tests/gpuhooks) rounds arrival and xfer_done instants up to a
    quantum, as the oracle's hook does: the test_event_ties matrix on the GPU.

Counts and seq are exact; summary floats are held to test_gpu_parity's bar, trace instants to 1e-12."""
import glob
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from conftest import ROOT, has_cuda
from distributed_cluster_gpus_b200 import scenarios as SC, spec as S
from test_gpu_parity import assert_rows_match

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not has_cuda(), reason="needs a CUDA device")]

SEED, REC = 900, 1                  # replica REC (key SEED + REC) is traced and logged
TRACE_CAP, JOBS_CAP, CLUSTER_CAP = 40000, 40000, 4000
MERGE_RING = 128                    # DCSIM_MERGE_RING (dcsim_core.cuh)
CPUS = os.cpu_count() or 1

# build -> (scenario, replicas, rng): the 8-lane build with a ragged last warp (41 replicas), the 32-lane build (8 DCs),
# the <CAP> build (power-cap controller), ECO routing, the MT19937 word source, and the fixtures themselves
BUILDS = {
    "lanes8_ragged41": ("cfg3_4x64_sinusoid_120s", 41, "philox"),
    "lanes32_cfg5": ("cfg5_8x256_sinusoid_60s", 8, "philox"),
    "cap_greedy": ("cap_greedy_4x64", 8, "philox"),
    "eco_route": ("sweep_eco_route", 8, "philox"),
    "mt19937": ("cfg3_4x64_sinusoid_120s", 8, "mt19937"),
}


def _scenario(name, wan):
    sc = dict(SC.BY_NAME[name])
    return dict(sc, wan=dict(wan), duration=min(sc["duration"], 60.0))


def _rng_kind(oracle, rng):
    return oracle.RNG_MT19937 if rng == "mt19937" else oracle.RNG_PHILOX


def tie_counts(trace):
    """Instants at which several events happen, by class: an arrival with an xfer_done, two arrivals (two streams due
    at once: one stream never has two pending), a list event (arrival / xfer_done) with a log tick."""
    t, k = trace["t"], trace["kind"]
    starts = np.flatnonzero(np.r_[True, t[1:] != t[:-1]])
    arr = np.add.reduceat((k <= 1).astype(np.int64), starts) if len(t) else np.zeros(0, np.int64)
    xfer = np.add.reduceat((k == 2).astype(np.int64), starts) if len(t) else arr
    log = np.add.reduceat((k == 4).astype(np.int64), starts) if len(t) else arr
    return {"arrival_xfer": int(np.sum((arr > 0) & (xfer > 0))), "two_arrivals": int(np.sum(arr > 1)),
            "list_log": int(np.sum(((arr + xfer) > 0) & (log > 0)))}


def max_arrivals_per_window(trace, width):
    """The most arrivals of the traced replica within `width` seconds of each other."""
    a = np.sort(trace["t"][trace["kind"] <= 1])
    return int(np.max(np.searchsorted(a, a + width, side="right") - np.arange(len(a)))) if len(a) else 0


def max_transfer(sp):
    x = np.ctypeslib.as_array(sp.transfer_s)[:sp.n_ing, :sp.n_dc]
    return float(x[np.isfinite(x)].max())


def oracle_replica(oracle, blob, rng_kind=0):
    sim = oracle.OracleSim(blob, SEED + REC, rng_kind, trace_cap=TRACE_CAP, joblog_cap=JOBS_CAP, clog_cap=CLUSTER_CAP)
    sim.advance(0)
    out = {"trace": sim.trace(), "jobs": sim.job_log(), "cluster": sim.cluster_log()}
    sim.close()
    assert len(out["trace"]) < TRACE_CAP, "the whole run must fit the trace"
    return out


def assert_logs_match(got, want):
    tr, wt = got["trace"], want["trace"]
    assert len(tr) == len(wt)
    assert np.array_equal(tr["kind"], wt["kind"]) and np.array_equal(tr["seq"], wt["seq"])
    np.testing.assert_allclose(tr["t"], wt["t"], rtol=1e-12, atol=0)
    jobs, wj, cl, wc = got["jobs"], want["jobs"], got["cluster"], want["cluster"]
    assert len(jobs) == len(wj) and len(cl) == len(wc)
    for f in ("jid", "ingress", "jtype", "dc", "n_gpus"):
        assert np.array_equal(jobs[f], wj[f]), f
    for f in ("size", "f_used", "start_s", "finish_s"):
        np.testing.assert_allclose(jobs[f], wj[f], rtol=1e-12)
    for f in ("dc", "busy", "run_total", "run_inf", "q_inf", "q_train"):
        assert np.array_equal(cl[f], wc[f]), f
    for f in ("time_s", "freq", "util_gpu_time", "util_begin_ts", "acc_job_unit", "power_w", "energy_j"):
        np.testing.assert_allclose(cl[f], wc[f], rtol=1e-9)


def run_device(sp, n, rng="philox", chunk=0, logged=True, seed=SEED):
    """Summary, event count and (logged) replica REC's trace and logs; chunk > 0: advance(chunk) until all are done."""
    from distributed_cluster_gpus_b200.engine import BatchedEngine
    with BatchedEngine(sp, n, base_seed=seed) as eng:
        if rng != "philox":
            eng.set_rng(rng)
        if logged:
            eng.set_trace(REC, TRACE_CAP)
            eng.set_logging(REC, JOBS_CAP, CLUSTER_CAP)
        if chunk:
            total, guard = 0, 0
            while not eng.all_done():
                total += eng.advance(chunk)
                guard += 1
                assert guard < 100000
        else:
            total = eng.advance(0)
        out = {"summary": eng.summary(), "events": total}
        if logged:
            out.update(trace=eng.trace(), jobs=eng.job_log(), cluster=eng.cluster_log())
    return out


def check_against_oracle(oracle, sc, n, rng, chunk):
    sp = SC.to_spec(sc)                                  # default capacities: they must hold
    blob = sp.to_bytes()
    kind = _rng_kind(oracle, rng)
    want, want_total = oracle.run_batch(blob, n, SEED, 0, kind, n_threads=CPUS)
    got = run_device(sp, n, rng, chunk)
    assert np.all(got["summary"][:, S.S_STATUS] == 0) and np.all(got["summary"][:, S.S_DONE] == 1)
    assert got["events"] == want_total
    assert_rows_match(got["summary"], want, sc["n_dc"])
    ref = oracle_replica(oracle, blob, kind)
    assert_logs_match(got, ref)
    if chunk == 0:                                       # the lean record layout (no job log) as well
        plain = run_device(sp, n, rng, 0, logged=False)
        assert np.array_equal(plain["summary"], got["summary"]) and plain["events"] == got["events"]
    return sp, ref


@pytest.mark.parametrize("chunk", [0, 13, 997])
@pytest.mark.parametrize("build", list(BUILDS) + ["fixture"])
def test_zero_transfer_matches_oracle(oracle, build, chunk):
    if build == "fixture":
        sc, n, rng = SC.BY_NAME["zero_xfer_4x64_sin10_60s"], 8, "philox"
    else:
        base, n, rng = BUILDS[build]
        sc = _scenario(base, SC.ZERO_WAN)
    sp, ref = check_against_oracle(oracle, sc, n, rng, chunk)
    assert max_transfer(sp) == 0.0
    ties = tie_counts(ref["trace"])
    print(f"zero transfer {build} chunk {chunk}: ties {ties}")
    assert ties["arrival_xfer"] > 100


@pytest.mark.parametrize("chunk", [0, 13, 997])
@pytest.mark.parametrize("build", list(BUILDS) + ["fixture"])
def test_slow_wan_matches_oracle(oracle, build, chunk):
    if build == "fixture":
        sc, n, rng = SC.BY_NAME["slow_wan_1g_4x64_sin10_60s"], 8, "philox"
    else:
        base, n, rng = BUILDS[build]
        sc = _scenario(base, SC.SLOW_WAN)
    sp, ref = check_against_oracle(oracle, sc, n, rng, chunk)
    # the merge's ring holds MERGE_RING arrivals; with more than twice that within one max_transfer (+ margin) a chunk's
    # scans reach behind the ring, stage 1 runs past it, and some of the chunk's own arrivals have left it
    window = max_arrivals_per_window(ref["trace"], max_transfer(sp) + 1e-9)
    print(f"slow WAN {build} chunk {chunk}: max_transfer {max_transfer(sp):.3f} s, {window} arrivals in one window")
    assert window > 2 * MERGE_RING


def test_slow_wan_large_batch_matches_threaded_oracle(oracle):
    sc = SC.BY_NAME["slow_wan_1g_4x64_sin10_60s"]
    sp = SC.to_spec(sc)
    n = 4096
    want, want_total = oracle.run_batch(sp.to_bytes(), n, 4242, 0, n_threads=CPUS)
    got = run_device(sp, n, logged=False, seed=4242)
    assert np.all(got["summary"][:, S.S_STATUS] == 0) and np.all(got["summary"][:, S.S_DONE] == 1)
    assert got["events"] == want_total
    worst = assert_rows_match(got["summary"], want, sc["n_dc"])
    print(f"slow WAN, {n} replicas, {want_total} events, worst float rel err {worst:.2e}")


def test_group_member_on_zero_transfer_lists(oracle):
    """A member (the <CAP> build, cap_greedy) reading a zero-transfer owner's lists equals its standalone batch and
    the oracle."""
    from distributed_cluster_gpus_b200.engine import BatchedEngine, arrivals_compatible
    owner_sp = SC.to_spec(SC.BY_NAME["zero_xfer_4x64_sin10_60s"])
    sc = SC.BY_NAME["zero_xfer_cap_greedy_4x64_60s"]
    sp = SC.to_spec(sc)
    assert arrivals_compatible(owner_sp, sp)
    n = 41
    with BatchedEngine(owner_sp, n, base_seed=SEED) as owner, BatchedEngine.shared(sp, owner) as member:
        owner.advance(0)
        total = member.advance(0)
        got = member.summary()
    alone = run_device(sp, n, logged=False)
    assert total == alone["events"] and np.array_equal(got, alone["summary"])
    want, want_total = oracle.run_batch(sp.to_bytes(), n, SEED, 0, n_threads=CPUS)
    assert total == want_total and np.all(got[:, S.S_STATUS] == 0)
    assert_rows_match(got, want, sc["n_dc"])


# ---- the hook build: every arrival and xfer_done instant rounded up to a multiple of q ---------------------------------
HOOK_CASES = ["cfg3_4x64_sinusoid_120s", "sweep_joint_nf", "sweep_eco_route", "ragged_3dc_12_5_40", "cap_greedy_4x64",
              "cfg5_8x256_sinusoid_60s", "no_inf_priority_perf_first", "cfg2_1x64_poisson_600s"]
HOOK_QUANTA = [2.0 ** -5, 0.25, 1.0]       # each divides log_interval (5 s): list events tie with log ticks
HOOK_REPLICAS = [3, 41]


def _hook_blob(name):
    sc = dict(SC.BY_NAME[name])
    sc["duration"] = min(sc["duration"], 60.0)
    return SC.to_spec(sc, caps={"cap_xfer": 4096}).to_bytes()   # coarse clocks pile transfers up: give the seq ring room


def _hook_job(name, q, n):
    return f"{name}__q{q}__n{n}"


@pytest.fixture(scope="session")
def hook_runs(tmp_path_factory):
    """Runs the whole matrix through the hook build, in a process of its own (tests/gpuhooks/driver.py)."""
    import __graft_entry__ as G
    srcs = glob.glob(os.path.join(G.CSRC, "*.cu*")) + [os.path.join(ROOT, "include", "dcsim_b200.h")]
    if not G._newer(G.HOOK_LIB, srcs):
        G.build()
    out = tmp_path_factory.mktemp("hook_runs")
    jobs = [{"name": _hook_job(name, q, n), "spec_hex": _hook_blob(name).hex(), "n": n, "seed": SEED, "q": q, "rec": REC,
             "trace_cap": TRACE_CAP, "jobs_cap": JOBS_CAP, "cluster_cap": CLUSTER_CAP}
            for name in HOOK_CASES for q in HOOK_QUANTA for n in HOOK_REPLICAS]
    with open(out / "jobs.json", "w") as f:
        json.dump(jobs, f)
    res = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "gpuhooks", "driver.py"), str(out / "jobs.json"), str(out)],
                         env=dict(os.environ, DCSIM_B200_LIB=G.HOOK_LIB), capture_output=True, text=True, timeout=1800)
    assert res.returncode == 0, res.stderr[-3000:]
    return out


@pytest.fixture
def quantum(oracle):
    yield oracle.set_test_time_quantum
    oracle.set_test_time_quantum(0.0)


@pytest.mark.parametrize("n", HOOK_REPLICAS)
@pytest.mark.parametrize("q", HOOK_QUANTA)
@pytest.mark.parametrize("name", HOOK_CASES)
def test_hook_build_same_instant_events(oracle, hook_runs, quantum, name, q, n):
    blob = _hook_blob(name)
    quantum(q)
    want, want_total = oracle.run_batch(blob, n, SEED, 0, n_threads=CPUS)
    ref = oracle_replica(oracle, blob)
    with np.load(hook_runs / (_hook_job(name, q, n) + ".npz")) as z:
        got = {k: z[k] for k in z.files}
    assert np.all(got["summary"][:, S.S_STATUS] == 0)
    assert int(got["events"]) == want_total
    assert_rows_match(got["summary"], want, SC.BY_NAME[name]["n_dc"])
    assert_logs_match(got, ref)
    ties = tie_counts(ref["trace"])
    window = max_arrivals_per_window(ref["trace"], max_transfer(SC.to_spec(SC.BY_NAME[name])) + q)
    print(f"hook {name} q={q} n={n}: ties {ties}, {window} arrivals in one window")
    assert min(ties.values()) >= 1, ties
