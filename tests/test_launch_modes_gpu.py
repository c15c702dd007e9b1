"""Every event-loop kernel the library ships, on the H100: dcsim_advance_kernel<CAP, MODE, PP> built for 8, 16 and 32
lanes per replica (dcsim_advance_impl.cuh) — 3 x 3 x 2 x 2 = 36 instantiations.  Each case forces its kernel
(DCSIM_GROUP for the lanes; DCSIM_RECORDS or a seq ring too large for shared memory for the staging mode; a cap_greedy
spec with a binding cap for CAP; the power-profile recorder for PP), asserts that this kernel is the one that ran, and
holds it to the oracle on 5 and 7 replicas (ghost lane groups in the last warp on 8 and 16 lanes), one shot and in
chunks of 61 events.  Every kernel of one scenario must return bit-identical summaries: power sums are sequential in a
fixed order and the build uses -fmad=false, so nothing legitimate depends on lanes or staging."""
import os

import numpy as np
import pytest

import hostemu_lib as H
from conftest import has_cuda
from distributed_cluster_gpus_b200 import scenarios as SC, spec as S
from test_gpu_parity import assert_rows_match
from test_power_profile_gpu import assert_close

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not has_cuda(), reason="needs a CUDA device")]

MODES = {"inplace": 0, "staged": 1, "head": 2}           # DCSIM_MODE_* (launch_info()["staging_mode"])
# cap_xfer 20000 -> a seq ring of 65536 entries, 256 kB per replica: not even one state block's head fits the 227 kB of
# shared memory an H100 CTA can opt in to, whatever the lanes, so the launch runs in place
INPLACE_CAP_XFER = 20000
SCENARIOS = {False: dict(SC.BY_NAME["ragged_3dc_12_5_40"], duration=30.0),
             True: dict(SC.BY_NAME["cap_greedy_4x64"], duration=30.0)}
SEED = 31
HIGH_WATER = (S.S_MAX_RUN, S.S_MAX_Q, S.S_UTIL_BEGIN)
_FIRST = {}      # (cap, n) -> the first kernel's summary: every other kernel must equal it bit for bit
_TABLE = []


def _engine(sp, n, seed):
    from distributed_cluster_gpus_b200.engine import BatchedEngine
    return BatchedEngine(sp, n, base_seed=seed)


def force_mode(monkeypatch, lanes, mode):
    monkeypatch.setenv("DCSIM_GROUP", str(lanes))
    if mode == "inplace":
        monkeypatch.delenv("DCSIM_RECORDS", raising=False)
    else:
        monkeypatch.setenv("DCSIM_RECORDS", "shared" if mode == "staged" else "global")


def spec_for(sc, mode):
    return SC.to_spec(sc, caps={"cap_xfer": INPLACE_CAP_XFER} if mode == "inplace" else None)


_ORACLE = {}


def oracle_rows(oracle, cap, n):
    if (cap, n) not in _ORACLE:
        blob = SC.to_spec(SCENARIOS[cap]).to_bytes()
        _ORACLE[(cap, n)] = oracle.run_batch(blob, n, SEED, 0, n_threads=os.cpu_count() or 1)
    return _ORACLE[(cap, n)]


def pp_threshold(want, sc):
    """A threshold the cluster power crosses: 0.8 x replica 0's mean power."""
    return 0.8 * want[0, S.S_TOTAL_ENERGY_J] / sc["duration"]


@pytest.mark.parametrize("pp", [False, True], ids=["rec_off", "rec_on"])
@pytest.mark.parametrize("cap", [False, True], ids=["nocap", "cap"])
@pytest.mark.parametrize("mode", ["staged", "head", "inplace"])
@pytest.mark.parametrize("lanes", [8, 16, 32])
def test_kernel_matches_oracle(oracle, monkeypatch, lanes, mode, cap, pp):
    force_mode(monkeypatch, lanes, mode)
    sc = SCENARIOS[cap]
    sp = spec_for(sc, mode)
    assert (sp.algo == S.ALGO_IDS["cap_greedy"] and sp.power_cap > 0) == cap
    for n in (5, 7):
        want, want_total = oracle_rows(oracle, cap, n)
        thr = pp_threshold(want, sc)
        for chunk in (0, 61):
            with _engine(sp, n, SEED) as eng:
                if pp:
                    eng.enable_power_profile(thr)
                total = eng.advance(chunk)
                guard = 0
                while chunk and not eng.all_done():
                    total += eng.advance(chunk)
                    guard += 1
                    assert guard < 100000
                got = eng.summary()
                info = eng.launch_info()
                rows = eng.power_profile_rows() if pp else None
            what = (lanes, mode, cap, pp, n, chunk)
            assert info["lanes_per_replica"] == lanes and info["staging_mode"] == MODES[mode], (what, info)
            assert total == want_total, what
            assert np.all(got[:, S.S_STATUS] == 0) and np.all(got[:, S.S_DONE] == 1), what
            assert_rows_match(got, want, sc["n_dc"])
            for col in HIGH_WATER:
                assert np.array_equal(got[:, col], want[:, col]), (what, col, got[:, col], want[:, col])
            first = _FIRST.setdefault((cap, n), (what, got))
            assert np.array_equal(got.view(np.uint64), first[1].view(np.uint64)), \
                (what, "differs from", first[0], np.argwhere(got != first[1])[:6])
            if pp:
                ref = H.run_batch(SC.to_spec(sc).to_bytes(), n, SEED, pp=True, pp_threshold=thr)["pp"]
                assert_close(rows, ref, str(what))
    _TABLE.append((lanes, mode, cap, pp, info["lanes_per_replica"], info["staging_mode"], info["regs_per_thread"],
                   info["smem_bytes_per_cta"]))


@pytest.mark.parametrize("mode", ["staged", "head", "inplace"])
def test_trace_and_logs_match_oracle(oracle, monkeypatch, mode):
    """Full (non-lean) running-job records with the trace and both logs on replica 2 of 5, 8 lanes: a ghost group next
    to replica 4 in the second warp."""
    force_mode(monkeypatch, 8, mode)
    sc = SCENARIOS[False]
    sp = spec_for(sc, mode)
    with _engine(sp, 5, 40) as eng:
        eng.set_trace(2, 20000)
        eng.set_logging(2, 20000, 2000)
        eng.advance(0)
        info = eng.launch_info()
        tr, jobs, cl = eng.trace(), eng.job_log(), eng.cluster_log()
    assert info["lanes_per_replica"] == 8 and info["staging_mode"] == MODES[mode], info
    sim = oracle.OracleSim(SC.to_spec(sc).to_bytes(), 42, trace_cap=20000, joblog_cap=20000, clog_cap=2000)
    sim.advance(0)
    wt, wj, wc = sim.trace(), sim.job_log(), sim.cluster_log()
    assert len(tr) == len(wt) > 100 and np.array_equal(tr["kind"], wt["kind"]) and np.array_equal(tr["seq"], wt["seq"])
    np.testing.assert_allclose(tr["t"], wt["t"], rtol=1e-12, atol=0)
    assert len(jobs) == len(wj) > 20 and len(cl) == len(wc) > 10
    for f in ("jid", "ingress", "jtype", "dc", "n_gpus"):
        assert np.array_equal(jobs[f], wj[f]), f
    for f in ("size", "f_used", "start_s", "finish_s"):
        np.testing.assert_allclose(jobs[f], wj[f], rtol=1e-12)
    for f in ("dc", "busy", "run_total", "run_inf", "q_inf", "q_train"):
        assert np.array_equal(cl[f], wc[f]), f
    for f in ("time_s", "freq", "util_gpu_time", "util_begin_ts", "acc_job_unit", "power_w", "energy_j"):
        np.testing.assert_allclose(cl[f], wc[f], rtol=1e-9)


def test_every_kernel_ran():
    """The table of the 36 kernels the cases above reached (run after them, in file order)."""
    print("\nlanes  mode     cap    recorder | lanes staging regs smem/CTA")
    for lanes, mode, cap, pp, got_lanes, got_mode, regs, smem in _TABLE:
        print(f"{lanes:5d}  {mode:8s} {str(cap):6s} {str(pp):8s} | {got_lanes:5d} {got_mode:7d} {regs:4d} {smem:8d}")
    reached = {(lanes, mode, cap, pp) for lanes, mode, cap, pp, *_ in _TABLE}
    assert len(reached) == 36, f"{len(reached)} of 36 kernels reached"
