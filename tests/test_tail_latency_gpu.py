"""Per-run tail latency on the H100: the selection kernel bit for bit against numpy over the device's own instants (its
slot buffer, and the arrival and xfer_done instants of the same pre-pass from the hook build, tests/gpuhooks) in every
staging mode, in 8- and 32-lane builds, one shot and in chunks; the instants and columns against the oracle and the
reference goldens; the reductions against the numpy mirror; one rank against two; the capacity retry; the error codes;
and the 65 536-replica bench batch."""
import glob
import json
import math
import os
import subprocess
import sys

import numpy as np
import pytest

import hostemu_tail_lib as HT
from conftest import has_cuda
from distributed_cluster_gpus_b200 import ensemble as E, scenarios as SC, spec as S
from test_launch_modes_gpu import SCENARIOS as LM_SCENARIOS, force_mode, spec_for
from test_tail_latency import GOLDEN_FILES, SLA, TAIL_GOLDEN, same

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not has_cuda(), reason="needs a CUDA device")]

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RTOL = 1e-9
SEED = 123
N_MODES = 5
BENCH_N, BENCH_PICK = 65536, list(range(0, 65536, 1024))
SC_MODES = {False: LM_SCENARIOS[False], True: dict(SC.BY_NAME["cfg3_4x64_sinusoid_120s"], duration=40.0)}


def _engine(sp, n, seed=SEED, **kw):
    from distributed_cluster_gpus_b200.engine import BatchedEngine
    return BatchedEngine(sp, n, base_seed=seed, **kw)


def _run(eng, chunk=0):
    eng.advance(chunk)
    guard = 0
    while chunk and not eng.all_done():
        eng.advance(chunk)
        guard += 1
        assert guard < 100000


@pytest.fixture(scope="module")
def prepass(tmp_path_factory):
    """The arrival and xfer_done instants and arrival metadata the device's pre-pass and merge leave for the batches
    below, through the hook build at quantum 0 (the product library's code; it has no way to hand them out)."""
    import __graft_entry__ as G
    srcs = glob.glob(os.path.join(G.CSRC, "*.cu*")) + [os.path.join(ROOT, "include", "dcsim_b200.h")]
    if not G._newer(G.HOOK_LIB, srcs):
        G.build()
    jobs = [{"kind": "prepass", "name": f"modes_{big}", "spec_hex": SC.to_spec(SC_MODES[big]).to_bytes().hex(),
             "n": N_MODES, "seed": SEED, "q": 0.0} for big in (False, True)]
    jobs.append({"kind": "prepass", "name": "bench", "spec_hex": SC.to_spec(SC.CFG3).to_bytes().hex(), "n": BENCH_N,
                 "seed": SEED, "q": 0.0, "replicas": BENCH_PICK})
    out = tmp_path_factory.mktemp("tail_prepass")
    with open(out / "jobs.json", "w") as f:
        json.dump(jobs, f)
    res = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "gpuhooks", "driver.py"), str(out / "jobs.json"), str(out)],
                         env=dict(os.environ, DCSIM_B200_LIB=G.HOOK_LIB), capture_output=True, text=True, timeout=1800)
    assert res.returncode == 0, res.stderr[-3000:]

    def load(name):
        with np.load(out / (name + ".npz")) as z:
            return {k: z[k] for k in z.files}
    return load


def check_replica(sp, rows, slots, pre, i, r, summ, seed, rng_kind=0):
    """Replica r (row i of the pre-pass arrays): the columns are numpy's order statistics over the device's own
    instants bit for bit; the instants and columns are the oracle's within RTOL, counts exact."""
    created = int(summ[r, S.S_JOBS_CREATED])
    dev = HT.jobs_from_slots(slots[r], pre["arr_t"][i], pre["arr_tx"][i], pre["arr_meta"][i], created)
    want = E.tail_rows_from_jobs([dev], [0], sp.n_dc, SLA)[:, 0]
    assert same(rows[:, r], want), (r, np.argwhere(~((rows[:, r] == want) | np.isnan(want)))[:5].ravel())
    ora = HT.oracle_created(sp.to_bytes(), seed + r, rng_kind)
    assert len(ora) == created
    assert np.array_equal(dev["jtype"], ora["jtype"]) and np.array_equal(dev["dc"], ora["dc"])
    fin = ~np.isnan(ora["finish"])
    assert np.array_equal(~np.isnan(dev["finish"]), fin)
    for f in ("arrival", "xfer_done", "start", "finish"):
        a, b = dev[f][fin], ora[f][fin]
        assert np.all(np.abs(a - b) <= RTOL * np.maximum(np.abs(b), 1e-300)), (r, f)
    close_to_oracle(rows[:, r], E.tail_rows_from_jobs([ora], [0], sp.n_dc, SLA)[:, 0], sp.n_dc, r)


def close_to_oracle(got, want, n_dc, what):
    """Counts and SLA bits exact, NaN where the oracle's are, values within RTOL relative (absolute below 1 s: a wait
    is a difference of two instants)."""
    integral = E._tail_integral(n_dc)
    assert np.array_equal(np.isnan(got), np.isnan(want)), what
    ok = ~np.isnan(want)
    assert np.array_equal(got[integral & ok], want[integral & ok]), what
    real = ~integral & ok
    assert np.all(np.abs(got[real] - want[real]) <= RTOL * np.maximum(np.abs(want[real]), 1.0)), what


@pytest.mark.parametrize("chunk", [0, 61])
@pytest.mark.parametrize("lanes", [8, 32])
@pytest.mark.parametrize("mode", ["staged", "head", "inplace"])
@pytest.mark.parametrize("big", [False, True], ids=["ragged", "cfg3"])
def test_device_columns(prepass, monkeypatch, big, mode, lanes, chunk):
    """The selection kernel, after the event loop in each staging mode and lane width, one shot and in chunks of 61
    events: bit for bit numpy's inverted_cdf over the device's own instants; within RTOL of the oracle."""
    force_mode(monkeypatch, lanes, mode)
    sc = SC_MODES[big]
    sp = spec_for(sc, mode)
    with _engine(sp, N_MODES) as eng:
        eng.enable_tail_latency(SLA)
        _run(eng, chunk)
        info = eng.launch_info()
        summ = eng.summary()
        rows = eng.tail_latency_rows()
        slots = eng.tail_latency_jobs()
    assert info["lanes_per_replica"] == lanes
    assert np.all(summ[:, S.S_STATUS] == 0)
    pre = prepass(f"modes_{big}")
    for r in range(N_MODES):
        check_replica(SC.to_spec(sc), rows, slots, pre, r, r, summ, SEED)


@pytest.mark.parametrize("fname", GOLDEN_FILES)
def test_reference_golden(fname):
    """The columns the unmodified reference gives (tests/golden/make_golden_tail.py), Philox and MT19937 runs: counts
    exact, values within RTOL."""
    with open(os.path.join(TAIL_GOLDEN, fname)) as f:
        doc = json.load(f)
    sp = SC.to_spec(doc["scenario"])
    for case in doc["cases"]:
        with _engine(sp, 1, case["seed"]) as eng:
            if case["rng"] == "mt":
                eng.set_rng("mt19937")
            eng.enable_tail_latency(doc["meta"]["sla_s"])
            eng.advance(0)
            got = eng.tail_latency_rows()[:, 0]
            summ = eng.summary()
        assert summ[0, S.S_JOBS_CREATED] == case["jobs_created"] and summ[0, S.S_JOBS_FINISHED] == case["jobs_finished"]
        want = np.array([np.nan if v is None else float.fromhex(v) for v in case["cols"]])
        close_to_oracle(got, want, sp.n_dc, (fname, case["seed"], case["rng"]))


def check_reductions(res, mirror):
    assert np.array_equal(res.n, mirror.n)
    assert np.array_equal(res.min, mirror.min, equal_nan=True) and np.array_equal(res.max, mirror.max, equal_nan=True)
    assert np.array_equal(res.quantiles, mirror.quantiles, equal_nan=True)
    assert np.allclose(res.mean, mirror.mean, rtol=1e-12, atol=0, equal_nan=True)
    assert np.allclose(res.std, mirror.std, rtol=1e-9, atol=1e-12, equal_nan=True)


def test_reductions_match_the_mirror():
    sp = SC.to_spec(dict(SC.CFG3, duration=30.0))
    with _engine(sp, 301) as eng:
        eng.enable_tail_latency(SLA)
        eng.advance(0)
        rows = eng.tail_latency_rows()
        summ = eng.summary()
        res = E.tail_latency(eng)
    assert res.sla_s == SLA
    check_reductions(res, E.tail_latency_from_rows(rows, summ[:, S.S_STATUS], SLA))
    assert res.n[res.column(None, 0, "jobs")] == 301


def test_bench_batch(prepass):
    """All 65 536 replicas of the bench batch: summaries bit-identical with the recorder on and off, every 1024th replica's columns against numpy over its own instants and against the oracle, and the
    reductions against the mirror."""
    sp = SC.to_spec(SC.CFG3)
    with _engine(sp, BENCH_N) as eng:
        eng.advance(0)
        off = eng.summary().copy()
    with _engine(sp, BENCH_N) as eng:
        eng.enable_tail_latency(SLA)
        eng.advance(0)
        on = eng.summary()
        rows = eng.tail_latency_rows()
        slots = np.stack([eng.tail_latency_jobs(r, 1)[0] for r in BENCH_PICK])
        res = E.tail_latency(eng)
    assert same(on, off), "summaries differ with the recorder on"
    assert np.all(on[:, S.S_STATUS] == 0)
    pre = prepass("bench")
    assert list(pre["replicas"]) == BENCH_PICK
    for i, r in enumerate(BENCH_PICK):
        check_replica(sp, rows[:, BENCH_PICK], slots, pre, i, i, on[BENCH_PICK], SEED + r - i)
    check_reductions(res, E.tail_latency_from_rows(rows, on[:, S.S_STATUS], SLA))


def test_capacity_retry_resizes_the_slots():
    """run_to_completion(tail_latency=True) from too small an arrival buffer: the retry re-enables the recorder with a
    slot buffer of the new cap_arrivals, and the columns equal a run that needed no retry."""
    from distributed_cluster_gpus_b200 import engine as EG
    sc = dict(SC.CFG3, duration=20.0)
    EG.free_cached_engine()
    tiny = {"cap_arrivals": 64}
    eng, _ = EG.run_to_completion(lambda caps: SC.to_spec(sc, caps=dict(caps) or tiny), 9, SEED, max_retries=10,
                                  tail_latency=True, tail_sla_s=SLA)
    try:
        assert eng.tail_latency_enabled and eng.spec.cap_arrivals > 64
        got = eng.tail_latency_rows()
        assert eng.tail_latency_jobs().shape[1] == eng.spec.cap_arrivals
    finally:
        eng.close()
    with _engine(SC.to_spec(sc), 9) as ref:
        ref.enable_tail_latency(SLA)
        ref.advance(0)
        want = ref.tail_latency_rows()
    assert same(got, want)


def test_error_codes_and_reset():
    """-1 for a NaN or negative SLA; -4 after the first advance, on a member and for a read while replicas still run;
    -3 with the byte count when the buffers do not fit; after reset the same keys give a fresh engine's columns."""
    import torch
    from distributed_cluster_gpus_b200 import _native as N
    from distributed_cluster_gpus_b200.engine import BatchedEngine
    sp = SC.to_spec(dict(SC.CFG3, duration=20.0))
    with _engine(sp, 16, 7) as eng:
        for bad in (float("nan"), -1.0):
            with pytest.raises(N.DcsimError) as ei:
                eng.enable_tail_latency(bad)
            assert ei.value.code == N.E_INVALID
        with pytest.raises(N.DcsimError) as ei:
            eng.tail_latency_rows()
        assert ei.value.code == N.E_STATE
        eng.enable_tail_latency(SLA)
        eng.advance(50)
        assert not eng.all_done()
        for read in (eng.tail_latency_rows, lambda: E.tail_latency(eng)):
            with pytest.raises(N.DcsimError) as ei:
                read()
            assert ei.value.code == N.E_STATE
        with pytest.raises(N.DcsimError) as ei:
            eng.enable_tail_latency(SLA)
        assert ei.value.code == N.E_STATE
        _run(eng, 100000)
        first = eng.tail_latency_rows()
        with BatchedEngine.shared(sp, eng) as member:
            with pytest.raises(N.DcsimError) as ei:
                member.enable_tail_latency(SLA)
            assert ei.value.code == N.E_STATE
        eng.reset(7)
        eng.enable_tail_latency(SLA)                   # a reset batch is fresh again
        eng.advance(0)
        again = eng.tail_latency_rows()
    with _engine(sp, 16, 7) as fresh:
        fresh.enable_tail_latency(SLA)
        fresh.advance(0)
        assert same(fresh.tail_latency_rows(), first) and same(again, first)
    # -3: the slot buffer of a batch does not fit next to what is held on the device
    big = SC.to_spec(dict(SC.CFG3, duration=20.0), caps={"cap_arrivals": 1 << 16})
    n = 4096
    need = n * (1 << 16) * 16 + S.tail_cols(big.n_dc) * n * 8
    with _engine(big, n) as eng:
        torch.cuda.synchronize()
        free, _ = torch.cuda.mem_get_info()
        hold = torch.empty(max(free - need // 2, 0), dtype=torch.uint8, device="cuda")
        try:
            with pytest.raises(N.DcsimError) as ei:
                eng.enable_tail_latency(SLA)
            assert ei.value.code == N.E_NOMEM and str(need) in str(ei.value)
        finally:
            del hold
            torch.cuda.empty_cache()
        eng.enable_tail_latency(SLA)                   # the handle stays usable
        assert eng.tail_latency_enabled


def _read_csv(path):
    import csv
    with open(path) as f:
        rd = csv.reader(f)
        return next(rd), [r for r in rd]


def test_cli_one_and_two_ranks(tmp_path):
    """run_sim_paper --tail-latency-csv / --summary-json on one rank and on two (gloo when the box has one GPU): n,
    min, max and the quantiles equal, the means to the last bits; --sla_p99_ms moves the *_sla_met rows."""
    import torch
    from test_gpu_parity import _run_cli
    common = ["--duration", "20", "--inf-mode", "sinusoid", "--inf-rate", "10", "--inf-period", "3600", "--trn-rate", "1",
              "--n-dc", "4", "--gpus-per-dc", "16", "--replicas", "301", "--seed", "77", "--progress", ""]
    one = _run_cli(common + ["--log-path", str(tmp_path / "one" / "x"), "--tail-latency-csv", str(tmp_path / "one.csv"),
                             "--summary-json", str(tmp_path / "one.json")])
    assert one.returncode == 0, one.stderr[-2000:]
    extra = {} if torch.cuda.device_count() >= 2 else {"DCSIM_DIST_BACKEND": "gloo"}
    two = _run_cli(common + ["--gpus", "2", "--log-path", str(tmp_path / "two" / "x"), "--tail-latency-csv",
                             str(tmp_path / "two.csv"), "--summary-json", str(tmp_path / "two.json")], extra)
    assert two.returncode == 0, two.stderr[-3000:]
    ha, a = _read_csv(tmp_path / "one.csv")
    hb, b = _read_csv(tmp_path / "two.csv")
    assert ha == hb == E.TAIL_CSV_HEADER
    assert len(a) == len(b) == S.tail_cols(4)
    for ra, rb in zip(a, b):
        assert ra[:4] == rb[:4], (ra, rb)
        for i, (x, y) in enumerate(zip(ra[4:], rb[4:])):
            x, y = float(x), float(y)
            if i in (0, 1):                            # mean, std: summation order
                assert x == y or abs(x - y) <= 1e-12 * max(abs(x), abs(y)) or (math.isnan(x) and math.isnan(y)), (ra, rb)
            else:
                assert x == y or (math.isnan(x) and math.isnan(y)), (ra, rb)
    assert [r[3] for r in a if r[2] == "jobs" and r[1] == ""] == ["301", "301"]
    ja, jb = (json.load(open(tmp_path / f)) for f in ("one.json", "two.json"))
    assert ja["tail_latency"]["inference"]["latency"]["sla_attainment"] == jb["tail_latency"]["inference"]["latency"]["sla_attainment"]
    strict = _run_cli(common + ["--log-path", str(tmp_path / "s" / "x"), "--tail-latency-csv", str(tmp_path / "s.csv"),
                                "--sla_p99_ms", "0.001", "--summary-json", str(tmp_path / "s.json")])
    assert strict.returncode == 0, strict.stderr[-2000:]
    _, s = _read_csv(tmp_path / "s.csv")
    met = {(r[0], r[2]): r for r in a if r[2].endswith("_sla_met")}
    met_strict = {(r[0], r[2]): r for r in s if r[2].endswith("_sla_met")}
    assert float(met[("inference", "latency_sla_met")][4]) > float(met_strict[("inference", "latency_sla_met")][4]) == 0.0
    plain = _run_cli(common + ["--log-path", str(tmp_path / "p" / "x"), "--summary-json", str(tmp_path / "p.json")])
    assert plain.returncode == 0 and "tail_latency" not in json.load(open(tmp_path / "p.json"))
