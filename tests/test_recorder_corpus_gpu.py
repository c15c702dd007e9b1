"""Every batch recorder at once on the H100, on the random corpus and the edge scenarios of test_recorder_corpus.py:
5 or 7 replicas per case (ghost lane groups in the last warp), one shot or in chunks of 61 events, each case on a forced
lane width and staging mode, round-robin (test_launch_modes_gpu.force_mode), with the kernel that ran read back from
launch_info().  Every recorder against the host build of the same batch — which the CPU file holds bit for bit to the
oracle on the same corpus, and which is held to the oracle here too — counts and discrete decisions exact, floats within
1e-9 relative (the rules of the per-recorder GPU tests); each recorder alone bit for bit the all-on run; the summaries
bit for bit the recorder-off kernel's; every statistic's device passes against the numpy mirror over the fetched rows."""
import numpy as np
import pytest

import test_recorder_corpus as RC
from conftest import has_cuda
from distributed_cluster_gpus_b200 import ensemble as EN, scenarios as SC, spec as S
from test_cluster_ensemble_gpu import FLT, INT
from test_gpu_parity import assert_rows_match
from test_launch_modes_gpu import INPLACE_CAP_XFER, MODES, SCENARIOS, force_mode
from test_occupancy_gpu import assert_close as occ_close
from test_power_profile_gpu import assert_close as pp_close
from test_tail_latency_gpu import close_to_oracle as tail_close

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not has_cuda(), reason="needs a CUDA device")]

RTOL = 1e-9
N_GPU = 90                    # the first 90 cases of the CPU corpus: test_random_scenarios_match_oracle's
LANES = (8, 16, 32)
MODE_NAMES = ("staged", "head", "inplace")
RECORDERS = ("lat", "ens", "jens", "jwait", "jres", "pp", "occ", "tail")
_RAN = {}                     # (lanes, staging mode, CAP) -> runs, what launch_info() reported
_ALL_ON = {}                  # case name -> its all-on outputs, for the alone-versus-together test


def is_cap(sp):
    return sp.algo == S.ALGO_IDS["cap_greedy"] and sp.power_cap > 0


def plan():
    """[(name, scenario, Spec, n, chunk, lanes, mode)]: the corpus, the edges, and a targeted cap_greedy case for every
    <CAP> kernel the corpus leaves with fewer than two planned runs.  CAP and non-CAP cases take the lane widths and
    staging modes round-robin on counters of their own."""
    out, turn, planned = [], {False: 0, True: 0}, {}
    cases = [(f"corpus{i}", sc, SC.to_spec(sc), seed) for i, (sc, seed) in enumerate(RC.corpus(N_GPU))]
    cases += [(name, *RC.edge_spec(name), 900) for name in RC.EDGES]
    for i, (name, sc, sp, seed) in enumerate(cases):
        cap = is_cap(sp)
        k = turn[cap]
        turn[cap] += 1
        lanes, mode = LANES[k % 3], MODE_NAMES[(k // 3) % 3]
        planned[(lanes, mode, cap)] = planned.get((lanes, mode, cap), 0) + 1
        out.append((name, sc, sp, seed, 5 if i % 2 == 0 else 7, 0 if (i // 2) % 2 == 0 else 61, lanes, mode))
    sc = SCENARIOS[True]
    for lanes in LANES:
        for mode in MODE_NAMES:
            for j in range(max(0, 2 - planned.get((lanes, mode, True), 0))):
                out.append((f"cap_{lanes}_{mode}_{j}", sc, SC.to_spec(sc), 31 + j, 5 + 2 * j, 61 * j, lanes, mode))
    return out


PLAN = plan()


def _engine(sp, n, seed):
    from distributed_cluster_gpus_b200.engine import BatchedEngine
    return BatchedEngine(sp, n, base_seed=seed)


def run_device(sc, sp, n, seed, chunk, recorders=RECORDERS, reductions=False):
    """The kernel with `recorders` on -> (outputs in the host build's layout, launch_info, reductions or None)."""
    thr = RC.pp_threshold(sc, sp.to_bytes())
    with _engine(sp, n, seed) as eng:
        on = set(recorders)
        if "lat" in on:
            eng.enable_latency_histogram()
        if "ens" in on:
            eng.enable_cluster_ensemble()
        if on & {"jens", "jwait", "jres"}:
            eng.enable_job_ensemble(sp.log_interval)
        if "jwait" in on:
            eng.enable_job_waits()
        if "jres" in on:
            eng.enable_job_resources()
        if "pp" in on:
            eng.enable_power_profile(thr)
        if "occ" in on:
            eng.enable_occupancy()
        if "tail" in on:
            eng.enable_tail_latency(RC.SLA)
        total = eng.advance(chunk)
        guard = 0
        while chunk and not eng.all_done():
            total += eng.advance(chunk)
            guard += 1
            assert guard < 1000000
        out = {"summary": eng.summary().copy(), "events": total}
        if "lat" in on:
            out["lat_batch"] = eng.latency_histogram()
        if "ens" in on:
            out["ens"] = eng.cluster_ensemble_rows()
        if on & {"jens", "jwait", "jres"}:
            rows, hist = eng.job_ensemble_rows()
            out["jens"], out["jens_hist"] = rows, np.moveaxis(hist, -1, 0)
        if "jwait" in on:
            rows, hist = eng.job_waits_rows()
            out["jwait"], out["jwait_hist"] = rows, np.moveaxis(hist, -1, 0)
        if "jres" in on:
            rows, mix, off, hist = eng.job_resources_rows()
            n_dc, G = mix.shape[0], mix.shape[2]
            out["jres"], out["jres_hist"] = rows, hist
            out["jres_mix"] = np.concatenate([mix.reshape(n_dc, 2, G * S.MAX_FREQ, n), off[:, :, None]], axis=2)
        if "pp" in on:
            out["pp"] = eng.power_profile_rows()
        if "occ" in on:
            out["occ"] = eng.occupancy_rows()
            out["occ_widths"] = eng.occupancy_bin_widths()
        if "tail" in on:
            out["tail_cols"] = eng.tail_latency_rows()
        info = eng.launch_info()
        red = reductions_of(eng, sp, out, thr) if reductions else None
    return out, info, red


def _rel(got, want):
    return np.where(got == want, 0.0, np.abs(got - want) / np.maximum(np.abs(want), 1e-300))


def assert_close_rows(got, want, exact_fields, what):
    """[rows, fields, ...] windowed cells: the count fields exact, the sums within RTOL."""
    assert got.shape == want.shape, (what, got.shape, want.shape)
    for f in range(got.shape[1]):
        g, w = got[:, f], want[:, f]
        if f in exact_fields:
            assert np.array_equal(g, w), (what, f, np.argwhere(g != w)[:5])
        else:
            assert float(_rel(g, w).max(initial=0.0)) <= RTOL, (what, f, float(_rel(g, w).max()))


def assert_close_outputs(dev, host, sp, what):
    """The device's outputs against the host build's: the tolerance rules of the per-recorder GPU tests."""
    n_dc = sp.n_dc
    assert_rows_match(dev["summary"], host["summary"], n_dc)
    if "lat_batch" in dev:                                 # the batch histogram sums every replica (dcsim_b200.h)
        assert np.array_equal(dev["lat_batch"], host["lat_hist"].sum(axis=0)), what
    if "ens" in dev and "ens" not in host:                 # a spec without a log tick: the host build records nothing
        assert dev["ens"].shape[0] == 0 and np.all(host["summary"][:, S.S_EV_LOG] == 0), what
    elif "ens" in dev:
        g, w = dev["ens"], host["ens"][:dev["ens"].shape[0]]
        assert g.shape[0] == int(host["summary"][:, S.S_EV_LOG].max()), what
        assert np.array_equal(np.isnan(g), np.isnan(w)), what
        assert np.array_equal(g[:, INT], w[:, INT], equal_nan=True), what
        gf, wf = np.nan_to_num(g[:, FLT]), np.nan_to_num(w[:, FLT])
        assert float(_rel(gf, wf).max(initial=0.0)) <= RTOL, (what, "ens")
    if "jens" in dev:
        assert_close_rows(dev["jens"], host["jens"], (0,), (what, "jens"))
        assert np.array_equal(dev["jens_hist"], host["jens_hist"]), what
    if "jwait" in dev:
        assert_close_rows(dev["jwait"], host["jwait"], (0,), (what, "jwait"))
        assert np.array_equal(dev["jwait_hist"], host["jwait_hist"]), what
    if "jres" in dev:
        assert_close_rows(dev["jres"], host["jres"], (0,), (what, "jres"))
        assert np.array_equal(dev["jres_mix"], host["jres_mix"]) and np.array_equal(dev["jres_hist"], host["jres_hist"]), what
    if "pp" in dev:
        pp_close(dev["pp"], host["pp"], str(what))
    if "occ" in dev:
        occ_close(dev["occ"], host["occ"], n_dc, str(what))
        assert list(dev["occ_widths"]) == [(sp.dc[d].total_gpus + S.OCC_BINS) // S.OCC_BINS for d in range(n_dc)]
    if "tail_cols" in dev:
        for r in range(dev["tail_cols"].shape[1]):
            tail_close(dev["tail_cols"][:, r], host["tail_cols"][:, r], n_dc, (what, r))


def reductions_of(eng, sp, out, thr):
    """Each statistic's device passes, called twice, and the numpy mirror over the fetched rows and status words."""
    st = out["summary"][:, S.S_STATUS]
    ens_rows = out["ens"]
    nlog = (~np.isnan(ens_rows[:, 0, 0, :])).sum(axis=0)
    jobs = out["jens"][:, 0]
    G = (out["jres_mix"].shape[2] - 1) // S.MAX_FREQ
    n = len(st)
    mix = out["jres_mix"]
    pairs = {
        "cluster": (lambda: EN.cluster_ensemble(eng), EN.cluster_ensemble_from_rows(ens_rows, nlog, sp.log_interval)),
        "job": (lambda: EN.job_ensemble(eng),
                EN.job_ensemble_from_rows(out["jens"], np.moveaxis(out["jens_hist"], 0, -1), st, sp.log_interval, sp.end_time)),
        "waits": (lambda: EN.job_waits(eng),
                  EN.job_waits_from_rows(out["jwait"], np.moveaxis(out["jwait_hist"], 0, -1), jobs, st, sp.log_interval,
                                         sp.end_time)),
        "resources": (lambda: EN.job_resources(eng),
                      EN.job_resources_from_rows(out["jres"], mix[:, :, :-1].reshape(sp.n_dc, 2, G, S.MAX_FREQ, n),
                                                 mix[:, :, -1], out["jres_hist"], jobs, st, EN._res_levels(sp),
                                                 sp.log_interval, sp.end_time)),
        "power": (lambda: EN.power_profile(eng, summary=out["summary"]),
                  EN.power_profile_from_rows(out["pp"], out["summary"], eng.power_profile_range(), thr)),
        "occupancy": (lambda: EN.occupancy(eng), EN.occupancy_from_rows(out["occ"], out["summary"], out["occ_widths"])),
        "tail": (lambda: EN.tail_latency(eng), EN.tail_latency_from_rows(out["tail_cols"], st, RC.SLA)),
    }
    return {k: (fn(), fn(), mirror) for k, (fn, mirror) in pairs.items()}


STAT_FIELDS = ("n", "min", "max", "quantiles", "mean", "std")


def check_reductions(red, what):
    """n, min, max and quantiles exact; mean within 1e-12, std within 1e-9 (over the columns some replica counts in); a
    second call bit for bit the first."""
    for k, (a, b, m) in red.items():
        for f in STAT_FIELDS:
            x, y = np.asarray(getattr(a, f), dtype=np.float64), np.asarray(getattr(b, f), dtype=np.float64)
            assert x.shape == y.shape and np.array_equal(RC.bits(x), RC.bits(y)), (what, k, f, "second call")
        assert np.array_equal(a.n, m.n), (what, k)
        ok = np.asarray(a.n) > 0
        for f in ("min", "max"):
            assert np.array_equal(getattr(a, f)[ok], getattr(m, f)[ok], equal_nan=True), (what, k, f)
        assert np.array_equal(a.quantiles[:, ok], m.quantiles[:, ok], equal_nan=True), (what, k, "quantiles")
        assert np.allclose(a.mean[ok], m.mean[ok], rtol=1e-12, atol=0, equal_nan=True), (what, k, "mean")
        # a column of (nearly) equal values has a spread that is rounding residue of the mean, about one ulp of it on
        # either side: its floor scales with |mean|, not a fixed 1e-12
        sa, sm, mu = a.std[ok], m.std[ok], np.abs(m.mean[ok])
        err = np.abs(sa - sm) - (1e-9 * np.abs(sm) + 1e-12 * np.maximum(mu, 1.0))
        assert np.all((err <= 0) | (np.isnan(sa) & np.isnan(sm))), (what, k, "std", sa[np.argmax(err)], sm[np.argmax(err)])


def _gpu_spec(sp, mode):
    """The case's spec with test_launch_modes_gpu's seq ring when the launch is to run in place: a copy with cap_xfer
    INPLACE_CAP_XFER (capacities size buffers, they decide nothing a replica computes)."""
    if mode != "inplace":
        return sp
    big = S.Spec.from_buffer_copy(sp.to_bytes())
    big.cap_xfer = max(big.cap_xfer, INPLACE_CAP_XFER)
    return big


@pytest.mark.parametrize("part", range(6))
def test_corpus_matches_host_build_and_oracle(oracle, monkeypatch, part):
    """Every case of the plan: the kernel that ran recorded; every recorder within the rules of the host build of the
    same batch, which equals the oracle bit for bit; the device passes of every statistic against the mirror."""
    for i, (name, sc, sp, seed, n, chunk, lanes, mode) in enumerate(PLAN):
        if i % 6 != part:
            continue
        force_mode(monkeypatch, lanes, mode)
        host = RC.run_all(sc, sp, n, seed)
        assert np.all(host["summary"][:, S.S_STATUS] == 0), name
        RC.check_oracle(oracle, sc, sp, host, seed, n)
        dev, info, red = run_device(sc, _gpu_spec(sp, mode), n, seed, chunk, reductions=True)
        what = (name, n, chunk, lanes, mode)
        assert dev["events"] == host["events"], what
        assert np.all(dev["summary"][:, S.S_DONE] == 1), what
        got = (info["lanes_per_replica"], info["staging_mode"], is_cap(sp))
        _RAN.setdefault(got, []).append((name, lanes, mode))
        assert_close_outputs(dev, host, sp, what)
        check_reductions(red, what)
        if name in ALONE_CASES:
            _ALL_ON[name] = dev


def test_every_profile_kernel_ran_twice():
    """The table of the 18 profile kernels (lanes x staging mode x CAP) the corpus reached, and how often; a forced
    combination the library refused shows under the kernel that ran instead."""
    inv = {v: k for k, v in MODES.items()}
    print("\nlanes  staging  cap    runs  (asked for when different)")
    for (lanes, mode, cap), runs in sorted(_RAN.items()):
        other = sorted({(l, m) for _, l, m in runs if (l, m) != (lanes, inv[mode])})
        print(f"{lanes:5d}  {inv[mode]:8s} {str(cap):6s} {len(runs):4d}  {other if other else ''}")
    missing = [(l, m, c) for l in LANES for m in MODES.values() for c in (False, True) if len(_RAN.get((l, m, c), ())) < 2]
    assert not missing, missing


# one case per lane width from the corpus, a <CAP> case, and the off-ladder edge
ALONE_CASES = sorted({next(p[0] for p in PLAN if p[6] == lanes and p[0].startswith("corpus") and not is_cap(p[2]))
                      for lanes in LANES} | {next(p[0] for p in PLAN if is_cap(p[2])), "off_ladder_debug"})


@pytest.mark.parametrize("name", ALONE_CASES)
def test_each_recorder_alone_equals_all_on(monkeypatch, name):
    """Each recorder alone (the job recorders with the job ensemble they hang off) gives bit for bit what it gives with
    every recorder on, and the summaries of every run are bit for bit the recorder-off kernel's: -fmad=false and fixed
    summation orders leave nothing for the profile instantiation or the job-log layout to move."""
    _, sc, sp, seed, n, chunk, lanes, mode = next(p for p in PLAN if p[0] == name)
    force_mode(monkeypatch, lanes, mode)
    gsp = _gpu_spec(sp, mode)
    together = _ALL_ON.get(name) or run_device(sc, gsp, n, seed, chunk)[0]
    off, _, _ = run_device(sc, gsp, n, seed, chunk, recorders=())
    assert np.array_equal(RC.bits(off["summary"]), RC.bits(together["summary"])), name
    for rec, keys in (("lat", ("lat_batch",)), ("ens", ("ens",)), ("jens", ("jens", "jens_hist")),
                      ("jwait", ("jwait", "jwait_hist")), ("jres", ("jres", "jres_mix", "jres_hist")), ("pp", ("pp",)),
                      ("occ", ("occ",)), ("tail", ("tail_cols",))):
        alone, _, _ = run_device(sc, gsp, n, seed, chunk, recorders=(rec,))
        assert np.array_equal(RC.bits(alone["summary"]), RC.bits(off["summary"])), (name, rec)
        for k in keys:
            assert np.array_equal(RC.bits(alone[k]), RC.bits(together[k])), (name, rec, k)


def test_zero_tick_run():
    """log_interval > duration: enabling the cluster ensemble succeeds, its rows have 0 ticks and its statistics are
    empty; the other recorders still see every job."""
    sc, sp = RC.edge_spec("no_log_tick")
    dev, _, red = run_device(sc, sp, 5, 900, 0, reductions=True)
    assert dev["ens"].shape == (0, len(EN.FIELDS), sp.n_dc, 5)
    res = red["cluster"][0]
    assert res.n.shape == (0, len(EN.FIELDS), sp.n_dc) and len(res.time_s) == 0
    assert np.all(dev["summary"][:, S.S_JOBS_FINISHED] > 0)


def test_empty_run():
    """No event at all: every recorder empty, the tail's order statistics and SLA bits NaN."""
    sc, sp = RC.edge_spec("empty_run")
    dev, _, red = run_device(sc, sp, 7, 900, 0, reductions=True)
    host = RC.run_all(sc, sp, 7, 900)
    assert_close_outputs(dev, host, sp, "empty_run")
    for k in ("jens", "jwait", "jres", "jres_mix", "jres_hist", "pp", "occ"):
        assert not np.any(dev[k]), k
    counts = [S.tail_col(sp.n_dc, jt, f, d) for jt in range(2) for f in (S.TAIL_JOBS, S.TAIL_UNFINISHED)
              for d in range(-1, sp.n_dc)]
    assert np.all(dev["tail_cols"][counts] == 0)
    assert np.all(np.isnan(np.delete(dev["tail_cols"], counts, axis=0)))
    check_reductions(red, "empty_run")


@pytest.mark.parametrize("lanes", LANES)
def test_status_bit_replicas(monkeypatch, lanes):
    """Replicas that overflow cap_run: exactly those carry the bit, their tail columns are NaN, every other replica's
    columns are the host build's, and every statistic leaves out exactly the failed replicas."""
    force_mode(monkeypatch, lanes, "staged")
    caps, need = RC.status_caps()
    sc, n = RC.STATUS_SC, RC.STATUS_REP
    sp = SC.to_spec(sc, caps=caps)
    dev, info, red = run_device(sc, sp, n, 0, 61, reductions=True)
    host = RC.run_all(sc, sp, n, 0)
    st = dev["summary"][:, S.S_STATUS].astype(np.int64)
    bad = need > caps["cap_run"]
    assert np.array_equal((st & S.ST_RUN_OVERFLOW) != 0, bad) and np.all(st[~bad] == 0)
    assert np.array_equal(st, host["summary"][:, S.S_STATUS].astype(np.int64))
    assert np.all(np.isnan(dev["tail_cols"][:, bad]))
    good = ~bad
    sub = {k: (v[good] if k in ("summary", "jens_hist", "jwait_hist", "lat_hist") else v[..., good])
           for k, v in host.items() if k in RC.OUTPUTS}
    dsub = {k: (v[good] if k in ("summary", "jens_hist", "jwait_hist") else v[..., good]) for k, v in dev.items()
            if k in RC.OUTPUTS and k != "ens"}
    dsub["occ_widths"] = dev["occ_widths"]
    assert_close_outputs(dsub, sub, sp, ("status", lanes))
    # the batch histogram sums every replica, a failed one with what it finished before it stopped: the device's own
    # per-replica histograms (fed by the same finish handler) sum to it, and it holds at least the valid replicas' jobs
    assert np.array_equal(dev["lat_batch"], dev["jens_hist"].sum(axis=(0, 1)))
    assert np.all(dev["lat_batch"] >= host["lat_hist"][good].sum(axis=0))
    check_reductions(red, ("status", lanes))
    ng = int(good.sum())
    assert np.all(red["power"][0].n == ng) and np.all(red["occupancy"][0].n <= ng)
    assert red["tail"][0].n[S.tail_col(sp.n_dc, 0, S.TAIL_JOBS)] == ng
