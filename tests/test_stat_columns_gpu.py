"""The column counts the library reduces for every batch recorder (dcsim_stat_columns) on the H100, against each
recorder's layout written out in Python: before and after the first advance, with every recorder off and on, on one,
three (ragged) and eight DCs, one and many job windows, max_gpus_per_job 1, 8 and 64, and a cluster ensemble at its
default capacity, at max_ticks=3 and without a log tick."""
import ctypes as C

import pytest

from conftest import has_cuda
from distributed_cluster_gpus_b200 import _native as N, ensemble as EN, scenarios as SC, spec as S
from distributed_cluster_gpus_b200.configs import paper_config as pc

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not has_cuda(), reason="needs a CUDA device")]


def _spec(name, duration, max_gpus_per_job, log_interval=None):
    sc = SC.BY_NAME[name]
    kw = SC.build_inputs(sc)
    return S.flatten(kw["ingresses"], kw["dcs"], kw["graph"], kw["arrival_inf"], kw["arrival_train"], kw["coeffs_map"],
                     pc.build_policy(name=sc["policy"], max_gpus_per_job=max_gpus_per_job),
                     carbon_intensity=kw["carbon_intensity"], energy_price=kw["energy_price"], sim_duration=duration,
                     log_interval=log_interval or sc["log_interval"], algo=sc["algo"], power_cap=sc["power_cap"],
                     num_fixed_gpus=sc["num_fixed_gpus"], fixed_freq=sc["fixed_freq"])


def want_columns(eng) -> dict:
    """(columns, spread_columns) of every recorder from its documented layout (include/dcsim_b200.h), with W and the
    tick capacity as the engine reports them (0 when that recorder is off)."""
    from distributed_cluster_gpus_b200.engine import jres_mix_g
    sp, n_dc = eng.spec, eng.spec.n_dc
    rows = eng.job_ensemble_windows + 1
    cluster = eng.cluster_ensemble_capacity * len(EN.FIELDS) * n_dc
    job = rows * len(EN.JOB_FIELDS) * n_dc * 2
    waits = rows * len(EN.WAIT_FIELDS) * n_dc * 2
    win = rows * len(EN.RES_FIELDS) * n_dc * 2
    G = jres_mix_g(sp.max_gpus_per_job)
    return {"cluster_ensemble": (cluster, cluster),
            "job_ensemble": (job, job),
            "power_profile": (len(EN.PP_FIELDS) + n_dc + EN.PP_BINS, len(EN.PP_FIELDS) + n_dc),
            "job_waits": (waits, waits),
            "occupancy": (len(EN.OCC_STATS) * n_dc + 2 * EN.OCC_BINS * n_dc, len(EN.OCC_STATS) * n_dc),
            "tail_latency": (S.tail_cols(n_dc), S.tail_cols(n_dc)),
            "job_resources": (win + n_dc * 2 * (G * EN.RES_MAX_FREQ + 1 + EN.RES_EBINS), win),
            "energy_cost": (S.cost_cols(n_dc), S.cost_cols(n_dc))}


def _columns(eng) -> dict:
    from distributed_cluster_gpus_b200.engine import RECORDERS
    return {name: eng.stat_columns(name) for name in RECORDERS}


# name, scenario, duration [s], log_interval (None: the scenario's), max_gpus_per_job, job bin_s, cluster max_ticks
CASES = [
    ("1dc", "underloaded_1x64", 10.0, None, 8, None, None),
    ("ragged_3dc", "ragged_3dc_12_5_40", 10.0, None, 1, 1e9, 3),
    ("8dc", "cli_defaults_8dc_180s", 10.0, None, 64, 1.0, None),
    ("no_log_tick", "cfg3_4x64_sinusoid_120s", 3.0, 5.0, 8, None, None),
]


@pytest.mark.parametrize("case,name,duration,log_interval,max_gpus,bin_s,max_ticks", CASES, ids=[c[0] for c in CASES])
def test_columns_match_the_recorder_layouts(case, name, duration, log_interval, max_gpus, bin_s, max_ticks):
    from distributed_cluster_gpus_b200.engine import BatchedEngine
    sp = _spec(name, duration, max_gpus, log_interval)
    with BatchedEngine(sp, 8, base_seed=17) as off, BatchedEngine(sp, 8, base_seed=17) as on:
        assert _columns(off) == want_columns(off)     # every recorder off: W = 0, no ticks
        on.enable_cluster_ensemble(max_ticks)
        on.enable_job_ensemble(bin_s)
        on.enable_power_profile(None)
        on.enable_job_waits()
        on.enable_occupancy()
        on.enable_tail_latency(0.5)
        on.enable_job_resources()
        on.enable_energy_cost()
        before = _columns(on)
        assert before == want_columns(on)
        on.advance(0)
        off.advance(0)
        assert _columns(on) == before
        assert _columns(off) == want_columns(off)
        windows, ticks = on.job_ensemble_windows, on.cluster_ensemble_capacity
        # each recorder's two passes run over exactly these counts
        for rec, (cols, spread_cols) in before.items():
            mom, m2, hist = EN._recorder_passes(on, rec)
            assert mom.shape == (4, cols) and m2.shape == (spread_cols,) and hist.shape == (spread_cols, EN.BINS), rec
    assert windows == EN.job_windows(sp.end_time, bin_s or sp.log_interval) == {"8dc": 10, "1dc": 2}.get(case, 1)
    assert ticks == (3 if max_ticks else (0 if case == "no_log_tick" else int(duration / sp.log_interval)))
    assert (before["cluster_ensemble"] == (0, 0)) == (case == "no_log_tick")
    assert before["job_resources"][0] - before["job_resources"][1] == \
        sp.n_dc * 2 * (min(max_gpus, 32) * EN.RES_MAX_FREQ + 1 + EN.RES_EBINS)


def test_a_recorder_that_is_off_names_the_enable_call():
    """A cluster ensemble that is off has no columns: an empty result without a library call.  A job ensemble that is
    off has its W = 0 columns, and its moments pass fails with the library's message, which names the call that
    enables it (dcsim_recorder_enable)."""
    from distributed_cluster_gpus_b200.engine import BatchedEngine
    with BatchedEngine(_spec("underloaded_1x64", 10.0, 8), 4, base_seed=3) as eng:
        eng.advance(0)
        assert EN.cluster_ensemble(eng).n.size == 0
        with pytest.raises(N.DcsimError, match=r"job ensemble not enabled \(dcsim_recorder_enable\)") as ei:
            EN.job_ensemble(eng)
        assert ei.value.code == N.E_STATE


def test_unknown_statistic_ids_are_invalid():
    import torch
    from distributed_cluster_gpus_b200.engine import BatchedEngine, RECORDERS
    assert len(RECORDERS) == 8
    buf = torch.zeros(1024, dtype=torch.float64, device="cuda")
    p = C.c_void_p(buf.data_ptr())
    with BatchedEngine(_spec("underloaded_1x64", 10.0, 8), 4, base_seed=3) as eng:
        lib, h = eng._lib, eng._h
        for stat in (-1, 8):
            cols, spread = C.c_uint64(7), C.c_uint64(7)
            assert lib.dcsim_stat_columns(h, stat, C.byref(cols), C.byref(spread)) == N.E_INVALID
            assert (cols.value, spread.value) == (7, 7)
            assert lib.dcsim_stat_moments(h, stat, p) == N.E_INVALID
            assert lib.dcsim_stat_spread(h, stat, p, p, p, p, p) == N.E_INVALID
            assert b"unknown statistic" in lib.dcsim_last_error(h)
