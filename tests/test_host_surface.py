"""Host-side mirror of the reference surface: builders, leaves, flattening, C-ABI symbols (no GPU compute)."""
import ctypes as C
import math
import os
import re
from fractions import Fraction

import pytest

from conftest import ROOT
from distributed_cluster_gpus_b200 import _native, scenarios as SC, spec as S
from distributed_cluster_gpus_b200.configs import paper_config as pc
from distributed_cluster_gpus_b200.simcore.arrivals import ArrivalConfig
from distributed_cluster_gpus_b200.simcore.coeffs import TrainLatencyCoeffs, TrainPowerCoeffs
from distributed_cluster_gpus_b200.simcore.energy_paper import gpu_power_w, task_power_w
from distributed_cluster_gpus_b200.simcore.latency_paper import step_time_s
from distributed_cluster_gpus_b200.simcore.models import DataCenter, GPUType
from distributed_cluster_gpus_b200.simcore.policy_paper import best_energy_freq, best_nf_grid, energy_tuple


def test_library_loads_and_exports_every_declared_symbol():
    lib = _native.load()
    header = open(os.path.join(ROOT, "include", "dcsim_b200.h")).read()
    declared = set(re.findall(r"\b(dcsim_[a-z_]+)\s*\(", header)) - {"dcsim_t"}
    assert declared == set(_native.EXPORTS), declared ^ set(_native.EXPORTS)
    for name in declared:
        assert hasattr(lib, name), name
    assert lib.dcsim_sizeof_spec() == C.sizeof(S.Spec)
    assert lib.dcsim_summary_k() == S.SUMMARY_K == 88


def test_statistic_ids_follow_the_recorder_order():
    """engine.stat_* pass RECORDERS.index(name) as the library's DCSIM_STAT_* id."""
    from distributed_cluster_gpus_b200.engine import RECORDERS
    header = open(os.path.join(ROOT, "include", "dcsim_b200.h")).read()
    block = re.search(r"enum \{\s*(DCSIM_STAT_CLUSTER_ENSEMBLE = 0,.*?)\};", header, re.S).group(1)
    assert block.rstrip().endswith("DCSIM_STATS")
    assert [i.lower() for i in re.findall(r"DCSIM_STAT_([A-Z_]+)", block)] == list(RECORDERS)


def test_create_rejects_bad_arguments_without_a_gpu():
    lib = _native.load()
    h = C.c_void_p()
    assert lib.dcsim_create(None, 0, 1, 0, 0, 0, C.byref(h)) == _native.E_INVALID
    blob = bytearray(SC.to_spec(SC.CFG1).to_bytes())
    blob[0] ^= 0xFF
    buf = C.create_string_buffer(bytes(blob), len(blob))
    assert lib.dcsim_create(buf, len(blob), 1, 0, 0, 0, C.byref(h)) == _native.E_INVALID
    assert b"magic" in lib.dcsim_last_error(None)
    sp = SC.to_spec(SC.CFG1)
    sp.algo = 99
    buf = C.create_string_buffer(sp.to_bytes(), C.sizeof(sp))
    assert lib.dcsim_create(buf, C.sizeof(sp), 1, 0, 0, 0, C.byref(h)) == _native.E_UNSUPPORTED


def test_leaves_follow_the_reference_formulas():
    p, t = TrainPowerCoeffs(75.0, 80.0, 110.0), TrainLatencyCoeffs(0.0045, 0.032, 0.0012)
    assert gpu_power_w(0.6, p) == 75.0 * (0.6 ** 3) + 80.0 * 0.6 + 110.0
    assert task_power_w(8, 0.6, p) == 8 * gpu_power_w(0.6, p)
    assert task_power_w(-3, 1.0, p) == 0
    assert step_time_s(1, 0.5, t) == 0.0045 + 0.032 / 0.5
    assert step_time_s(4, 0.5, t) == (0.0045 + 0.032 / 0.5 + 0.0012 * 4) / 4
    assert step_time_s(0, 0.0, t) == 0.0045 + 0.032 / 1e-9
    T, P, E = energy_tuple(2, 0.8, p, t)
    assert E == P * T
    levels = [0.3, 0.4, 0.5, 0.6, 0.7, 0.8, 0.9, 1.0]
    n, f, *_ = best_nf_grid(8, levels, p, t)
    brute = min(((energy_tuple(nn, ff, p, t)[2], nn, ff) for nn in range(1, 9) for ff in levels))
    assert (n, f) == (brute[1], brute[2])
    assert best_energy_freq(n, levels, p, t) == f
    assert best_nf_grid(8, levels, p, t, objective="carbon", carbon_intensity=0.0)[:2] == (1, 0.3)  # all-zero scores: first wins


def test_cube_used_on_device_equals_libm_pow_for_every_frequency_in_use():
    """csrc dcsim_cube() returns the correctly rounded f^3; CPython's f ** 3 is libm pow(f, 3.0)."""
    freqs = {0.3, 0.4, 0.5, 0.6, 0.7, 0.8, 0.9, 1.0, 0.0, 1e-9, 0.55, 1.2}
    for f in freqs:
        assert float(Fraction(f) ** 3) == f ** 3, f


def test_datacenter_semantics():
    gt = GPUType("x", p_idle=45.0, p_peak=350.0, p_sleep=28.0)
    with pytest.raises(AssertionError):
        DataCenter("a", gt, 4, [0.5, 0.8], default_freq=1.0)
    dc = DataCenter("a", gt, 4, [0.5, 1.0])
    dc.busy_gpus, dc.current_freq = 3, 0.5
    assert dc.free_gpus == 1
    assert dc.instantaneous_power_w() == 3 * (45.0 + 350.0 * (0.5 ** 3.0)) + 1 * 28.0
    dc.accrue_energy(2.0)
    assert dc.energy_joules == 0.0 and dc.last_energy_time == 2.0   # first touch only arms the sentinel
    dc.accrue_energy(5.0, power_fn=lambda d: 10.0)
    assert dc.energy_joules == 30.0


def test_arrival_config_errors_and_edges():
    with pytest.raises(ValueError):
        ArrivalConfig("bogus", 1.0).lambda_t(0.0)
    with pytest.raises(ValueError):
        ArrivalConfig("bogus", 1.0).next_interarrival(0.0)
    assert ArrivalConfig("off", 5.0).next_interarrival(0.0) == math.inf
    assert ArrivalConfig("poisson", 0.0).next_interarrival(0.0) == math.inf
    a = ArrivalConfig("sinusoid", 10.0, amp=0.6, period=3600.0)
    assert a.lambda_t(900.0) == 10.0 * (1.0 + 0.6 * math.sin(2 * math.pi * 900.0 / 3600.0))


def test_flatten_validation_mirrors_reference_errors():
    kw = SC.build_inputs(SC.CFG3)
    base = dict(carbon_intensity=kw["carbon_intensity"], energy_price=kw["energy_price"])
    args = (kw["ingresses"], kw["dcs"], kw["graph"], kw["arrival_inf"], kw["arrival_train"], kw["coeffs_map"])
    with pytest.raises(ValueError, match="Unknown policy name"):
        S.flatten(*args, pc.build_policy(name="nope"), **base)
    with pytest.raises(ValueError, match="Unknown mode"):
        S.flatten(args[0], args[1], args[2], ArrivalConfig("weird", 1.0), *args[4:], kw["policy"], **base)
    with pytest.raises(NotImplementedError):
        S.flatten(*args, kw["policy"], algo="chsac_af", **base)
    with pytest.raises(ValueError, match="never terminate"):
        S.flatten(args[0], args[1], args[2], ArrivalConfig("sinusoid", 4.0, amp=1.5), *args[4:], kw["policy"], **base)
    with pytest.raises(ZeroDivisionError):
        S.flatten(*args, kw["policy"], log_interval=0.0, **base)


def test_flatten_tables():
    sp = SC.to_spec(SC.BY_NAME["sweep_carbon_cost"])
    assert sp.n_dc == 4 and sp.n_ing == 4 and sp.xfer_rule == S.START_NF_LUT and sp.deq_rule == S.START_NF_LUT
    # gw-us-west -> us-west is the 12 ms access link; unreachable pairs are +inf (their jobs are silently dropped)
    assert sp.transfer_s[0][0][0] == 12 / 1000.0
    assert sp.price_kwh_ok if hasattr(sp, "price_kwh_ok") else True
    assert [sp.dc[0].price_kwh[h] for h in (0, 7, 19)] == [0.12, 0.20, 0.16]
    assert sp.dc[0].carbon_intensity == 350.0 and sp.dc[1].carbon_intensity == 0.0
    sp5 = SC.to_spec(SC.CFG5)
    finite = [sp5.transfer_s[i][d][0] for i in range(8) for d in range(8) if math.isfinite(sp5.transfer_s[i][d][0])]
    assert len(finite) == 64 and max(finite) <= 0.4     # full 8x8 graph is connected
    assert sp5.nv_magicconst == 4 * math.exp(-0.5) / math.sqrt(2.0) and sp5.lognorm_mu == math.log(50000)


def test_cli_parses_reference_flags():
    from distributed_cluster_gpus_b200.run_sim_paper import parse_args
    a = parse_args(["--duration", "60", "--inf-mode", "poisson", "--inf-rate", "1.0", "--trn-mode", "off",
                    "--log-path", "/tmp/x", "--progress", "", "--algo", "joint_nf", "--eco-objective", "carbon",
                    "--num_fixed_gpus", "2", "--upgr-device", "cpu", "--replicas", "128", "--n-dc", "4"])
    assert a.duration == 60 and a.algo == "joint_nf" and a.replicas == 128 and a.n_dc == 4


def test_energy_price_map_forms():
    """SIM:986-1005: a global {hour: price} map, a per-DC {dc: {hour: price}} map, or nothing."""
    kw = SC.build_inputs(SC.BY_NAME["sweep_carbon_cost"])
    args = (kw["ingresses"], kw["dcs"], kw["graph"], kw["arrival_inf"], kw["arrival_train"], kw["coeffs_map"], kw["policy"])
    per_dc = {"us-west": {h: 0.5 for h in range(24)}, "us-east": {3: 0.25}}
    sp = S.flatten(*args, carbon_intensity=kw["carbon_intensity"], energy_price=per_dc, algo="carbon_cost")
    assert sp.dc[0].price_kwh[7] == 0.5 and sp.dc[1].price_kwh[3] == 0.25 and sp.dc[1].price_kwh[4] == 0.0
    assert sp.dc[2].price_kwh[0] == 0.0                      # DC absent from the map
    sp = S.flatten(*args, carbon_intensity=None, energy_price=None, algo="carbon_cost")
    assert all(sp.dc[d].price_kwh[h] == 0.0 for d in range(4) for h in range(24))
    assert sp.dc[0].carbon_intensity == 0.0
    # price 0 everywhere -> the carbon objective with CI = 0: every score is 0, the first grid point wins (n=1, f=levels[0])
    assert (sp.dc[0].nf_xfer[0][12].n, sp.dc[0].nf_xfer[0][12].f) == (1, 0.5)


def test_cli_gpus_flag_relaunches_through_torchrun(monkeypatch):
    """`run_sim_paper --gpus N` outside a launcher re-launches itself as N ranks (one process per GPU, rendezvous on
    127.0.0.1) with its own arguments; under a launcher (WORLD_SIZE set) it does not."""
    import subprocess
    from distributed_cluster_gpus_b200 import run_sim_paper as cli
    seen = {}

    class Done:
        returncode = 0

    def fake_run(cmd, check=False):
        seen["cmd"] = cmd
        return Done()
    monkeypatch.setattr(subprocess, "run", fake_run)
    monkeypatch.delenv("WORLD_SIZE", raising=False)
    argv = ["--gpus", "4", "--replicas", "1000", "--n-dc", "4", "--gpus-per-dc", "64", "--duration", "5"]
    assert cli.main(argv) is None
    cmd = seen["cmd"]
    assert "torch.distributed.run" in cmd and "--nproc-per-node=4" in cmd and "127.0.0.1" in cmd
    assert cmd[cmd.index("distributed_cluster_gpus_b200.run_sim_paper") + 1:] == argv


def test_shard_covers_every_replica_once():
    from distributed_cluster_gpus_b200 import sharding
    for total, world in ((1048576, 8), (65536, 3), (5, 8), (301, 2)):
        spans = [sharding.shard(total, r, world) for r in range(world)]
        assert spans[0][0] == 0 and sum(c for _, c in spans) == total
        for (f0, c0), (f1, _c1) in zip(spans, spans[1:]):
            assert f0 + c0 == f1


def test_summary_copy_helper_is_exact_for_small_and_large_arrays():
    """engine._copy_rows: the (threaded, for large arrays) private copy of the page-locked summary mirror."""
    import numpy as np
    from distributed_cluster_gpus_b200 import engine as E
    rng = np.random.default_rng(3)
    for rows in (1, 7, 4096, 65536, 65537):
        src = rng.random((rows, S.SUMMARY_K))
        dst = E._copy_rows(src)
        assert dst is not src and dst.flags["C_CONTIGUOUS"] and not np.shares_memory(dst, src)
        assert np.array_equal(dst, src)


def test_status_bits_of_header_and_python_mirror_agree():
    """include/dcsim_b200.h DCSIM_ST_* against spec.ST_* and the engine's descriptions (every bit has a name)."""
    import re
    from distributed_cluster_gpus_b200 import engine as E
    text = open(os.path.join(ROOT, "include", "dcsim_b200.h")).read()
    bits = {name: int(val) for name, val in re.findall(r"DCSIM_(ST_[A-Z_]+)\s*=\s*(\d+)", text)}
    assert bits and all(getattr(S, name) == val for name, val in bits.items())
    assert set(E.STATUS_NAMES) == set(bits.values())
    assert E.describe_status(0) == "ok" and "2^28" in E.describe_status(S.ST_SEQ_OVERFLOW)
