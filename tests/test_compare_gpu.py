"""Policy comparisons on the H100: members of a group (one arrival pre-pass) against standalone batches of the same
variants and against the oracle, the group's lifecycle and error codes, its memory, the paired reduction kernels against
the numpy mirror, capacity retries, a variant with its own pre-pass, and the CLI at one and two ranks."""
import csv

import numpy as np
import pytest

from conftest import has_cuda
from distributed_cluster_gpus_b200 import compare as CP, scenarios as SC, spec as S

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not has_cuda(), reason="needs a CUDA device")]

SWEEP = ["sweep_default_energy_aware", "sweep_default_perf_first", "sweep_joint_nf", "sweep_carbon_cost", "sweep_debug_n2",
         "sweep_debug_n8_f08", "sweep_bandit", "cap_greedy_4x64"]
WIDE = [SC.BY_NAME["cfg5_8x256_sinusoid_60s"], dict(SC.BY_NAME["cfg5_8x256_sinusoid_60s"], name="cfg5_joint_nf", algo="joint_nf"),
        dict(SC.BY_NAME["cfg5_8x256_sinusoid_60s"], name="cfg5_perf_first", policy="perf_first")]
RTOL = 1e-9


def _engine(sp, n, seed, **kw):
    from distributed_cluster_gpus_b200.engine import BatchedEngine
    return BatchedEngine(sp, n, base_seed=seed, **kw)


def _run(eng, chunk):
    if chunk:
        while not eng.all_done():
            eng.advance(chunk)
    else:
        eng.advance(0)
    return eng.summary()


def _standalone(sp, n, seed, chunk=0):
    with _engine(sp, n, seed) as eng:
        return _run(eng, chunk)


def _group(specs, n, seed, chunk=0):
    """The first spec owns the group; every other one is a member, run after the owner, all alive together."""
    from distributed_cluster_gpus_b200.engine import BatchedEngine
    owner = _engine(specs[0], n, seed)
    members = [BatchedEngine.shared(sp, owner) for sp in specs[1:]]
    try:
        out = [_run(e, chunk) for e in [owner] + members]
        infos = [e.launch_info() for e in [owner] + members]
    finally:
        for e in members + [owner]:
            e.close()
    return out, infos


def _close_to_oracle(got, sp, seed0):
    import oracle_lib
    want, _ = oracle_lib.run_batch(sp.to_bytes(), got.shape[0], seed0)
    for col in (S.S_STATUS, S.S_EVENTS, S.S_JOBS_FINISHED, S.S_JOBS_CREATED, S.S_FIN_INF, S.S_FIN_TRN, S.S_RNG_WORDS, S.S_SEQ,
                S.S_EV_ARRIVAL, S.S_EV_XFER, S.S_EV_FINISH, S.S_EV_LOG):
        assert np.array_equal(got[:, col], want[:, col]), col
    for col in (S.S_TOTAL_ENERGY_J, S.S_LAT_SUM, S.S_LAT_SUM_INF, S.S_LAT_SUM_TRN):
        g, w = got[:, col], want[:, col]
        rel = np.where(g == w, 0.0, np.abs(g - w) / np.maximum(np.abs(w), 1e-300))
        assert rel.max() <= RTOL, (col, float(rel.max()))


@pytest.mark.parametrize("chunk", [0, 997])
@pytest.mark.parametrize("build", ["lanes8_ragged", "lanes32"])
def test_members_equal_standalone_batches(build, chunk):
    """8 lanes per replica with 41 replicas (a ragged last warp; cap_greedy_4x64 is the <CAP> build), and 32 lanes
    (8 DC x 256): every member's summary rows are bit-identical to the same variant's standalone batch, one-shot and
    chunked; every member consumed the same random words; a small batch matches the oracle."""
    scs = [SC.BY_NAME[k] for k in SWEEP] if build == "lanes8_ragged" else WIDE
    n, seed = (41, 700) if build == "lanes8_ragged" else (16, 710)
    specs = [SC.to_spec(sc) for sc in scs]
    got, infos = _group(specs, n, seed, chunk)
    lanes = {i["lanes_per_replica"] for i in infos[:-1]}
    assert lanes == ({8} if build == "lanes8_ragged" else {32})
    for sp, g in zip(specs, got):
        assert np.all(g[:, S.S_STATUS] == 0)
        assert np.array_equal(g, _standalone(sp, n, seed, chunk))
        assert np.array_equal(g[:, S.S_RNG_WORDS], got[0][:, S.S_RNG_WORDS])
    if chunk == 0:
        for sp, g in zip(specs, got):
            _close_to_oracle(g[:8], sp, seed)


def test_lifecycle_reset_stale_streams_and_destroy_order():
    from distributed_cluster_gpus_b200 import _native as N
    from distributed_cluster_gpus_b200.engine import BatchedEngine
    a, b = SC.to_spec(SC.BY_NAME["sweep_default_energy_aware"]), SC.to_spec(SC.BY_NAME["sweep_joint_nf"])
    n = 24
    want_b_5, want_b_9 = _standalone(b, n, 5), _standalone(b, n, 9)
    owner = _engine(a, n, 5)
    m = BatchedEngine.shared(b, owner)
    try:
        m.advance(0)
        assert np.array_equal(m.summary(), want_b_5)
        owner.reset(9)                                    # new keys: the member's lists are stale
        with pytest.raises(N.DcsimError) as e:
            m.advance(0)
        assert e.value.code == N.E_STATE and "arrival source was reset" in str(e.value)
        with pytest.raises(N.DcsimError) as e:
            m.reset(5)                                    # not the owner's keys
        assert e.value.code == N.E_INVALID
        m.reset()                                         # the owner's current keys
        m.advance(0)
        assert np.array_equal(m.summary(), want_b_9)
        owner.advance(0)
        assert np.array_equal(owner.summary(), _standalone(a, n, 9))
        for call in (lambda: m.set_stream(0), lambda: m.set_rng("philox")):
            with pytest.raises(N.DcsimError) as e:
                call()
            assert e.value.code == N.E_STATE
        with pytest.raises(N.DcsimError) as e:
            BatchedEngine.shared(b, m)                    # no chains
        assert e.value.code == N.E_INVALID
        with pytest.raises(N.DcsimError) as e:
            BatchedEngine.shared(SC.to_spec(SC.BY_NAME["sweep_eco_route"]), owner)
        assert e.value.code == N.E_INVALID and "route_rule" in str(e.value)
        owner.close()                                     # the owner first: the member keeps the lists
        m.reset(9)
        m.advance(0)
        assert np.array_equal(m.summary(), want_b_9)
    finally:
        m.close()
        owner.close()


def test_seq_ring_size_decides_membership():
    """A spec whose cap_xfer implies a smaller seq ring would read list headers flagged against the owner's ring: it is
    refused, naming cap_xfer.  Other capacities with the same ring share, whichever handle runs the pre-pass: the member
    advancing first gives both handles their standalone rows."""
    from distributed_cluster_gpus_b200 import _native as N
    from distributed_cluster_gpus_b200.engine import BatchedEngine
    a = SC.to_spec(SC.BY_NAME["sweep_default_energy_aware"])
    n = 33
    with _engine(a, n, 12) as owner:
        with pytest.raises(N.DcsimError) as e:
            BatchedEngine.shared(SC.to_spec(SC.BY_NAME["sweep_joint_nf"], caps={"cap_xfer": 1}), owner)
        assert e.value.code == N.E_INVALID and "cap_xfer" in str(e.value)
        b = SC.to_spec(SC.BY_NAME["sweep_joint_nf"], caps={"cap_run": 9, "cap_q_inf": 7000, "cap_stale": 99, "cap_xfer": 40})
        with BatchedEngine.shared(b, owner) as m:
            m.advance(0)
            owner.advance(0)
            assert np.array_equal(m.summary(), _standalone(b, n, 12))
            assert np.array_equal(owner.summary(), _standalone(a, n, 12))
    small = SC.to_spec(SC.BY_NAME["sweep_joint_nf"], caps={"cap_xfer": 1})
    assert np.all(_standalone(small, 4, 12)[:, S.S_STATUS].astype(int) & S.ST_XFER_OVERFLOW)


def test_member_memory():
    import torch
    from distributed_cluster_gpus_b200.engine import BatchedEngine
    a, b = SC.to_spec(SC.BY_NAME["sweep_default_energy_aware"]), SC.to_spec(SC.BY_NAME["sweep_bandit"])
    n = 8192
    with _engine(a, n, 3) as owner:
        arr_bytes = owner.launch_info()["hbm_bytes_arrivals"]
        torch.cuda.synchronize()
        free0, _ = torch.cuda.mem_get_info()
        with BatchedEngine.shared(b, owner) as m:
            free1, _ = torch.cuda.mem_get_info()
            assert m.launch_info()["hbm_bytes_arrivals"] == 0
            assert free0 - free1 < arr_bytes
            m.advance(0)
            assert np.array_equal(m.summary()[:64], _standalone(b, 64, 3))


def test_paired_kernels_match_numpy_mirror_and_are_bit_stable():
    import torch
    from distributed_cluster_gpus_b200.engine import BatchedEngine
    a, b = SC.to_spec(SC.BY_NAME["sweep_default_energy_aware"]), SC.to_spec(SC.BY_NAME["cap_greedy_4x64"])
    n = 3001
    dev = torch.device("cuda", 0)
    with _engine(a, n, 17) as owner, BatchedEngine.shared(b, owner) as m:
        owner.advance(0)
        m.advance(0)
        base, var = owner.summary(), m.summary()
        vt = torch.from_numpy(var).to(dev)
        first = CP._paired_on_device(owner, vt, 4, dev, CP.EN.DEFAULT_QUANTILES)
        second = CP._paired_on_device(owner, vt, 4, dev, CP.EN.DEFAULT_QUANTILES)
    host = CP.paired_from_summaries(base, var, n_dc=4)
    for k in ("moments", "m2", "hist", "diff_quantiles", "n", "frac_lower"):
        assert np.array_equal(getattr(first, k), getattr(second, k), equal_nan=True), k
    assert np.array_equal(first.moments[[0, 2, 3]], host.moments[[0, 2, 3]])          # n, min, max
    assert np.array_equal(first.hist, host.hist) and np.array_equal(first.n, host.n)
    np.testing.assert_allclose(first.moments[1], host.moments[1], rtol=1e-12, atol=1e-6)
    np.testing.assert_allclose(first.diff_mean, host.diff_mean, rtol=1e-12, atol=1e-9)
    from test_compare import numpy_pair_check
    numpy_pair_check(first, base, var, 4)


def _factory(sc, tiny=None):
    def f(caps):
        c = dict(caps)
        for k, v in (tiny or {}).items():
            c.setdefault(k, v)
        return SC.to_spec(sc, caps=c)
    return f


def test_compare_variants_retries_and_own_prepass():
    """A member started with a tiny cap_run retries alone (still shared); a too-small cap_arrivals or cap_xfer rebuilds
    the group; eco_route runs with its own pre-pass.  Every summary equals its standalone batch."""
    from distributed_cluster_gpus_b200 import engine as E
    n, seed = 33, 4242
    scs = {k: SC.BY_NAME[k] for k in ("sweep_default_energy_aware", "sweep_joint_nf", "sweep_eco_route", "cap_greedy_4x64")}
    plain = {k: E.run_to_completion(_factory(sc), n, seed)[1] for k, sc in scs.items()}
    E.free_cached_engine()
    res = CP.compare_variants({"base": _factory(scs["sweep_default_energy_aware"]),
                               "joint_nf": _factory(scs["sweep_joint_nf"], {"cap_run": 2}),
                               "eco": _factory(scs["sweep_eco_route"]),
                               "cap": _factory(scs["cap_greedy_4x64"])}, "base", n, seed)
    assert res.shared_arrivals == {"joint_nf": True, "eco": False, "cap": True}
    for name, key in (("base", "sweep_default_energy_aware"), ("joint_nf", "sweep_joint_nf"), ("eco", "sweep_eco_route"),
                      ("cap", "cap_greedy_4x64")):
        assert np.array_equal(res.summaries[name], plain[key]), name
        if name != "base":
            np.testing.assert_allclose(res.stats[name].diff_mean,
                                       CP.paired_from_summaries(plain["sweep_default_energy_aware"], plain[key], n_dc=4).diff_mean,
                                       rtol=1e-12, atol=1e-9)
    small = CP.compare_variants({"base": _factory(scs["sweep_default_energy_aware"], {"cap_arrivals": 6000}),
                                 "cap": _factory(scs["cap_greedy_4x64"], {"cap_arrivals": 6000})}, "base", n, seed)
    assert small.shared_arrivals == {"cap": True}
    assert np.array_equal(small.summaries["base"], plain["sweep_default_energy_aware"])
    assert np.array_equal(small.summaries["cap"], plain["cap_greedy_4x64"])
    # a seq ring too small for the lists (max_ahead ~43 here, 12 -> 32 entries): the owner is rebuilt with cap_xfer 24,
    # the members take it and stay in the group
    ring = CP.compare_variants({"base": _factory(scs["sweep_default_energy_aware"], {"cap_xfer": 12}),
                                "joint_nf": _factory(scs["sweep_joint_nf"], {"cap_xfer": 12}),
                                "cap": _factory(scs["cap_greedy_4x64"], {"cap_xfer": 12})}, "base", n, seed)
    assert ring.shared_arrivals == {"joint_nf": True, "cap": True}
    for name, key in (("base", "sweep_default_energy_aware"), ("joint_nf", "sweep_joint_nf"), ("cap", "cap_greedy_4x64")):
        assert np.array_equal(ring.summaries[name], plain[key]), name


def _read_csv(path):
    with open(path) as f:
        rd = csv.reader(f)
        return next(rd), [r for r in rd]


def test_cli_compare_one_and_two_ranks(tmp_path):
    import json
    import torch
    from test_gpu_parity import _run_cli
    common = ["--duration", "20", "--inf-mode", "sinusoid", "--inf-rate", "10", "--inf-period", "3600", "--trn-rate", "1",
              "--n-dc", "4", "--gpus-per-dc", "64", "--replicas", "301", "--seed", "77", "--progress", "",
              "--power-cap", "20000", "--compare-algos", "default_policy,joint_nf,cap_greedy"]
    one = _run_cli(common + ["--log-path", str(tmp_path / "one" / "x"), "--compare-csv", str(tmp_path / "one.csv"),
                             "--summary-json", str(tmp_path / "one.json")])
    assert one.returncode == 0, one.stderr[-2000:]
    assert one.stdout.count("Done.") == 3
    extra = {} if torch.cuda.device_count() >= 2 else {"DCSIM_DIST_BACKEND": "gloo"}
    two = _run_cli(common + ["--gpus", "2", "--log-path", str(tmp_path / "two" / "x"), "--compare-csv",
                             str(tmp_path / "two.csv")], extra)
    assert two.returncode == 0, two.stderr[-3000:]
    ha, a = _read_csv(tmp_path / "one.csv")
    hb, b = _read_csv(tmp_path / "two.csv")
    assert ha == hb and ha[-2:] == ["var_ratio", "shared_arrivals"]
    assert len(a) == len(b) == 2 * (len(CP.METRICS) + 4)
    exact = {ha.index(k) for k in ("variant", "baseline", "metric", "dc", "n", "frac_lower", "frac_higher", "shared_arrivals")}
    for ra, rb in zip(a, b):
        for i, (x, y) in enumerate(zip(ra, rb)):
            if i in exact or x == y:
                assert x == y, (ha[i], ra, rb)
            else:
                fx, fy = float(x), float(y)
                assert abs(fx - fy) <= 1e-9 * max(abs(fx), abs(fy), 1e-300) or ha[i].startswith("diff_p"), (ha[i], ra, rb)
    doc = json.load(open(tmp_path / "one.json"))
    assert set(doc["algos"]) == {"default_policy", "joint_nf", "cap_greedy"} and doc["algos"]["joint_nf"]["replicas"] == 301
    assert not (tmp_path / "one" / "x" / "cluster_log.csv").exists()
    bad = _run_cli(common + ["--ensemble-csv", str(tmp_path / "e.csv")])
    assert bad.returncode != 0 and "--compare-algos" in bad.stderr
