"""The arrival pre-pass and the list merge on the device, entry by entry.

The hook build (-DDCSIM_TEST_HOOKS, tests/gpuhooks) exports dcsim_test_poison_prepass and dcsim_test_fetch_prepass:
the pre-pass and merge buffers are filled with 0xee bytes before dcsim_prepare, and afterwards the arrivals, the
merged list and the header of chosen replicas are copied out.  They are held to the references of
test_arrival_lists.py:

  * the list equals tests/list_reference.py built from the device's own arrivals, byte for byte, for every entry below
    ml_count; max_ahead and the status bits are exact;
  * the arrivals equal the stepped oracle (tests/oracle_jobs/oracle_lists.c): meta, pred, the next-arrival bit, count,
    first_mask and rng_words exactly, instants within 1e-12 relative (the trace bar of test_event_ties_gpu.py), job
    sizes within SIZE_ULP units in the last place (libdevice pow / exp against glibc; the largest distance seen is
    printed);
  * every discrete field equals the host build's.

At quantum 0 the hook build and the product library give bit-identical summaries on the same scenarios, which ties
what is pinned here to the product's kernels."""
import glob
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import hostemu_lib as H
import list_reference as LR
from conftest import ROOT, has_cuda
from distributed_cluster_gpus_b200 import scenarios as SC, spec as S
from test_arrival_lists import (CASES, COUNT_EDGE_BATCH, COUNT_EDGES, ST_ARRIVALS_OVERFLOW, check_arrivals, check_lists,
                                count_edge_specs, edge_reached, huge_transfer_spec, _short)

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not has_cuda(), reason="needs a CUDA device")]

T_RTOL = 1e-12
SIZE_ULP = 8
CPUS = os.cpu_count() or 1
GPU_REPLICAS = {"cfg3": 41}            # a ragged last warp in the arrivals kernel's flush and a partial merge CTA
BENCH_N, BENCH_SEED = 65536, 123       # bench.py's batch (cfg3, 120 s)
BENCH_PICK = sorted({0, 31, 32, 65535} | set(np.random.default_rng(7).choice(BENCH_N, 252, replace=False).tolist()))
RESET = {"seed": 5150, "first_replica_id": 1000}


def _case(name):
    make, n, seed, rng, q = CASES[name]
    return make(), GPU_REPLICAS.get(name, n), seed, rng, q


def _cap_specs():
    sc = _short("cfg3_4x64_sinusoid_120s", 10.0)
    full = SC.to_spec(sc)
    counts = H.prepass(full.to_bytes(), 12, 600)["hdr"]["count"].astype(int)
    return full, SC.to_spec(sc, caps={"cap_arrivals": int(np.sort(counts)[6])}), counts


def _jobs():
    jobs = []
    for name in CASES:
        sp, n, seed, rng, q = _case(name)
        jobs.append({"kind": "prepass", "name": f"case_{name}", "spec_hex": sp.to_bytes().hex(), "n": n, "seed": seed, "q": q,
                     "rng": "mt19937" if rng else "philox"})
        if q == 0.0:
            jobs.append({"kind": "summary", "name": f"summary_{name}", "spec_hex": sp.to_bytes().hex(), "n": n, "seed": seed,
                         "q": 0.0, "rng": "mt19937" if rng else "philox"})
    for (i, n), sp in zip(COUNT_EDGE_BATCH, count_edge_specs()):
        jobs.append({"kind": "prepass", "name": f"counts_{i}", "spec_hex": sp.to_bytes().hex(), "n": n, "seed": 4000 + i, "q": 0.0})
    full, capped, _ = _cap_specs()
    for tag, sp in (("full", full), ("capped", capped)):
        jobs.append({"kind": "prepass", "name": f"cap_{tag}", "spec_hex": sp.to_bytes().hex(), "n": 12, "seed": 600, "q": 0.0})
    sp = SC.to_spec(_short("cfg3_4x64_sinusoid_120s"))
    jobs.append({"kind": "prepass", "name": "reseeded", "spec_hex": sp.to_bytes().hex(), "n": 9, "seed": 11, "q": 0.0,
                 "reset": RESET})
    jobs.append({"kind": "prepass", "name": "bench", "spec_hex": SC.to_spec(SC.CFG3).to_bytes().hex(), "n": BENCH_N,
                 "seed": BENCH_SEED, "q": 0.0, "replicas": BENCH_PICK})
    return jobs


@pytest.fixture(scope="module")
def dev(tmp_path_factory):
    """Runs every job through the hook build, in a process of its own (tests/gpuhooks/driver.py)."""
    import __graft_entry__ as G
    srcs = glob.glob(os.path.join(G.CSRC, "*.cu*")) + [os.path.join(ROOT, "include", "dcsim_b200.h")]
    if not G._newer(G.HOOK_LIB, srcs):
        G.build()
    out = tmp_path_factory.mktemp("prepass_runs")
    with open(out / "jobs.json", "w") as f:
        json.dump(_jobs(), f)
    res = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "gpuhooks", "driver.py"), str(out / "jobs.json"), str(out)],
                         env=dict(os.environ, DCSIM_B200_LIB=G.HOOK_LIB), capture_output=True, text=True, timeout=1800)
    assert res.returncode == 0, res.stderr[-3000:]

    def load(name):
        with np.load(out / (name + ".npz")) as z:
            d = {k: z[k] for k in z.files}
        if "hdr" in d:
            d["hdr"] = d["hdr"].view(H.HDR_DTYPE).reshape(-1)
        return d
    return load


def _same_discrete(d, h, rows_d, rows_h):
    """Device rows rows_d of d against host rows rows_h of h: every discrete field equal."""
    for i, j in zip(rows_d, rows_h):
        hd, hh = d["hdr"][i], h["hdr"][j]
        for f in ("count", "first_mask", "rng_words", "status", "ml_count", "max_ahead"):
            assert hd[f] == hh[f], (i, f, hd[f], hh[f])
        c, m = int(hd["count"]), int(hd["ml_count"])
        for f in ("arr_meta", "arr_pred"):
            assert np.array_equal(d[f][i, :c], h[f][j, :c]), (i, f)
        assert np.array_equal(d["ml_meta"][i, :m], h["ml_meta"][j, :m]), i
        xin = (d["ml_meta"][i, :m] & 1) == 0                # arrival entries: aux is the xfer_done's position
        assert np.array_equal(d["ml_aux"][i, :m][xin].view(np.uint64), h["ml_aux"][j, :m][xin].view(np.uint64)), i


def _report(label, worst_t, worst_ulp):
    print(f"{label}: largest t deviation from the oracle {worst_t:.3e} (relative), largest size distance {worst_ulp} ulp")


@pytest.mark.parametrize("name", list(CASES))
def test_device_lists_and_arrivals(dev, name):
    sp, n, seed, rng, q = _case(name)
    d = dev(f"case_{name}")
    assert np.array_equal(d["replicas"], np.arange(n))
    assert np.all((d["hdr"]["status"] | LR.ST_XFER_OVERFLOW) == LR.ST_XFER_OVERFLOW)
    refs = check_lists(sp, d, range(n), q)
    rows, worst_t, worst_ulp = check_arrivals(sp, d, range(n), seed, rng, q, T_RTOL, SIZE_ULP)
    edge_reached(name, sp, refs, rows)
    h = H.prepass(sp.to_bytes(), n, seed, rng, "plain", q)
    _same_discrete(d, h, range(n), range(n))
    _report(name, worst_t, worst_ulp)


@pytest.mark.parametrize("name", [k for k in CASES if CASES[k][4] == 0.0])
def test_hook_build_equals_product_library(dev, oracle, name):
    """At quantum 0 the hook build computes what the product library does, bit for bit; the product equals the oracle's
    event count."""
    from distributed_cluster_gpus_b200.engine import BatchedEngine
    sp, n, seed, rng, _ = _case(name)
    d = dev(f"summary_{name}")
    with BatchedEngine(sp, n, base_seed=seed) as eng:
        if rng:
            eng.set_rng("mt19937")
        events = eng.advance(0)
        got = eng.summary()
    assert int(d["events"]) == events and np.array_equal(d["summary"], got)
    want, want_total = oracle.run_batch(sp.to_bytes(), n, seed, 0, rng, n_threads=CPUS)
    if name != "xfer_ring_overflow":                        # that one stops at its status bit
        assert events == want_total and np.array_equal(got[:, S.S_EVENTS], want[:, S.S_EVENTS])


def test_device_counts_at_chunk_edges(dev):
    seen, worst_t, worst_ulp = set(), 0.0, 0
    for (i, n), sp in zip(COUNT_EDGE_BATCH, count_edge_specs()):
        d = dev(f"counts_{i}")
        counts = d["hdr"]["count"]
        seen |= set(int(c) for c in counts)
        check_lists(sp, d, range(n), 0.0)
        pick = [r for r in range(n) if counts[r] in COUNT_EDGES]
        _, wt, wu = check_arrivals(sp, d, pick, 4000 + i, 0, 0.0, T_RTOL, SIZE_ULP)
        worst_t, worst_ulp = max(worst_t, wt), max(worst_ulp, wu)
        _same_discrete(d, H.prepass(sp.to_bytes(), n, 4000 + i), range(n), range(n))
    assert set(COUNT_EDGES) <= seen, sorted(set(COUNT_EDGES) - seen)
    _report("count edges", worst_t, worst_ulp)


def test_device_arrival_capacity_edge(dev):
    full_sp, sp, counts = _cap_specs()
    full, d = dev("cap_full"), dev("cap_capped")
    over = counts > sp.cap_arrivals
    assert np.any(counts == sp.cap_arrivals) and np.any(over)
    assert np.array_equal(full["hdr"]["count"], counts)
    assert np.array_equal((d["hdr"]["status"] & ST_ARRIVALS_OVERFLOW) != 0, over)
    check_lists(sp, d, range(12), 0.0)
    check_arrivals(sp, d, range(12), 600, 0, 0.0, T_RTOL, SIZE_ULP)
    w_full, w_cap = full_sp.cap_arrivals, sp.cap_arrivals
    for r in np.flatnonzero(~over):                          # rows of the replicas that fit are intact
        c, m = counts[r], int(full["hdr"]["ml_count"][r])
        assert d["hdr"]["ml_count"][r] == m
        for f in ("arr_t", "arr_raw", "arr_meta", "arr_pred"):
            assert np.array_equal(d[f][r, :c], full[f][r, :c]), (r, f)
        for f in ("ml_t", "ml_aux", "ml_meta"):
            assert np.array_equal(d[f][r, :m].view(np.uint8), full[f][r, :m].view(np.uint8)), (r, f)
    assert d["arr_t"].shape[1] == w_cap and full["arr_t"].shape[1] == w_full


def test_device_second_batch_after_reset(dev):
    """The same handle reseeded with another key and a nonzero first_replica_id: replica r has key seed + first + r."""
    sp = SC.to_spec(_short("cfg3_4x64_sinusoid_120s"))
    first, again = dev("reseeded"), dev("reseeded__reset")
    key0 = RESET["seed"] + RESET["first_replica_id"]
    for d, k in ((first, 11), (again, key0)):
        check_lists(sp, d, range(9), 0.0)
        check_arrivals(sp, d, range(9), k, 0, 0.0, T_RTOL, SIZE_ULP)
    assert not np.array_equal(first["hdr"]["count"], again["hdr"]["count"])


def test_device_bench_batch_sample(dev):
    """256 replicas of bench.py's 65 536-replica batch, replicas 0, 31, 32 and 65 535 among them."""
    sp = SC.to_spec(SC.CFG3)
    d = dev("bench")
    assert np.array_equal(d["replicas"], BENCH_PICK) and {0, 31, 32, BENCH_N - 1} <= set(BENCH_PICK)
    rows = range(len(BENCH_PICK))
    assert np.all(d["hdr"]["status"] == 0)
    check_lists(sp, d, rows, 0.0)
    worst_t, worst_ulp = 0.0, 0
    for i, r in enumerate(BENCH_PICK):
        sub = {k: v[i:i + 1] for k, v in d.items() if k != "replicas"}
        _, wt, wu = check_arrivals(sp, sub, [0], BENCH_SEED + r, 0, 0.0, T_RTOL, SIZE_ULP)
        worst_t, worst_ulp = max(worst_t, wt), max(worst_ulp, wu)
        h = H.prepass(sp.to_bytes(), 1, BENCH_SEED + r)
        _same_discrete(sub, h, [0], [0])
    _report("bench sample", worst_t, worst_ulp)


def test_device_huge_finite_transfer_end_to_end(oracle):
    """The product library on the huge-transfer spec: event counts equal the oracle's, every replica clean."""
    from distributed_cluster_gpus_b200.engine import BatchedEngine
    sp = huge_transfer_spec()
    want, want_total = oracle.run_batch(sp.to_bytes(), 41, 123, 0, n_threads=CPUS)
    with BatchedEngine(sp, 41, base_seed=123) as eng:
        events = eng.advance(0)
        got = eng.summary()
    assert np.all(got[:, S.S_STATUS] == 0)
    assert events == want_total and np.array_equal(got[:, S.S_EVENTS], want[:, S.S_EVENTS])
