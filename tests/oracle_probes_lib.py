"""TEST-ONLY ctypes access to the probes of the stepped C oracle (tests/oracle_jobs/oracle_probes.c): per-job instants,
the per-arrival record, the occupancy checkers, every created job, the power profile and the energy cost."""
import ctypes as C
import os
import subprocess

import numpy as np

from distributed_cluster_gpus_b200 import ensemble as EN, spec as S

_HERE = os.path.dirname(os.path.abspath(__file__))
_DIR = os.path.join(_HERE, "oracle_jobs")
_SO = os.path.join(_DIR, "_build", "liboracle_probes.so")
_SRCS = tuple(os.path.join(_DIR, f) for f in ("oracle_probes.c", "oracle_jobs.c", "oracle_lists.c", "oracle_occ.c",
                                              "oracle_tail.c", "oracle_power.c", "oracle_cost.c", "build.sh")) + (
    os.path.join(_HERE, "..", "oracle", "dcsim_oracle.c"), os.path.join(_HERE, "..", "include", "dcsim_b200.h"))
JOB_ROW_DTYPE = np.dtype([("jid", "<u4"), ("dc", "<i4"), ("jtype", "<i4"), ("at_xfer", "<i4"), ("arrival", "<f8"),
                          ("xfer_done", "<f8"), ("start", "<f8"), ("finish", "<f8")])
ARR_ROW_DTYPE = np.dtype([("t", "<f8"), ("size", "<f8"), ("tx", "<f8"), ("stream", "<u4"), ("dc", "<i4"), ("pred", "<u4"),
                          ("next", "<u4")])
REACHED_DTYPE = np.dtype([("jid", "<u4"), ("dc", "<i4"), ("jtype", "<i4"), ("pad", "<u4"), ("xfer_done", "<f8"),
                          ("start", "<f8"), ("finish", "<f8")])
TAIL_ROW_DTYPE = np.dtype([("jid", "<u4"), ("jtype", "<i4"), ("dc", "<i4"), ("finished", "<i4"), ("arrival", "<f8"),
                           ("xfer_done", "<f8"), ("start", "<f8"), ("finish", "<f8")])
_lib = None


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(_SO) or any(os.path.getmtime(s) > os.path.getmtime(_SO) for s in _SRCS):
            subprocess.run([os.path.join(_DIR, "build.sh")], check=True, capture_output=True)
        L = C.CDLL(_SO)
        vp, u64 = C.c_void_p, C.c_uint64
        L.dcoracle_set_test_time_quantum.argtypes = [C.c_double]
        for name, extra in (("oraclejobs_run", [C.c_uint32]), ("oraclelists_run", [C.c_uint32, vp]),
                            ("oracleocc_occupancy", []), ("oracleocc_reached", [C.c_uint32]),
                            ("oracletail_run", [C.c_uint32]), ("oraclecost_run", [])):
            getattr(L, name).restype = C.c_longlong
            getattr(L, name).argtypes = [vp, C.c_size_t, u64, C.c_int, vp] + extra
        L.oraclepower_profile.restype = C.c_longlong
        L.oraclepower_profile.argtypes = [vp, C.c_size_t, u64, C.c_int, vp, C.c_double, C.c_double]
        _lib = L
    return _lib


def set_test_time_quantum(q):
    """The oracle's tie hook (0 = off)."""
    lib().dcoracle_set_test_time_quantum(float(q))


def _rows(fn, spec_bytes, seed, rng_kind, dtype, cap, *extra):
    out = np.zeros(cap, dtype=dtype)
    n = fn(spec_bytes, len(spec_bytes), seed & (2**64 - 1), rng_kind, out.ctypes.data, cap, *extra)
    if n < 0:
        raise ValueError("the oracle rejected the spec blob")
    assert n <= cap, "raise cap"
    return out[:n]


def oracle_jobs(spec_bytes, seed, rng_kind=0, cap=200000):
    """One replica's finished jobs in finish order (JOB_ROW_DTYPE): jid, dc, jtype, at_xfer (started by its own
    xfer_done event), arrival, xfer_done, start, finish — the oracle's instants."""
    return _rows(lib().oraclejobs_run, spec_bytes, seed, rng_kind, JOB_ROW_DTYPE, cap)


def arrivals(spec_bytes, seed, rng_kind=0, quantum=0.0, cap=1 << 20):
    """One replica's arrivals as the oracle processes them -> (rows ARR_ROW_DTYPE, first_mask, rng_words).  `quantum`:
    the oracle's tie-quantizing hook, reset to 0 afterwards."""
    info = np.zeros(2, dtype=np.uint64)
    set_test_time_quantum(quantum)
    try:
        rows = _rows(lib().oraclelists_run, spec_bytes, seed, rng_kind, ARR_ROW_DTYPE, cap, info.ctypes.data)
    finally:
        set_test_time_quantum(0.0)
    return rows, int(info[0]), int(info[1])


def oracle_occupancy(spec_bytes, seed, rng_kind=0):
    """One replica's occupancy columns [1 + OCC_FIELDS * n_dc + 2 * OCC_BINS * n_dc] from the oracle stepped one event
    at a time."""
    n_dc = S.Spec.from_buffer_copy(spec_bytes).n_dc
    row = np.zeros(1 + S.OCC_FIELDS * n_dc + 2 * S.OCC_BINS * n_dc)
    if lib().oracleocc_occupancy(spec_bytes, len(spec_bytes), seed & (2**64 - 1), rng_kind, row.ctypes.data) < 0:
        raise ValueError("the oracle rejected the spec blob")
    return row


def oracle_power_profile(spec_bytes, seed, threshold, rng_kind=0, hi=None):
    """One replica's power-profile column [PP_FIELDS + n_dc + PP_BINS] from the oracle stepped one event at a time,
    over `threshold` (+inf: none).  `hi`: the histogram range; None takes the library's (dcsim_power_profile_range
    through the host build), which tests/test_power_profile.py pins against the reference fixtures."""
    if hi is None:
        import hostemu_lib
        hi = hostemu_lib.power_range(spec_bytes)
    n_dc = S.Spec.from_buffer_copy(spec_bytes).n_dc
    row = np.zeros(S.PP_FIELDS + n_dc + S.PP_BINS)
    n = lib().oraclepower_profile(spec_bytes, len(spec_bytes), seed & (2**64 - 1), rng_kind, row.ctypes.data,
                                  float(threshold), float(hi))
    if n == -2:
        raise AssertionError("the oracle's DCs accrued energy at different instants")
    if n < 0:
        raise ValueError("the oracle rejected the spec blob")
    return row


def oracle_energy_cost(spec_bytes, seed, rng_kind=0):
    """One replica's energy-cost column [cost_cols(n_dc)] from the oracle stepped one event at a time."""
    n_dc = S.Spec.from_buffer_copy(spec_bytes).n_dc
    row = np.zeros(S.cost_cols(n_dc))
    if lib().oraclecost_run(spec_bytes, len(spec_bytes), seed & (2**64 - 1), rng_kind, row.ctypes.data) < 0:
        raise ValueError("the oracle rejected the spec blob")
    return row


def oracle_reached(spec_bytes, seed, rng_kind=0, cap=400000):
    """Every job that reached its DC (REACHED_DTYPE, xfer_done order); start / finish +inf when not by end_time."""
    return _rows(lib().oracleocc_reached, spec_bytes, seed, rng_kind, REACHED_DTYPE, cap)


def oracle_created(spec_bytes, seed, rng_kind=0, cap=400000):
    """One replica's created jobs in jid order (EN.TAIL_JOB_DTYPE; finish NaN: not finished by end_time) — the
    oracle's instants."""
    rows = _rows(lib().oracletail_run, spec_bytes, seed, rng_kind, TAIL_ROW_DTYPE, cap)
    n = len(rows)
    assert np.array_equal(rows["jid"], np.arange(1, n + 1))
    jobs = np.zeros(n, dtype=EN.TAIL_JOB_DTYPE)
    for f in ("jtype", "dc", "arrival", "xfer_done", "start", "finish"):
        jobs[f] = rows[f]
    assert np.all(np.isnan(jobs["finish"]) == (rows["finished"] == 0))
    return jobs
