"""TEST-ONLY ctypes access to the host build of the device core with the waiting / response-time recorder
(tests/hostemu_ens/hostemu_jwait.cpp) and to the oracle's per-job instants (tests/oracle_jobs/oracle_jobs.c)."""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_DIR = os.path.join(_HERE, "hostemu_ens")
_SO = os.path.join(_DIR, "_build", "libdcsim_hostemu_jwait.so")
_SO_UNIFORM = os.path.join(_DIR, "_build", "libdcsim_hostemu_jwait_uniform.so")
_SRCS = (os.path.join(_DIR, "hostemu_jwait.cpp"), os.path.join(_DIR, "build_jwait.sh"),
         os.path.join(_HERE, "..", "distributed_cluster_gpus_b200", "csrc", "dcsim_core.cuh"),
         os.path.join(_HERE, "..", "include", "dcsim_b200.h"))
_ODIR = os.path.join(_HERE, "oracle_jobs")
_OSO = os.path.join(_ODIR, "_build", "liboracle_jobs.so")
_OSRCS = (os.path.join(_ODIR, "oracle_jobs.c"), os.path.join(_ODIR, "build.sh"),
          os.path.join(_HERE, "..", "oracle", "dcsim_oracle.c"), os.path.join(_HERE, "..", "include", "dcsim_b200.h"))
SUMMARY_K = 24 + 8 * 8
LAT_BINS = 128
_libs = {}

JOB_ROW_DTYPE = np.dtype([("jid", "<u4"), ("dc", "<i4"), ("jtype", "<i4"), ("at_xfer", "<i4"), ("arrival", "<f8"),
                          ("xfer_done", "<f8"), ("start", "<f8"), ("finish", "<f8")])


def _stale(so, srcs):
    return not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in srcs)


def _bind(path):
    L = C.CDLL(path)
    L.hostemu_jwait_set_test_time_quantum.argtypes = [C.c_double]
    L.hostemu_jwait_windows.restype = C.c_uint64
    L.hostemu_jwait_windows.argtypes = [C.c_void_p, C.c_double]
    L.hostemu_jwait_run_batch.restype = C.c_longlong
    L.hostemu_jwait_run_batch.argtypes = [C.c_void_p, C.c_size_t, C.c_uint64, C.c_uint64, C.c_uint64, C.c_void_p,
                                          C.c_int, C.c_double, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    return L


def lib(uniform=False):
    if not _libs:
        if _stale(_SO, _SRCS) or _stale(_SO_UNIFORM, _SRCS):
            subprocess.run([os.path.join(_DIR, "build_jwait.sh")], check=True, capture_output=True)
        _libs[False], _libs[True] = _bind(_SO), _bind(_SO_UNIFORM)
    return _libs[bool(uniform)]


def oracle_lib():
    if "oracle" not in _libs:
        if _stale(_OSO, _OSRCS):
            subprocess.run([os.path.join(_ODIR, "build.sh")], check=True, capture_output=True)
        L = C.CDLL(_OSO)
        L.oraclejobs_set_test_time_quantum.argtypes = [C.c_double]
        L.oraclejobs_run.restype = C.c_longlong
        L.oraclejobs_run.argtypes = [C.c_void_p, C.c_size_t, C.c_uint64, C.c_int, C.c_void_p, C.c_uint32]
        _libs["oracle"] = L
    return _libs["oracle"]


def set_test_time_quantum(q):
    """The tie hook (0 = off) in both the host build and the oracle's per-job run."""
    lib(False).hostemu_jwait_set_test_time_quantum(float(q))
    lib(True).hostemu_jwait_set_test_time_quantum(float(q))
    oracle_lib().oraclejobs_set_test_time_quantum(float(q))


def oracle_jobs(spec_bytes, seed, rng_kind=0, cap=200000):
    """One replica's finished jobs in finish order (JOB_ROW_DTYPE): jid, dc, jtype, at_xfer (started by its own
    xfer_done event), arrival, xfer_done, start, finish — the oracle's instants."""
    out = np.zeros(cap, dtype=JOB_ROW_DTYPE)
    buf = C.create_string_buffer(spec_bytes, len(spec_bytes))
    n = oracle_lib().oraclejobs_run(buf, len(spec_bytes), seed & (2**64 - 1), rng_kind, out.ctypes.data, cap)
    if n < 0:
        raise ValueError("oracle_jobs rejected the spec blob")
    assert n <= cap, "raise cap"
    return out[:n]


def run_batch(spec_bytes, n_replicas, seed0, bin_s, chunk_events=0, rng_kind=0, uniform=False, waits=True):
    """-> {"summary": [n, SUMMARY_K], "events": int, "jens": [W + 1, 2, n_dc, 2, n], "jens_hist": [n, n_dc, 2, LAT_BINS],
    "rows": [W + 1, 3, n_dc, 2, n] float64 or None, "hist": [n, n_dc, 2 kinds, 2, LAT_BINS] uint32 or None}.
    waits=False: the waits recorder off (the job ensemble stays on)."""
    out = np.zeros((n_replicas, SUMMARY_K))
    buf = C.create_string_buffer(spec_bytes, len(spec_bytes))
    n_dc = C.c_int32.from_buffer_copy(spec_bytes[16:20]).value      # dcsim_spec_t.n_dc
    W = int(lib().hostemu_jwait_windows(buf, float(bin_s)))
    jens = np.zeros((W + 1, 2, n_dc, 2, n_replicas))
    jens_hist = np.zeros((n_replicas, n_dc, 2, LAT_BINS), dtype=np.uint32)
    rows = np.zeros((W + 1, 3, n_dc, 2, n_replicas)) if waits else None
    hist = np.zeros((n_replicas, n_dc, 2, 2, LAT_BINS), dtype=np.uint32) if waits else None
    total = lib(uniform).hostemu_jwait_run_batch(buf, len(spec_bytes), n_replicas, seed0 & (2**64 - 1), chunk_events,
                                                 out.ctypes.data, rng_kind, float(bin_s), jens.ctypes.data,
                                                 jens_hist.ctypes.data, rows.ctypes.data if waits else None,
                                                 hist.ctypes.data if waits else None)
    if total < 0:
        raise ValueError("hostemu_jwait rejected the spec blob")
    return {"summary": out, "events": int(total), "jens": jens, "jens_hist": jens_hist, "rows": rows, "hist": hist}
