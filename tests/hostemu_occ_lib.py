"""TEST-ONLY ctypes access to the host build of the device core with the occupancy recorder
(tests/hostemu_ens/hostemu_occ.cpp) and to the oracle-stepping occupancy checkers (tests/oracle_jobs/oracle_occ.c)."""
import ctypes as C
import os
import subprocess

import numpy as np

import hostemu_jwait_lib as HW

_HERE = os.path.dirname(os.path.abspath(__file__))
_DIR = os.path.join(_HERE, "hostemu_ens")
_SO = os.path.join(_DIR, "_build", "libdcsim_hostemu_occ.so")
_SO_UNIFORM = os.path.join(_DIR, "_build", "libdcsim_hostemu_occ_uniform.so")
_SRCS = (os.path.join(_DIR, "hostemu_occ.cpp"), os.path.join(_DIR, "build_occ.sh"),
         os.path.join(_HERE, "..", "distributed_cluster_gpus_b200", "csrc", "dcsim_core.cuh"),
         os.path.join(_HERE, "..", "include", "dcsim_b200.h"))
_ODIR = os.path.join(_HERE, "oracle_jobs")
_OSO = os.path.join(_ODIR, "_build", "liboracle_occ.so")
_OSRCS = (os.path.join(_ODIR, "oracle_occ.c"), os.path.join(_ODIR, "build_occ.sh"),
          os.path.join(_HERE, "..", "oracle", "dcsim_oracle.c"), os.path.join(_HERE, "..", "include", "dcsim_b200.h"))
SUMMARY_K = 24 + 8 * 8
OCC_FIELDS = 8
OCC_BINS = 128
PP_FIELDS = 8
PP_BINS = 1024
_libs = {}
_oracle_libs = {}

REACHED_DTYPE = np.dtype([("jid", "<u4"), ("dc", "<i4"), ("jtype", "<i4"), ("pad", "<u4"), ("xfer_done", "<f8"),
                          ("start", "<f8"), ("finish", "<f8")])


def _bind(path):
    L = C.CDLL(path)
    L.hostemu_occ_set_test_time_quantum.argtypes = [C.c_double]
    L.hostemu_occ_run_batch.restype = C.c_longlong
    L.hostemu_occ_run_batch.argtypes = [C.c_void_p, C.c_size_t, C.c_uint64, C.c_uint64, C.c_uint64, C.c_void_p, C.c_int,
                                        C.c_void_p, C.c_void_p]
    return L


def lib(uniform=False):
    if not _libs:
        if HW._stale(_SO, _SRCS) or HW._stale(_SO_UNIFORM, _SRCS):
            subprocess.run([os.path.join(_DIR, "build_occ.sh")], check=True, capture_output=True)
        _libs[False], _libs[True] = _bind(_SO), _bind(_SO_UNIFORM)
    return _libs[bool(uniform)]


def _oracle():
    if "oracle" not in _oracle_libs:
        if HW._stale(_OSO, _OSRCS):
            subprocess.run([os.path.join(_ODIR, "build_occ.sh")], check=True, capture_output=True)
        L = C.CDLL(_OSO)
        L.oracleocc_set_test_time_quantum.argtypes = [C.c_double]
        L.oracleocc_occupancy.restype = C.c_longlong
        L.oracleocc_occupancy.argtypes = [C.c_void_p, C.c_size_t, C.c_uint64, C.c_int, C.c_void_p]
        L.oracleocc_reached.restype = C.c_longlong
        L.oracleocc_reached.argtypes = [C.c_void_p, C.c_size_t, C.c_uint64, C.c_int, C.c_void_p, C.c_uint32]
        _oracle_libs["oracle"] = L
    return _oracle_libs["oracle"]


def set_test_time_quantum(q):
    """The tie hook (0 = off) in the host build and in the oracle."""
    lib(False).hostemu_occ_set_test_time_quantum(float(q))
    lib(True).hostemu_occ_set_test_time_quantum(float(q))
    _oracle().oracleocc_set_test_time_quantum(float(q))


def n_rows(n_dc):
    return 1 + OCC_FIELDS * n_dc + 2 * OCC_BINS * n_dc


def _n_dc(spec_bytes):
    return C.c_int32.from_buffer_copy(spec_bytes[16:20]).value      # dcsim_spec_t.n_dc


def oracle_occupancy(spec_bytes, seed, rng_kind=0):
    """One replica's occupancy columns [n_rows(n_dc)] from the oracle stepped one event at a time."""
    row = np.zeros(n_rows(_n_dc(spec_bytes)))
    buf = C.create_string_buffer(spec_bytes, len(spec_bytes))
    if _oracle().oracleocc_occupancy(buf, len(spec_bytes), seed & (2**64 - 1), rng_kind, row.ctypes.data) < 0:
        raise ValueError("oracle_jobs rejected the spec blob")
    return row


def oracle_reached(spec_bytes, seed, rng_kind=0, cap=400000):
    """Every job that reached its DC (REACHED_DTYPE, xfer_done order); start / finish +inf when not by end_time."""
    out = np.zeros(cap, dtype=REACHED_DTYPE)
    buf = C.create_string_buffer(spec_bytes, len(spec_bytes))
    n = _oracle().oracleocc_reached(buf, len(spec_bytes), seed & (2**64 - 1), rng_kind, out.ctypes.data, cap)
    if n < 0:
        raise ValueError("oracle_jobs rejected the spec blob")
    assert n <= cap, "raise cap"
    return out[:n]


def run_batch(spec_bytes, n_replicas, seed0, chunk_events=0, rng_kind=0, uniform=False, occ=True, pp=False):
    """-> {"summary": [n, SUMMARY_K], "events": int, "rows": [n_rows(n_dc), n] float64 or None (occ=False),
    "pp": [PP_FIELDS + n_dc + PP_BINS, n] or None (pp=False; threshold none)}."""
    out = np.zeros((n_replicas, SUMMARY_K))
    buf = C.create_string_buffer(spec_bytes, len(spec_bytes))
    n_dc = _n_dc(spec_bytes)
    rows = np.zeros((n_rows(n_dc), n_replicas)) if occ else None
    pprows = np.zeros((PP_FIELDS + n_dc + PP_BINS, n_replicas)) if pp else None
    total = lib(uniform).hostemu_occ_run_batch(buf, len(spec_bytes), n_replicas, seed0 & (2**64 - 1), chunk_events,
                                               out.ctypes.data, rng_kind, rows.ctypes.data if occ else None,
                                               pprows.ctypes.data if pp else None)
    if total < 0:
        raise ValueError("hostemu_occ rejected the spec blob")
    return {"summary": out, "events": int(total), "rows": rows, "pp": pprows}
