"""TEST-ONLY ctypes access to the stepped oracle's per-arrival record (tests/oracle_jobs/oracle_lists.c)."""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_DIR = os.path.join(_HERE, "oracle_jobs")
_SO = os.path.join(_DIR, "_build", "liboracle_lists.so")
_SRCS = (os.path.join(_DIR, "oracle_lists.c"), os.path.join(_DIR, "build.sh"),
         os.path.join(_HERE, "..", "oracle", "dcsim_oracle.c"), os.path.join(_HERE, "..", "include", "dcsim_b200.h"))
ROW_DTYPE = np.dtype([("t", "<f8"), ("size", "<f8"), ("tx", "<f8"), ("stream", "<u4"), ("dc", "<i4"), ("pred", "<u4"),
                      ("next", "<u4")])
_lib = None


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(_SO) or any(os.path.getmtime(s) > os.path.getmtime(_SO) for s in _SRCS):
            subprocess.run([os.path.join(_DIR, "build.sh")], check=True, capture_output=True)
        L = C.CDLL(_SO)
        L.oraclelists_set_test_time_quantum.argtypes = [C.c_double]
        L.oraclelists_run.restype = C.c_longlong
        L.oraclelists_run.argtypes = [C.c_void_p, C.c_size_t, C.c_uint64, C.c_int, C.c_void_p, C.c_uint32, C.c_void_p]
        _lib = L
    return _lib


def arrivals(spec_bytes, seed, rng_kind=0, quantum=0.0, cap=1 << 20):
    """One replica's arrivals as the oracle processes them -> (rows ROW_DTYPE, first_mask, rng_words).  `quantum`: the
    oracle's tie-quantizing hook, reset to 0 afterwards."""
    rows = np.zeros(cap, dtype=ROW_DTYPE)
    info = np.zeros(2, dtype=np.uint64)
    L = lib()
    L.oraclelists_set_test_time_quantum(float(quantum))
    try:
        n = L.oraclelists_run(spec_bytes, len(spec_bytes), seed & (2**64 - 1), rng_kind, rows.ctypes.data, cap,
                              info.ctypes.data)
    finally:
        L.oraclelists_set_test_time_quantum(0.0)
    if n < 0:
        raise ValueError("oracle_lists rejected the spec blob")
    assert n <= cap, "more arrivals than rows"
    return rows[:n], int(info[0]), int(info[1])
