"""TEST-ONLY ctypes access to the host build of the device core with the job-log ensemble recorder
(tests/hostemu_ens/hostemu_jens.cpp)."""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_DIR = os.path.join(_HERE, "hostemu_ens")
_SO = os.path.join(_DIR, "_build", "libdcsim_hostemu_jens.so")
_SO_UNIFORM = os.path.join(_DIR, "_build", "libdcsim_hostemu_jens_uniform.so")
_SRCS = (os.path.join(_DIR, "hostemu_jens.cpp"), os.path.join(_DIR, "build_jens.sh"),
         os.path.join(_HERE, "..", "distributed_cluster_gpus_b200", "csrc", "dcsim_core.cuh"),
         os.path.join(_HERE, "..", "include", "dcsim_b200.h"))
SUMMARY_K = 24 + 8 * 8
LAT_BINS = 128
_libs = {}


def _bind(path):
    L = C.CDLL(path)
    L.hostemu_jens_sizeof_spec.restype = C.c_size_t
    L.hostemu_jens_windows.restype = C.c_uint64
    L.hostemu_jens_windows.argtypes = [C.c_void_p, C.c_double]
    L.hostemu_jens_run_batch.restype = C.c_longlong
    L.hostemu_jens_run_batch.argtypes = [C.c_void_p, C.c_size_t, C.c_uint64, C.c_uint64, C.c_uint64, C.c_void_p, C.c_int,
                                         C.c_double, C.c_void_p, C.c_void_p, C.c_void_p]
    return L


def lib(uniform=False):
    if not _libs:
        if any(not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in _SRCS)
               for so in (_SO, _SO_UNIFORM)):
            subprocess.run([os.path.join(_DIR, "build_jens.sh")], check=True, capture_output=True)
        _libs[False], _libs[True] = _bind(_SO), _bind(_SO_UNIFORM)
    return _libs[bool(uniform)]


def job_windows(spec_bytes, bin_s):
    """The library's window count for a resolved bin width (dcsim_jens_windows of the device core)."""
    buf = C.create_string_buffer(spec_bytes, len(spec_bytes))
    return int(lib().hostemu_jens_windows(buf, float(bin_s)))


def run_batch(spec_bytes, n_replicas, seed0, bin_s, chunk_events=0, rng_kind=0, uniform=False, record=True):
    """-> {"summary": [n, SUMMARY_K], "events": int, "rows": [W + 1, 2, n_dc, 2, n] float64 or None,
    "hist": [n, n_dc, 2, LAT_BINS] uint32 or None, "lat_hist": [n, 2, LAT_BINS] uint32 (the batch histogram)}.
    record=False: the job recorder off (the batch histogram stays on)."""
    out = np.zeros((n_replicas, SUMMARY_K))
    buf = C.create_string_buffer(spec_bytes, len(spec_bytes))
    n_dc = C.c_int32.from_buffer_copy(spec_bytes[16:20]).value      # dcsim_spec_t.n_dc
    W = job_windows(spec_bytes, bin_s)
    rows = np.zeros((W + 1, 2, n_dc, 2, n_replicas)) if record else None
    hist = np.zeros((n_replicas, n_dc, 2, LAT_BINS), dtype=np.uint32) if record else None
    lat_hist = np.zeros((n_replicas, 2, LAT_BINS), dtype=np.uint32)
    total = lib(uniform).hostemu_jens_run_batch(buf, len(spec_bytes), n_replicas, seed0 & (2**64 - 1), chunk_events,
                                                out.ctypes.data, rng_kind, float(bin_s),
                                                rows.ctypes.data if record else None,
                                                hist.ctypes.data if record else None, lat_hist.ctypes.data)
    if total < 0:
        raise ValueError("hostemu_jens rejected the spec blob")
    return {"summary": out, "events": int(total), "rows": rows, "hist": hist, "lat_hist": lat_hist}
