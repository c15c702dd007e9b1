"""TEST-ONLY ctypes access to the host build of the device core with the power-profile recorder
(tests/hostemu_ens/hostemu_pp.cpp)."""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_DIR = os.path.join(_HERE, "hostemu_ens")
_SO = os.path.join(_DIR, "_build", "libdcsim_hostemu_pp.so")
_SO_UNIFORM = os.path.join(_DIR, "_build", "libdcsim_hostemu_pp_uniform.so")
_SRCS = (os.path.join(_DIR, "hostemu_pp.cpp"), os.path.join(_DIR, "build_pp.sh"),
         os.path.join(_HERE, "..", "distributed_cluster_gpus_b200", "csrc", "dcsim_core.cuh"),
         os.path.join(_HERE, "..", "include", "dcsim_b200.h"))
SUMMARY_K = 24 + 8 * 8
PP_FIELDS = 8
PP_BINS = 1024
_libs = {}


def _bind(path):
    L = C.CDLL(path)
    L.hostemu_pp_sizeof_spec.restype = C.c_size_t
    L.hostemu_pp_range.restype = C.c_double
    L.hostemu_pp_range.argtypes = [C.c_void_p]
    L.hostemu_pp_run_batch.restype = C.c_longlong
    L.hostemu_pp_run_batch.argtypes = [C.c_void_p, C.c_size_t, C.c_uint64, C.c_uint64, C.c_uint64, C.c_void_p, C.c_int,
                                       C.c_double, C.c_void_p]
    return L


def lib(uniform=False):
    if not _libs:
        if any(not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in _SRCS)
               for so in (_SO, _SO_UNIFORM)):
            subprocess.run([os.path.join(_DIR, "build_pp.sh")], check=True, capture_output=True)
        _libs[False], _libs[True] = _bind(_SO), _bind(_SO_UNIFORM)
    return _libs[bool(uniform)]


def power_range(spec_bytes):
    """The library's histogram range hi for a spec (dcsim_pp_range of the device core)."""
    buf = C.create_string_buffer(spec_bytes, len(spec_bytes))
    return float(lib().hostemu_pp_range(buf))


def run_batch(spec_bytes, n_replicas, seed0, threshold=float("inf"), chunk_events=0, rng_kind=0, uniform=False,
              record=True):
    """-> {"summary": [n, SUMMARY_K], "events": int, "rows": [PP_FIELDS + n_dc + PP_BINS, n] float64 or None}."""
    out = np.zeros((n_replicas, SUMMARY_K))
    buf = C.create_string_buffer(spec_bytes, len(spec_bytes))
    n_dc = C.c_int32.from_buffer_copy(spec_bytes[16:20]).value      # dcsim_spec_t.n_dc
    rows = np.zeros((PP_FIELDS + n_dc + PP_BINS, n_replicas)) if record else None
    total = lib(uniform).hostemu_pp_run_batch(buf, len(spec_bytes), n_replicas, seed0 & (2**64 - 1), chunk_events,
                                              out.ctypes.data, rng_kind, float(threshold),
                                              rows.ctypes.data if record else None)
    if total < 0:
        raise ValueError("hostemu_pp rejected the spec blob")
    return {"summary": out, "events": int(total), "rows": rows}
