"""TEST-ONLY ctypes access to the host build of the device core with the cluster-log ensemble recorder
(tests/hostemu_ens/hostemu_ens.cpp)."""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_DIR = os.path.join(_HERE, "hostemu_ens")
_SO = os.path.join(_DIR, "_build", "libdcsim_hostemu_ens.so")
_SO_UNIFORM = os.path.join(_DIR, "_build", "libdcsim_hostemu_ens_uniform.so")
_SRCS = (os.path.join(_DIR, "hostemu_ens.cpp"), os.path.join(_DIR, "build.sh"),
         os.path.join(_HERE, "..", "distributed_cluster_gpus_b200", "csrc", "dcsim_core.cuh"),
         os.path.join(_HERE, "..", "include", "dcsim_b200.h"))
SUMMARY_K = 24 + 8 * 8
ENS_FIELDS = 11
_libs = {}


def _bind(path):
    L = C.CDLL(path)
    L.hostemu_ens_sizeof_spec.restype = C.c_size_t
    L.hostemu_ens_ticks.restype = C.c_uint32
    L.hostemu_ens_ticks.argtypes = [C.c_void_p]
    L.hostemu_ens_run_batch.restype = C.c_longlong
    L.hostemu_ens_run_batch.argtypes = [C.c_void_p, C.c_size_t, C.c_uint64, C.c_uint64, C.c_uint64, C.c_void_p, C.c_int,
                                        C.c_void_p, C.c_uint32]
    return L


def lib(uniform=False):
    if not _libs:
        if any(not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in _SRCS)
               for so in (_SO, _SO_UNIFORM)):
            subprocess.run([os.path.join(_DIR, "build.sh")], check=True, capture_output=True)
        _libs[False], _libs[True] = _bind(_SO), _bind(_SO_UNIFORM)
    return _libs[bool(uniform)]


def ens_ticks(spec_bytes):
    """The library's default tick capacity of the cluster-log ensemble (dcsim_ens_ticks of the device core)."""
    buf = C.create_string_buffer(spec_bytes, len(spec_bytes))
    return int(lib().hostemu_ens_ticks(buf))


def run_batch(spec_bytes, n_replicas, seed0, ens_cap, chunk_events=0, rng_kind=0, uniform=False):
    """-> {"summary": [n, SUMMARY_K], "events": int, "ensemble": [ens_cap, 11, n_dc, n] float64 or None}; ticks a
    replica did not reach stay NaN.  ens_cap = 0: recorder off."""
    out = np.zeros((n_replicas, SUMMARY_K))
    buf = C.create_string_buffer(spec_bytes, len(spec_bytes))
    n_dc = C.c_int32.from_buffer_copy(spec_bytes[16:20]).value      # dcsim_spec_t.n_dc
    ens = np.full((ens_cap, ENS_FIELDS, n_dc, n_replicas), np.nan) if ens_cap else None
    total = lib(uniform).hostemu_ens_run_batch(buf, len(spec_bytes), n_replicas, seed0 & (2**64 - 1), chunk_events,
                                               out.ctypes.data, rng_kind, ens.ctypes.data if ens is not None else None,
                                               ens_cap)
    if total < 0:
        raise ValueError("hostemu_ens rejected the spec blob")
    return {"summary": out, "events": int(total), "ensemble": ens}
