"""TEST-ONLY ctypes access to the host build of the device core with the job-resources recorder
(tests/hostemu_ens/hostemu_jres.cpp)."""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_DIR = os.path.join(_HERE, "hostemu_ens")
_SO = os.path.join(_DIR, "_build", "libdcsim_hostemu_jres.so")
_SO_UNIFORM = os.path.join(_DIR, "_build", "libdcsim_hostemu_jres_uniform.so")
_SRCS = (os.path.join(_DIR, "hostemu_jres.cpp"), os.path.join(_DIR, "build_jres.sh"),
         os.path.join(_HERE, "..", "distributed_cluster_gpus_b200", "csrc", "dcsim_core.cuh"),
         os.path.join(_HERE, "..", "include", "dcsim_b200.h"))
SUMMARY_K = 24 + 8 * 8
LAT_BINS = 128
MAX_FREQ = 16
EBINS = 128
_libs = {}


def _stale(so, srcs):
    return not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in srcs)


def _bind(path):
    L = C.CDLL(path)
    L.hostemu_jres_windows.restype = C.c_uint64
    L.hostemu_jres_windows.argtypes = [C.c_void_p, C.c_double]
    L.hostemu_jres_run_batch.restype = C.c_longlong
    L.hostemu_jres_run_batch.argtypes = [C.c_void_p, C.c_size_t, C.c_uint64, C.c_uint64, C.c_uint64, C.c_void_p,
                                         C.c_int, C.c_double, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                         C.c_void_p]
    return L


def lib(uniform=False):
    if not _libs:
        if _stale(_SO, _SRCS) or _stale(_SO_UNIFORM, _SRCS):
            subprocess.run([os.path.join(_DIR, "build_jres.sh")], check=True, capture_output=True)
        _libs[False], _libs[True] = _bind(_SO), _bind(_SO_UNIFORM)
    return _libs[bool(uniform)]


def mix_g(max_gpus_per_job):
    """G = DCSIM_JRES_G(max_gpus_per_job): the GPU-count rows of the mix (the last one takes g >= G)."""
    return min(max(int(max_gpus_per_job), 1), 32)


def run_batch(spec_bytes, n_replicas, seed0, bin_s, max_gpus_per_job, chunk_events=0, rng_kind=0, uniform=False,
              resources=True):
    """-> {"summary": [n, SUMMARY_K], "events": int, "jens": [W + 1, 2, n_dc, 2, n], "jens_hist": [n, n_dc, 2, LAT_BINS],
    "rows": [W + 1, 3, n_dc, 2, n] float64, "mix": [n_dc, 2, G * 16 + 1, n] uint32, "hist": [n_dc, 2, 128, n] uint32
    (the last three None with resources=False: the recorder off, the job ensemble on)."""
    out = np.zeros((n_replicas, SUMMARY_K))
    buf = C.create_string_buffer(spec_bytes, len(spec_bytes))
    n_dc = C.c_int32.from_buffer_copy(spec_bytes[16:20]).value      # dcsim_spec_t.n_dc
    W = int(lib().hostemu_jres_windows(buf, float(bin_s)))
    G = mix_g(max_gpus_per_job)
    jens = np.zeros((W + 1, 2, n_dc, 2, n_replicas))
    jens_hist = np.zeros((n_replicas, n_dc, 2, LAT_BINS), dtype=np.uint32)
    rows = np.zeros((W + 1, 3, n_dc, 2, n_replicas)) if resources else None
    mix = np.zeros((n_dc, 2, G * MAX_FREQ + 1, n_replicas), dtype=np.uint32) if resources else None
    hist = np.zeros((n_dc, 2, EBINS, n_replicas), dtype=np.uint32) if resources else None
    ptr = (lambda a: a.ctypes.data if a is not None else None)
    total = lib(uniform).hostemu_jres_run_batch(buf, len(spec_bytes), n_replicas, seed0 & (2**64 - 1), chunk_events,
                                                out.ctypes.data, rng_kind, float(bin_s), jens.ctypes.data,
                                                jens_hist.ctypes.data, ptr(rows), ptr(mix), ptr(hist))
    if total < 0:
        raise ValueError("hostemu_jres rejected the spec blob")
    return {"summary": out, "events": int(total), "jens": jens, "jens_hist": jens_hist, "rows": rows, "mix": mix,
            "hist": hist}
