"""TEST-ONLY ctypes access to the host build of shared arrival lists (tests/hostemu_pair/hostemu_pair.cpp)."""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_DIR = os.path.join(_HERE, "hostemu_pair")
_SO = os.path.join(_DIR, "_build", "libdcsim_hostemu_pair.so")
_SO_UNIFORM = os.path.join(_DIR, "_build", "libdcsim_hostemu_pair_uniform.so")
_SRCS = (os.path.join(_DIR, "hostemu_pair.cpp"), os.path.join(_DIR, "build.sh"),
         os.path.join(_HERE, "..", "distributed_cluster_gpus_b200", "csrc", "dcsim_core.cuh"),
         os.path.join(_HERE, "..", "include", "dcsim_b200.h"))
SUMMARY_K = 24 + 8 * 8
HDR_DTYPE = np.dtype([("count", "<u4"), ("first_mask", "<u4"), ("rng_words", "<u4"), ("status", "<u4"), ("ml_count", "<u4"),
                      ("max_ahead", "<u4"), ("_pad", "<u4", (2,))])
_libs = {}


def _bind(path):
    L = C.CDLL(path)
    vp, u64 = C.c_void_p, C.c_uint64
    L.hostemu_pair_sizeof_spec.restype = C.c_size_t
    L.hostemu_pair_sizeof_arrhdr.restype = C.c_size_t
    L.hostemu_pair_compatible.restype = C.c_int
    L.hostemu_pair_compatible.argtypes = [vp, C.c_size_t, vp, C.c_size_t, C.c_char_p, C.c_size_t]
    L.hostemu_pair_lists.restype = C.c_int
    L.hostemu_pair_lists.argtypes = [vp, C.c_size_t, u64, u64, C.c_int, vp, vp, vp, vp]
    L.hostemu_pair_run.restype = C.c_longlong
    L.hostemu_pair_run.argtypes = [vp, vp, C.c_size_t, u64, u64, u64, C.c_int, vp]
    assert L.hostemu_pair_sizeof_arrhdr() == HDR_DTYPE.itemsize
    return L


def lib(uniform=False):
    if not _libs:
        if any(not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in _SRCS)
               for so in (_SO, _SO_UNIFORM)):
            subprocess.run([os.path.join(_DIR, "build.sh")], check=True, capture_output=True)
        _libs[False], _libs[True] = _bind(_SO), _bind(_SO_UNIFORM)
    return _libs[bool(uniform)]


def compatible(spec_a: bytes, spec_b: bytes):
    """(dcsim_arrival_inputs_equal, the first differing field or "")."""
    field = C.create_string_buffer(64)
    rc = lib().hostemu_pair_compatible(spec_a, len(spec_a), spec_b, len(spec_b), field, len(field))
    if rc < 0:
        raise ValueError("hostemu_pair rejected a spec blob")
    return bool(rc), field.value.decode()


def _cap_arr(spec_bytes):
    cap = C.c_int32.from_buffer_copy(spec_bytes[-4:]).value          # dcsim_spec_t.cap_arrivals (the last field)
    return cap if cap > 0 else 16384


def lists(spec_bytes, n_replicas, seed0, rng_kind=0):
    """-> (per replica (ml_t, ml_aux, ml_meta) trimmed to its ml_count, headers [n] HDR_DTYPE)."""
    w = 2 * _cap_arr(spec_bytes)
    t, aux = np.zeros((n_replicas, w)), np.zeros((n_replicas, w))
    meta = np.zeros((n_replicas, w), dtype=np.uint32)
    hdr = np.zeros(n_replicas, dtype=HDR_DTYPE)
    rc = lib().hostemu_pair_lists(spec_bytes, len(spec_bytes), n_replicas, seed0 & (2**64 - 1), rng_kind, t.ctypes.data,
                                  aux.ctypes.data, meta.ctypes.data, hdr.ctypes.data)
    if rc < 0:
        raise ValueError("hostemu_pair rejected the spec blob")
    return [(t[r, :k], aux[r, :k], meta[r, :k]) for r, k in enumerate(hdr["ml_count"])], hdr


def run(spec_src, spec_run, n_replicas, seed0, chunk_events=0, rng_kind=0, uniform=False):
    """The event loop of spec_run on the lists drawn under spec_src -> {"summary": [n, SUMMARY_K], "events": int}."""
    out = np.zeros((n_replicas, SUMMARY_K))
    total = lib(uniform).hostemu_pair_run(spec_src, spec_run, len(spec_src), n_replicas, seed0 & (2**64 - 1), chunk_events,
                                          rng_kind, out.ctypes.data)
    if total < 0:
        raise ValueError("hostemu_pair rejected the specs")
    return {"summary": out, "events": int(total)}
