"""TEST-ONLY ctypes access to the host build of shared arrival lists (tests/hostemu_pair/hostemu_pair.cpp)."""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_DIR = os.path.join(_HERE, "hostemu_pair")
_SO = os.path.join(_DIR, "_build", "libdcsim_hostemu_pair.so")
_SO_UNIFORM = os.path.join(_DIR, "_build", "libdcsim_hostemu_pair_uniform.so")
_SO_SMALLRING = os.path.join(_DIR, "_build", "libdcsim_hostemu_pair_smallring.so")  # DCSIM_MERGE_RING = 32
VARIANTS = ("plain", "uniform", "smallring")
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
    L.hostemu_pair_prepass.restype = C.c_int
    L.hostemu_pair_prepass.argtypes = [vp, C.c_size_t, u64, u64, C.c_int] + [vp] * 9
    L.hostemu_pair_merge_ring.restype = C.c_uint32
    L.hostemu_pair_set_test_time_quantum.restype = None
    L.hostemu_pair_set_test_time_quantum.argtypes = [C.c_double]
    assert L.hostemu_pair_sizeof_arrhdr() == HDR_DTYPE.itemsize
    return L


def lib(uniform=False, variant=None):
    """The plain build, or the warp-uniform one (uniform=True), or any of VARIANTS by name."""
    if not _libs:
        if any(not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in _SRCS)
               for so in (_SO, _SO_UNIFORM, _SO_SMALLRING)):
            subprocess.run([os.path.join(_DIR, "build.sh")], check=True, capture_output=True)
        for name, so in zip(VARIANTS, (_SO, _SO_UNIFORM, _SO_SMALLRING)):
            _libs[name] = _bind(so)
    return _libs[variant or ("uniform" if uniform else "plain")]


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


def prepass(spec_bytes, n_replicas, seed0, rng_kind=0, variant="plain", quantum=0.0):
    """What the pre-pass and the merge leave, full rows: {"arr_t", "arr_raw" (the job sizes), "arr_meta", "arr_pred",
    "arr_tx": [n, cap_arr]; "ml_t", "ml_aux", "ml_meta": [n, 2 * cap_arr]; "hdr": [n] HDR_DTYPE}.  `quantum`: the
    tie-quantizing test hook (dcsim_test_quantize), reset to 0 afterwards."""
    cap = _cap_arr(spec_bytes)
    out = {"arr_t": np.zeros((n_replicas, cap)), "arr_raw": np.zeros((n_replicas, cap)),
           "arr_meta": np.zeros((n_replicas, cap), np.uint32), "arr_pred": np.zeros((n_replicas, cap), np.uint32),
           "arr_tx": np.zeros((n_replicas, cap)), "ml_t": np.zeros((n_replicas, 2 * cap)),
           "ml_aux": np.zeros((n_replicas, 2 * cap)), "ml_meta": np.zeros((n_replicas, 2 * cap), np.uint32),
           "hdr": np.zeros(n_replicas, dtype=HDR_DTYPE)}
    L = lib(variant=variant)
    L.hostemu_pair_set_test_time_quantum(float(quantum))
    try:
        rc = L.hostemu_pair_prepass(spec_bytes, len(spec_bytes), n_replicas, seed0 & (2**64 - 1), rng_kind,
                                    *(out[k].ctypes.data for k in ("arr_t", "arr_raw", "arr_meta", "arr_pred", "arr_tx",
                                                                  "ml_t", "ml_aux", "ml_meta", "hdr")))
    finally:
        L.hostemu_pair_set_test_time_quantum(0.0)
    if rc < 0:
        raise ValueError("hostemu_pair rejected the spec blob")
    return out


def run(spec_src, spec_run, n_replicas, seed0, chunk_events=0, rng_kind=0, uniform=False):
    """The event loop of spec_run on the lists drawn under spec_src -> {"summary": [n, SUMMARY_K], "events": int}."""
    out = np.zeros((n_replicas, SUMMARY_K))
    total = lib(uniform).hostemu_pair_run(spec_src, spec_run, len(spec_src), n_replicas, seed0 & (2**64 - 1), chunk_events,
                                          rng_kind, out.ctypes.data)
    if total < 0:
        raise ValueError("hostemu_pair rejected the specs")
    return {"summary": out, "events": int(total)}
