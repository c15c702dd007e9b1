"""TEST-ONLY ctypes access to the host build with the energy-cost recorder (tests/hostemu_cost/hostemu_cost.cpp): the
host emulation of tests/hostemu_lib.py, run through its own run_batch, with the recorder's columns added."""
import ctypes as C
import os
import subprocess

import numpy as np

import hostemu_lib as H
from distributed_cluster_gpus_b200 import spec as S

_HERE = os.path.dirname(os.path.abspath(__file__))
_DIR = os.path.join(_HERE, "hostemu_cost")
_SRCS = (os.path.join(_DIR, "hostemu_cost.cpp"), os.path.join(_DIR, "build.sh"), os.path.join(_HERE, "hostemu", "hostemu.cpp"),
         os.path.join(_HERE, "..", "distributed_cluster_gpus_b200", "csrc", "dcsim_core.cuh"),
         os.path.join(_HERE, "..", "include", "dcsim_b200.h"))
_SOS = {False: os.path.join(_DIR, "_build", "libdcsim_hostemu_cost.so"),
        True: os.path.join(_DIR, "_build", "libdcsim_hostemu_cost_uniform.so")}
_libs = {}


def lib(uniform=False):
    """The plain build, or uniform=True the warp-uniform event-loop skeleton of the lane-group GPU builds."""
    if not _libs:
        if any(not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in _SRCS)
               for so in _SOS.values()):
            subprocess.run([os.path.join(_DIR, "build.sh")], check=True, capture_output=True)
        for k, so in _SOS.items():
            L = C.CDLL(so)
            L.hostemu_cost_run_batch.restype = C.c_longlong
            L.hostemu_cost_run_batch.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_uint64, C.c_uint64, C.c_uint64,
                                                 C.c_int, C.POINTER(H.Out), C.c_void_p]
            L.hostemu_sizeof_out.restype = C.c_size_t
            assert L.hostemu_sizeof_out() == C.sizeof(H.Out)
            L.hostemu_cost_window.restype = C.c_double
            L.hostemu_cost_window.argtypes = [C.c_double]
            L.hostemu_current_hour.restype = C.c_int
            L.hostemu_current_hour.argtypes = [C.c_double]
            _libs[k] = L
    return _libs[bool(uniform)]


class _WithCost:
    """What hostemu_lib.run_batch calls as its library: hostemu_run_batch, routed to this build with `cost` as output."""

    def __init__(self, L, cost):
        self._L, self._cost = L, cost

    def hostemu_run_batch(self, *args):
        return self._L.hostemu_cost_run_batch(*args, self._cost.ctypes.data)


def run_batch(spec_bytes, n_replicas, seed0, cost=False, uniform=False, **kw):
    """hostemu_lib.run_batch (same keywords and results) with, when ``cost``, "cost" [cost_cols(n_dc), n] added: the
    energy-cost recorder's columns.  cost=False is hostemu_lib.run_batch itself."""
    if not cost:
        return H.run_batch(spec_bytes, n_replicas, seed0, uniform=uniform, **kw)
    n_dc = S.Spec.from_buffer_copy(spec_bytes).n_dc
    out = np.zeros((S.cost_cols(n_dc), n_replicas))
    H.lib()                                     # the base builds first: run_batch sizes its buffers through them
    key = "cost_uniform" if uniform else "cost_plain"
    H._libs[key] = _WithCost(lib(uniform), out)
    try:
        res = H.run_batch(spec_bytes, n_replicas, seed0, variant=key, **kw)
    finally:
        del H._libs[key]
    res["cost"] = out
    return res


def cost_window(t):
    """The energy-cost recorder's hour window k of instant t: 3600 k <= t < 3600 (k + 1) (dcsim_cost_window)."""
    return float(lib().hostemu_cost_window(float(t)))


def current_hour(t):
    """The hour of day the handlers use at instant t (dcsim_current_hour, SIM:982-984)."""
    return int(lib().hostemu_current_hour(float(t)))
