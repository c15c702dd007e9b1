"""TEST-ONLY ctypes access to the energy-cost probe of the stepped C oracle (tests/oracle_jobs/oracle_cost.c)."""
import ctypes as C
import os
import subprocess

import numpy as np

from distributed_cluster_gpus_b200 import spec as S

_HERE = os.path.dirname(os.path.abspath(__file__))
_DIR = os.path.join(_HERE, "oracle_jobs")
_SO = os.path.join(_DIR, "_build", "liboracle_cost.so")
_SRCS = (os.path.join(_DIR, "oracle_cost.c"), os.path.join(_DIR, "build_cost.sh"),
         os.path.join(_HERE, "..", "oracle", "dcsim_oracle.c"), os.path.join(_HERE, "..", "include", "dcsim_b200.h"))
_lib = None


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(_SO) or any(os.path.getmtime(s) > os.path.getmtime(_SO) for s in _SRCS):
            subprocess.run([os.path.join(_DIR, "build_cost.sh")], check=True, capture_output=True)
        L = C.CDLL(_SO)
        L.oraclecost_run.restype = C.c_longlong
        L.oraclecost_run.argtypes = [C.c_void_p, C.c_size_t, C.c_uint64, C.c_int, C.c_void_p]
        _lib = L
    return _lib


def oracle_energy_cost(spec_bytes, seed, rng_kind=0):
    """One replica's energy-cost column [cost_cols(n_dc)] from the oracle stepped one event at a time."""
    n_dc = S.Spec.from_buffer_copy(spec_bytes).n_dc
    row = np.zeros(S.cost_cols(n_dc))
    if lib().oraclecost_run(spec_bytes, len(spec_bytes), seed & (2**64 - 1), rng_kind, row.ctypes.data) < 0:
        raise ValueError("the oracle rejected the spec blob")
    return row
