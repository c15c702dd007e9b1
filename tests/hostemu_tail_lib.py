"""TEST-ONLY ctypes access to the host build of the device core with the per-run tail-latency recorder and its
selection pass (tests/hostemu_ens/hostemu_tail.cpp), and to the oracle's record of every created job
(tests/oracle_jobs/oracle_tail.c)."""
import ctypes as C
import os
import subprocess

import numpy as np

from distributed_cluster_gpus_b200 import ensemble as EN, spec as S

_HERE = os.path.dirname(os.path.abspath(__file__))
_DIR = os.path.join(_HERE, "hostemu_ens")
_SO = os.path.join(_DIR, "_build", "libdcsim_hostemu_tail.so")
_SO_UNIFORM = os.path.join(_DIR, "_build", "libdcsim_hostemu_tail_uniform.so")
_SRCS = (os.path.join(_DIR, "hostemu_tail.cpp"), os.path.join(_DIR, "build_tail.sh"),
         os.path.join(_HERE, "..", "distributed_cluster_gpus_b200", "csrc", "dcsim_core.cuh"),
         os.path.join(_HERE, "..", "include", "dcsim_b200.h"))
_ODIR = os.path.join(_HERE, "oracle_jobs")
_OSO = os.path.join(_ODIR, "_build", "liboracle_tail.so")
_OSRCS = (os.path.join(_ODIR, "oracle_tail.c"), os.path.join(_ODIR, "oracle_jobs.c"), os.path.join(_ODIR, "build_tail.sh"),
          os.path.join(_HERE, "..", "oracle", "dcsim_oracle.c"), os.path.join(_HERE, "..", "include", "dcsim_b200.h"))
SUMMARY_K = 24 + 8 * 8
_libs = {}

ORACLE_ROW_DTYPE = np.dtype([("jid", "<u4"), ("jtype", "<i4"), ("dc", "<i4"), ("finished", "<i4"), ("arrival", "<f8"),
                             ("xfer_done", "<f8"), ("start", "<f8"), ("finish", "<f8")])


def _stale(so, srcs):
    return not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in srcs)


def _bind(path):
    L = C.CDLL(path)
    vp = C.c_void_p
    L.hostemu_tail_set_test_time_quantum.argtypes = [C.c_double]
    L.hostemu_tail_cap_arr.restype = C.c_uint32
    L.hostemu_tail_cap_arr.argtypes = [vp]
    L.hostemu_tail_run_batch.restype = C.c_longlong
    L.hostemu_tail_run_batch.argtypes = [vp, C.c_size_t, C.c_uint64, C.c_uint64, C.c_uint64, vp, C.c_int, C.c_double,
                                         vp, vp, vp, vp, vp]
    L.hostemu_tail_select_synthetic.argtypes = [C.c_uint32, vp, vp, vp, vp, C.c_double, C.c_double, vp]
    return L


def lib(uniform=False):
    if not _libs.get(False):
        if _stale(_SO, _SRCS) or _stale(_SO_UNIFORM, _SRCS):
            subprocess.run([os.path.join(_DIR, "build_tail.sh")], check=True, capture_output=True)
        _libs[False], _libs[True] = _bind(_SO), _bind(_SO_UNIFORM)
    return _libs[bool(uniform)]


def oracle_lib():
    if "oracle" not in _libs:
        if _stale(_OSO, _OSRCS):
            subprocess.run([os.path.join(_ODIR, "build_tail.sh")], check=True, capture_output=True)
        L = C.CDLL(_OSO)
        L.oraclejobs_set_test_time_quantum.argtypes = [C.c_double]
        L.oracletail_run.restype = C.c_longlong
        L.oracletail_run.argtypes = [C.c_void_p, C.c_size_t, C.c_uint64, C.c_int, C.c_void_p, C.c_uint32]
        _libs["oracle"] = L
    return _libs["oracle"]


def set_test_time_quantum(q):
    """The tie hook (0 = off) in both the host builds and the oracle's run."""
    lib(False).hostemu_tail_set_test_time_quantum(float(q))
    lib(True).hostemu_tail_set_test_time_quantum(float(q))
    oracle_lib().oraclejobs_set_test_time_quantum(float(q))


def oracle_created(spec_bytes, seed, rng_kind=0, cap=400000):
    """One replica's created jobs in jid order (EN.TAIL_JOB_DTYPE; finish NaN: not finished by end_time) — the
    oracle's instants."""
    out = np.zeros(cap, dtype=ORACLE_ROW_DTYPE)
    buf = C.create_string_buffer(spec_bytes, len(spec_bytes))
    n = oracle_lib().oracletail_run(buf, len(spec_bytes), seed & (2**64 - 1), rng_kind, out.ctypes.data, cap)
    if n < 0:
        raise ValueError("oracle_tail rejected the spec blob")
    assert n <= cap, "raise cap"
    rows = out[:n]
    assert np.array_equal(rows["jid"], np.arange(1, n + 1))
    jobs = np.zeros(n, dtype=EN.TAIL_JOB_DTYPE)
    for f in ("jtype", "dc", "arrival", "xfer_done", "start", "finish"):
        jobs[f] = rows[f]
    assert np.all(np.isnan(jobs["finish"]) == (rows["finished"] == 0))
    return jobs


def jobs_from_slots(slots, arr_t, arr_tx, arr_meta, created):
    """One replica's created jobs (EN.TAIL_JOB_DTYPE) from its slot buffer [cap, 2] and the pre-pass / merge buffers
    [cap] — the instants the device itself recorded and ran the events at."""
    n = int(created)
    jobs = np.zeros(n, dtype=EN.TAIL_JOB_DTYPE)
    meta = np.asarray(arr_meta[:n], dtype=np.uint32)
    jobs["jtype"] = meta & 1
    jobs["dc"] = (meta >> 4) & 7
    jobs["arrival"], jobs["xfer_done"] = arr_t[:n], arr_tx[:n]
    jobs["start"], jobs["finish"] = slots[:n, 0], slots[:n, 1]
    return jobs


def run_batch(spec_bytes, n_replicas, seed0, chunk_events=0, rng_kind=0, uniform=False, sla_s=None, tail=True):
    """-> {"summary": [n, SUMMARY_K], "events": int, "slots": [n, cap, 2] or None, "cols": [tail cols, n] or None,
    "arr_t" / "arr_tx": [n, cap], "arr_meta": [n, cap] uint32}.  tail=False: the recorder off (the records stay lean)."""
    out = np.zeros((n_replicas, SUMMARY_K))
    buf = C.create_string_buffer(spec_bytes, len(spec_bytes))
    n_dc = C.c_int32.from_buffer_copy(spec_bytes[16:20]).value      # dcsim_spec_t.n_dc
    cap = int(lib().hostemu_tail_cap_arr(buf))
    slots = np.zeros((n_replicas, cap, 2)) if tail else None
    cols = np.zeros((S.tail_cols(n_dc), n_replicas)) if tail else None
    arr_t, arr_tx = np.zeros((n_replicas, cap)), np.zeros((n_replicas, cap))
    arr_meta = np.zeros((n_replicas, cap), dtype=np.uint32)
    ptr = lambda a: a.ctypes.data if a is not None else None  # noqa: E731
    total = lib(uniform).hostemu_tail_run_batch(buf, len(spec_bytes), n_replicas, seed0 & (2**64 - 1), chunk_events,
                                                out.ctypes.data, rng_kind, float("inf") if sla_s is None else float(sla_s),
                                                ptr(slots), ptr(cols), arr_t.ctypes.data, arr_tx.ctypes.data,
                                                arr_meta.ctypes.data)
    if total < 0:
        raise ValueError("hostemu_tail rejected the spec blob")
    return {"summary": out, "events": int(total), "slots": slots, "cols": cols, "arr_t": arr_t, "arr_tx": arr_tx,
            "arr_meta": arr_meta}


def select_synthetic(tx, start, finish, jtype=None, sla_s=None, status=0.0):
    """The selection pass alone over one replica of a 1-DC spec whose created jobs arrived at 0 with these xfer_done,
    start and finish instants (finish NaN: unfinished) -> its [tail cols] column values."""
    n = len(start)
    tx, start, finish = (np.ascontiguousarray(a, dtype=np.float64) for a in (tx, start, finish))
    jt = np.ascontiguousarray(np.zeros(n) if jtype is None else jtype, dtype=np.int32)
    cols = np.zeros(S.tail_cols(1))
    lib().hostemu_tail_select_synthetic(n, tx.ctypes.data, start.ctypes.data, finish.ctypes.data, jt.ctypes.data,
                                        float("inf") if sla_s is None else float(sla_s), float(status), cols.ctypes.data)
    return cols
