"""TEST-ONLY ctypes access to the single-lane host build of the device core (tests/hostemu/hostemu.cpp)."""
import ctypes as C
import os
import subprocess

import numpy as np

from distributed_cluster_gpus_b200 import engine as E, ensemble as EN, spec as S

_HERE = os.path.dirname(os.path.abspath(__file__))
_DIR = os.path.join(_HERE, "hostemu")
_SRCS = (os.path.join(_DIR, "hostemu.cpp"), os.path.join(_DIR, "build.sh"),
         os.path.join(_HERE, "..", "distributed_cluster_gpus_b200", "csrc", "dcsim_core.cuh"),
         os.path.join(_HERE, "..", "include", "dcsim_b200.h"))
_SOS = {name: os.path.join(_DIR, "_build", f"libdcsim_hostemu{suffix}.so")
        for name, suffix in (("plain", ""), ("uniform", "_uniform"), ("perturbed", "_perturbed"), ("smallring", "_smallring"))}
VARIANTS = ("plain", "uniform", "smallring")  # the builds that differ in the pre-pass / merge / loop code they run
TRACE_DTYPE = E.TRACE_DTYPE
HDR_DTYPE = np.dtype([("count", "<u4"), ("first_mask", "<u4"), ("rng_words", "<u4"), ("status", "<u4"), ("ml_count", "<u4"),
                      ("max_ahead", "<u4"), ("_pad", "<u4", (2,))])
_vp, _u32, _f64 = C.c_void_p, C.c_uint32, C.c_double


class Out(C.Structure):
    """hostemu_out_t: the outputs of one run, NULL when off."""
    _fields_ = [("summary", _vp), ("rec_replica", C.c_int64), ("trace", _vp), ("jobs", _vp), ("cluster", _vp),
                ("trace_cap", _u32), ("jobs_cap", _u32), ("cluster_cap", _u32), ("ens_cap", _u32),
                ("counts", _vp), ("layout", _vp), ("lat_hist", _vp), ("ens", _vp),
                ("jens", _vp), ("jens_hist", _vp), ("jens_bin", _f64), ("jwait", _vp), ("jwait_hist", _vp),
                ("jres", _vp), ("jres_mix", _vp), ("jres_hist", _vp), ("pp", _vp), ("pp_threshold", _f64),
                ("occ", _vp), ("tail", _vp), ("tail_cols", _vp), ("tail_sla", _f64), ("cost", _vp),
                ("arr_t", _vp), ("arr_raw", _vp), ("arr_meta", _vp), ("arr_pred", _vp), ("arr_tx", _vp),
                ("ml_t", _vp), ("ml_aux", _vp), ("ml_meta", _vp), ("arr_hdr", _vp), ("lists_only", C.c_int32)]


_libs = {}


def _bind(path):
    L = C.CDLL(path)
    for name in ("hostemu_sizeof_spec", "hostemu_sizeof_arrhdr", "hostemu_sizeof_out"):
        getattr(L, name).restype = C.c_size_t
    L.hostemu_merge_ring.restype = _u32
    L.hostemu_set_test_time_quantum.argtypes = [_f64]
    for name, res in (("hostemu_cap_arr", _u32), ("hostemu_ens_ticks", _u32), ("hostemu_pp_range", _f64),
                      ("hostemu_jres_g", _u32)):
        getattr(L, name).restype = res
        getattr(L, name).argtypes = [_vp]
    L.hostemu_jens_windows.restype = C.c_uint64
    L.hostemu_jens_windows.argtypes = [_vp, _f64]
    L.hostemu_energy_cost_window.restype = _f64
    L.hostemu_energy_cost_window.argtypes = [_f64]
    L.hostemu_current_hour.restype = C.c_int
    L.hostemu_current_hour.argtypes = [_f64]
    L.hostemu_compatible.restype = C.c_int
    L.hostemu_compatible.argtypes = [_vp, C.c_size_t, _vp, C.c_size_t, C.c_char_p, C.c_size_t]
    L.hostemu_run_batch.restype = C.c_longlong
    L.hostemu_run_batch.argtypes = [_vp, _vp, C.c_size_t, C.c_uint64, C.c_uint64, C.c_uint64, C.c_int, C.POINTER(Out)]
    L.hostemu_tail_select_synthetic.argtypes = [_u32, _vp, _vp, _vp, _vp, _f64, _f64, _vp]
    assert L.hostemu_sizeof_spec() == C.sizeof(S.Spec)
    assert L.hostemu_sizeof_arrhdr() == HDR_DTYPE.itemsize
    assert L.hostemu_sizeof_out() == C.sizeof(Out)
    return L


def lib(perturbed=False, smallring=False, uniform=False, variant=None):
    """The plain build, or: uniform=True the event-loop skeleton of the lane-group GPU builds (replicas switched off
    instead of leaving); perturbed=True the conditioning probe (every 5th pow() result moved by one ulp, see
    hostemu.cpp); smallring=True the list merge built with a one-chunk ring (its HBM fall-back paths do all the work).
    `variant`: any of those by name."""
    if not _libs:
        if any(not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in _SRCS)
               for so in _SOS.values()):
            subprocess.run([os.path.join(_DIR, "build.sh")], check=True, capture_output=True)
        for name, so in _SOS.items():
            _libs[name] = _bind(so)
    return _libs[variant or ("uniform" if uniform else "smallring" if smallring else "perturbed" if perturbed else "plain")]


def set_test_time_quantum(q):
    """TEST HOOK (dcsim_core.cuh dcsim_test_quantize): 0 = off."""
    lib()
    for L in _libs.values():
        L.hostemu_set_test_time_quantum(float(q))


def _spec(spec_bytes):
    return S.Spec.from_buffer_copy(spec_bytes)


def cap_arr(spec_bytes):
    return int(lib().hostemu_cap_arr(spec_bytes))


def ens_ticks(spec_bytes):
    """The library's default tick capacity of the cluster-log ensemble (dcsim_ens_ticks of the device core)."""
    return int(lib().hostemu_ens_ticks(spec_bytes))


def job_windows(spec_bytes, bin_s):
    """The library's window count for a resolved bin width (dcsim_jens_windows of the device core)."""
    return int(lib().hostemu_jens_windows(spec_bytes, float(bin_s)))


def power_range(spec_bytes):
    """The library's histogram range hi for a spec (dcsim_pp_range of the device core)."""
    return float(lib().hostemu_pp_range(spec_bytes))


def jres_g(spec_bytes):
    """G = DCSIM_JRES_G(max_gpus_per_job): the GPU-count rows of the job-resources mix."""
    return int(lib().hostemu_jres_g(spec_bytes))


def cost_window(t):
    """The energy-cost recorder's hour window k of instant t: 3600 k <= t < 3600 (k + 1) (dcsim_cost_window)."""
    return float(lib().hostemu_energy_cost_window(float(t)))


def current_hour(t):
    """The hour of day the handlers use at instant t (dcsim_current_hour, SIM:982-984)."""
    return int(lib().hostemu_current_hour(float(t)))


def occ_rows(n_dc):
    return 1 + S.OCC_FIELDS * n_dc + 2 * S.OCC_BINS * n_dc


def compatible(spec_a: bytes, spec_b: bytes):
    """(dcsim_arrival_inputs_equal, the first differing field or "")."""
    field = C.create_string_buffer(64)
    rc = lib().hostemu_compatible(spec_a, len(spec_a), spec_b, len(spec_b), field, len(field))
    if rc < 0:
        raise ValueError("hostemu rejected a spec blob")
    return bool(rc), field.value.decode()


def run_batch(spec_bytes, n_replicas, seed0, chunk_events=0, trace_cap=0, rec_replica=-1, job_dtype=None,
              jobs_cap=0, cluster_dtype=None, cluster_cap=0, rng_kind=0, perturbed=False, smallring=False, uniform=False,
              variant=None, run_spec=None, lat_hist=True, ens_cap=0, jens_bin=None, jwait=False, jres=False, pp=False,
              pp_threshold=float("inf"), occ=False, tail=False, tail_sla=None, cost=False, prepass=False,
              lists_only=False):
    """n replicas from keys seed0, seed0 + 1, ...: the pre-pass and the merge under `spec_bytes`, then the event loop of
    `run_spec` (default: the same spec; else a spec whose arrival inputs equal it) on those lists, in launches of
    `chunk_events` events (0: to the end).  The batch latency histogram is on unless lat_hist=False ("lat_hist"
    [n, 2, LAT_BINS]); every other recorder is off unless asked for, as in the library:

      ens_cap=T       "ens" [T, ENS_FIELDS, n_dc, n] (ticks a replica did not reach stay NaN)
      jens_bin=b      "jens" [W + 1, JENS_STORED, n_dc, 2, n], "jens_hist" [n, n_dc, 2, LAT_BINS]
      jwait=True      "jwait" [W + 1, JWAIT_STORED, n_dc, 2, n], "jwait_hist" [n, n_dc, 2 kinds, 2, LAT_BINS] (needs jens_bin)
      jres=True       "jres" [W + 1, JRES_STORED, n_dc, 2, n], "jres_mix" [n_dc, 2, G * MAX_FREQ + 1, n],
                      "jres_hist" [n_dc, 2, JRES_EBINS, n] (needs jens_bin)
      pp=True         "pp" [PP_FIELDS + n_dc + PP_BINS, n] over `pp_threshold`
      occ=True        "occ" [occ_rows(n_dc), n]
      tail=True       "tail" [n, cap_arr, 2], "tail_cols" [tail_cols(n_dc), n] under `tail_sla` (None: none)
      cost=True       "cost" [cost_cols(n_dc), n]

    plus trace / jobs / cluster of `rec_replica`.  prepass=True adds what the pre-pass and the merge left ("arr_t",
    "arr_raw" (the job sizes), "arr_meta", "arr_pred", "arr_tx": [n, cap_arr]; "ml_t", "ml_aux", "ml_meta":
    [n, 2 * cap_arr]; "hdr": [n] HDR_DTYPE; unwritten entries hold 0xee bytes); lists_only=True stops there."""
    run_spec = spec_bytes if run_spec is None else run_spec
    n_dc, cap = _spec(run_spec).n_dc, cap_arr(spec_bytes)
    o = Out(rec_replica=rec_replica, trace_cap=trace_cap, jobs_cap=jobs_cap, cluster_cap=cluster_cap, ens_cap=ens_cap,
            jens_bin=float(jens_bin or 0.0), pp_threshold=float(pp_threshold),
            tail_sla=float("inf") if tail_sla is None else float(tail_sla), lists_only=int(lists_only))
    res = {}

    def out(name, shape, dtype=np.float64, fill=0):
        res[name] = a = np.full(shape, fill, dtype=dtype)
        setattr(o, name, a.ctypes.data)
        return a

    out("summary", (n_replicas, S.SUMMARY_K))
    counts = out("counts", 4, np.uint32)
    layout = out("layout", 8, np.int32)
    for name, cap_, dtype in (("trace", trace_cap, TRACE_DTYPE), ("jobs", jobs_cap, job_dtype),
                              ("cluster", cluster_cap, cluster_dtype)):
        if dtype is not None:
            out(name, cap_, dtype)
            if not cap_:
                setattr(o, name, None)
    if lat_hist:
        out("lat_hist", (n_replicas, 2, E.LAT_BINS), np.uint32)
    if ens_cap:
        out("ens", (ens_cap, E.ENS_FIELDS, n_dc, n_replicas), fill=np.nan)
    if jens_bin is not None:
        W = job_windows(run_spec, jens_bin)
        out("jens", (W + 1, E.JENS_STORED, n_dc, 2, n_replicas))
        out("jens_hist", (n_replicas, n_dc, 2, E.LAT_BINS), np.uint32)
        if jwait:
            out("jwait", (W + 1, E.JWAIT_STORED, n_dc, 2, n_replicas))
            out("jwait_hist", (n_replicas, n_dc, 2, 2, E.LAT_BINS), np.uint32)
        if jres:
            out("jres", (W + 1, E.JRES_STORED, n_dc, 2, n_replicas))
            out("jres_mix", (n_dc, 2, jres_g(run_spec) * S.MAX_FREQ + 1, n_replicas), np.uint32)
            out("jres_hist", (n_dc, 2, E.JRES_EBINS, n_replicas), np.uint32)
    if pp:
        out("pp", (S.PP_FIELDS + n_dc + S.PP_BINS, n_replicas))
    if occ:
        out("occ", (occ_rows(n_dc), n_replicas))
    if tail:
        out("tail", (n_replicas, cap, 2))
        out("tail_cols", (S.tail_cols(n_dc), n_replicas))
    if cost:
        out("cost", (S.cost_cols(n_dc), n_replicas))
    if prepass or lists_only:
        for name in ("arr_t", "arr_raw", "arr_tx"):
            out(name, (n_replicas, cap))
        for name in ("arr_meta", "arr_pred"):
            out(name, (n_replicas, cap), np.uint32)
        for name in ("ml_t", "ml_aux"):
            out(name, (n_replicas, 2 * cap))
        out("ml_meta", (n_replicas, 2 * cap), np.uint32)
        res["hdr"] = np.zeros(n_replicas, dtype=HDR_DTYPE)
        o.arr_hdr = res["hdr"].ctypes.data
    total = lib(perturbed, smallring, uniform, variant).hostemu_run_batch(
        spec_bytes, run_spec, len(spec_bytes), n_replicas, seed0 & (2**64 - 1), chunk_events, rng_kind, C.byref(o))
    if total < 0:
        raise ValueError("hostemu rejected the spec blob(s)")
    res["events"] = int(total)
    res["layout"] = {"total_bytes": int(layout[0]), "cap_xfer": int(layout[1]), "cap_run": int(layout[2]),
                     "cap_q_inf": int(layout[3]), "cap_q_trn": int(layout[4])}
    for name, i, cap_ in (("trace", 0, trace_cap), ("jobs", 1, jobs_cap), ("cluster", 2, cluster_cap)):
        if name in res:
            res[name] = res[name][:min(int(counts[i]), cap_)]
    return res


def prepass(spec_bytes, n_replicas, seed0, rng_kind=0, variant="plain", quantum=0.0):
    """What the pre-pass and the merge leave, full rows (run_batch's prepass outputs).  `quantum`: the tie-quantizing
    test hook (dcsim_test_quantize), reset to 0 afterwards."""
    set_test_time_quantum(quantum)
    try:
        res = run_batch(spec_bytes, n_replicas, seed0, rng_kind=rng_kind, variant=variant, lists_only=True)
    finally:
        set_test_time_quantum(0.0)
    return {k: res[k] for k in ("arr_t", "arr_raw", "arr_meta", "arr_pred", "arr_tx", "ml_t", "ml_aux", "ml_meta", "hdr")}


def lists(spec_bytes, n_replicas, seed0, rng_kind=0):
    """-> (per replica (ml_t, ml_aux, ml_meta) trimmed to its ml_count, headers [n] HDR_DTYPE)."""
    d = run_batch(spec_bytes, n_replicas, seed0, rng_kind=rng_kind, lists_only=True)
    return [(d["ml_t"][r, :k], d["ml_aux"][r, :k], d["ml_meta"][r, :k]) for r, k in enumerate(d["hdr"]["ml_count"])], d["hdr"]


def jobs_from_slots(slots, arr_t, arr_tx, arr_meta, created):
    """One replica's created jobs (EN.TAIL_JOB_DTYPE) from its tail slots [cap, 2] and the pre-pass / merge buffers
    [cap] — the instants the device itself recorded and ran the events at."""
    n = int(created)
    jobs = np.zeros(n, dtype=EN.TAIL_JOB_DTYPE)
    meta = np.asarray(arr_meta[:n], dtype=np.uint32)
    jobs["jtype"] = meta & 1
    jobs["dc"] = (meta >> 4) & 7
    jobs["arrival"], jobs["xfer_done"] = arr_t[:n], arr_tx[:n]
    jobs["start"], jobs["finish"] = slots[:n, 0], slots[:n, 1]
    return jobs


def select_synthetic(tx, start, finish, jtype=None, sla_s=None, status=0.0):
    """The tail selection pass alone over one replica of a 1-DC spec whose created jobs arrived at 0 with these
    xfer_done, start and finish instants (finish NaN: unfinished) -> its [tail cols] column values."""
    n = len(start)
    tx, start, finish = (np.ascontiguousarray(a, dtype=np.float64) for a in (tx, start, finish))
    jt = np.ascontiguousarray(np.zeros(n) if jtype is None else jtype, dtype=np.int32)
    cols = np.zeros(S.tail_cols(1))
    lib().hostemu_tail_select_synthetic(n, tx.ctypes.data, start.ctypes.data, finish.ctypes.data, jt.ctypes.data,
                                        float("inf") if sla_s is None else float(sla_s), float(status), cols.ctypes.data)
    return cols
